"""The halo shift-GEMM epilogue (conv3x3.cu) with one or two staging tiles, against fp64 torch.

The halo kernel stages each output tile in shared memory and writes it with a TMA store.  Where the operand ring still
gets two slots it alternates two staging tiles, so a tile's epilogue does not wait for the store of the tile before to
drain; the 256-wide tiles of 14x14 layers keep one.  The training epilogues (statistics-fusing forward pass, data
gradient with or without a residual) run branch-free, the others (bias, residual + ReLU) through the generic variant.
The cases here cover each of these on the schedule it runs on: statistics, residual + ReLU, bias, the data gradient,
the 4x4 ImageNet stem, window (grouped) mode, an odd tile count per CTA, a ragged last row tile (H % RT != 0) and a
256-wide tile with one staging tile.  Each runs through the sweep's tier-1 (exact, bit for bit) and tier-2
(rounding-realistic) checks, and test_schedule_coverage fails when a case no longer takes the schedule it is meant to
test.
"""
import pytest

import test_gpu_conv_sweep as cs_sweep

pytestmark = pytest.mark.gpu


def _images(tiles, tiles_per_img):
    return -(-tiles // tiles_per_img)


def cases(sm):
    """name -> case (test_gpu_conv_sweep._case), shaped from the SM count: T = 2S + S/2 m-tiles give the busiest CTA
    three tiles, 4S + S/2 five"""
    h = sm // 2
    t3, t5 = 2 * sm + h, 4 * sm + h
    case = cs_sweep._case
    return {
        # 28 x 28: 4 rows per tile, 7 tiles per image
        'stats_two_bufs_w64': case(_images(t5, 7), 28, 28, 64, 64, 3, 3, 1, 1, ops='f', stats=True),
        'res_relu_two_bufs_w128': case(_images(t3, 7), 28, 28, 64, 128, 3, 3, 1, 1, ops='fd', res=True, act=1),
        'bias_two_bufs_w64': case(_images(t3, 7), 28, 28, 64, 64, 3, 3, 1, 1, ops='f', bias=True),
        # layer1's data gradient: 56 x 56, 2 rows per tile
        'dgrad_two_bufs_56': case(_images(t3, 28), 56, 56, 64, 64, 3, 3, 1, 1, ops='d'),
        # the ImageNet stem: 115 x 115 x 16 bordered source, one output row per tile
        'stem_halo4_stats': case(_images(t3, 112), 115, 115, 16, 64, 4, 4, 1, 0, ops='f', stats=True),
        # window mode: two 64-channel windows, each walked by sm / 2 CTAs
        'window_stats_two_bufs': case(_images(2 * h + 1, 7), 28, 28, 128, 128, 3, 3, 1, 1, ops='fd', stats=True,
                                      groups=32, window=64),
        # 14 x 14: 8 rows per tile, the second tile of an image has 6
        'ragged_rows_14_stats': case(_images(t3, 2), 14, 14, 64, 64, 3, 3, 1, 1, ops='fd', stats=True),
        'one_buf_w256_14': case(_images(t3, 2), 14, 14, 256, 256, 3, 3, 1, 1, ops='fd', stats=True, res_d=True),
    }


_NAMES = list(cases(132))


def _get(name):
    return cases(cs_sweep._sm_count())[name]


@pytest.mark.parametrize('name', _NAMES)
def test_tier1_exact(name):
    cs_sweep.check_exact(_get(name), 'halo_epilogue_' + name)


@pytest.mark.parametrize('name', _NAMES)
def test_tier2_rounding(name):
    cs_sweep.check_rounding(_get(name), 'halo_epilogue_' + name)


def _max_tiles(r):
    """the busiest CTA's tile count of a halo launch record"""
    if r['diag']:
        return -(-r['m_tiles'] // (r['grid'] // r['n_tiles']))
    return -(-(r['m_tiles'] * r['n_tiles']) // r['grid'])


def _ragged(r):
    """the last row tile of each image is shorter than the others (H % RT != 0)"""
    wp = r['W'] + (3 if r['taps'] == 16 else 2)
    rt = min(128 // wp, r['H'])
    return r['H'] % rt != 0


def test_schedule_coverage(monkeypatch, capfd):
    """every case takes the staging schedule it is meant to test (per-launch debug line field epi_bufs)"""
    cs_sweep.enable_debug_lines(monkeypatch)
    sm = cs_sweep._sm_count()
    recs = cs_sweep.coverage_records(cases(sm), capfd)
    two = lambda r: r['kind'] == 'halo' and r['epi_bufs'] == 2
    one = lambda r: r['kind'] == 'halo' and r['epi_bufs'] == 1
    req = {
        'two staging tiles, statistics': lambda r: two(r) and r['taps'] == 9 and r['stats'],
        'two staging tiles, >= 5 tiles per CTA': lambda r: two(r) and _max_tiles(r) >= 5,
        'two staging tiles, odd tile count per CTA': lambda r: two(r) and _max_tiles(r) >= 3 and _max_tiles(r) % 2,
        'two staging tiles, fprop residual + ReLU': lambda r: two(r) and r['dir'] == 0 and r['res'] and r['act'] == 1,
        'two staging tiles, dgrad residual': lambda r: two(r) and r['dir'] == 1 and r['res'],
        'two staging tiles, bias': lambda r: two(r) and r['bias'],
        'two staging tiles, dgrad': lambda r: two(r) and r['dir'] == 1 and not r['res'],
        'two staging tiles, 4x4 stem + statistics': lambda r: two(r) and r['taps'] == 16 and r['stats'],
        'two staging tiles, streamed weights': lambda r: two(r) and r['bstat'] == 0,
        'two staging tiles, window mode': lambda r: two(r) and r['diag'] and _max_tiles(r) >= 2,
        'two staging tiles, ragged last row tile': lambda r: two(r) and _ragged(r) and _max_tiles(r) >= 3,
        'one staging tile, block_n 256 + statistics': lambda r: one(r) and r['block_n'] == 256 and r['stats'],
        'one staging tile, dgrad residual': lambda r: one(r) and r['dir'] == 1 and r['res'],
    }
    missing = [label for label, pred in req.items() if not any(pred(r) for r in recs)]
    assert not missing, 'staging schedules no longer reached (SMs=%d): %s' % (sm, missing)
