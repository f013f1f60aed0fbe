"""The implicit-GEMM TMA-store epilogue with two staging tiles per warpgroup, against fp64 torch.

A tile that stores at least as many bytes as it loads (1x1 layers with C <= 128 expanding to more output channels, and
their data gradients) is staged through two alternating shared-memory tiles per consumer warpgroup, so that its
epilogue does not wait for the previous TMA store to drain.  The sweep of test_gpu_conv_sweep.py reaches that schedule
for plain, biased and statistics-fusing forward convolutions; the cases here add the residual of the data gradient
(the engine's bottleneck-entry 1x1 layers), the fused residual + ReLU and bias + ReLU6 forward epilogues with two
staging tiles, and a deep-K layer that keeps one staging tile.  Each case runs through the sweep's tier-1 (exact, bit
for bit) and tier-2 (rounding-realistic) checks, and test_schedule_coverage fails when a case no longer takes the
schedule it is meant to test.
"""
import pytest

import test_gpu_conv_sweep as cs_sweep

pytestmark = pytest.mark.gpu


def cases(sm):
    """name -> case (test_gpu_conv_sweep._case), shaped from the SM count like the sweep's: 8x8 maps, N = 2T - 1
    images for T m-tiles with a 64-row M tail"""
    h = sm // 2
    t2, t3, t5 = sm + h, 2 * sm + h, 4 * sm + h
    own_ctas = sm // 2
    m_own = 4 * own_ctas + own_ctas // 2
    case = cs_sweep._case
    return {
        'dgrad_res_own_w128': case(2 * m_own - 1, 8, 8, 256, 64, ops='d', res_d=True),   # 64 -> 256 channels
        'dgrad_res_w128_odd': case(2 * t3 - 1, 8, 8, 128, 64, ops='d', res_d=True),
        'fprop_res_relu_w128': case(2 * t5 - 1, 8, 8, 64, 128, ops='f', res=True, act=1),
        'fprop_bias_relu6_w64_c32': case(2 * t2 - 1, 8, 8, 32, 64, ops='f', bias=True, act=2),
        'deep_k_one_buf_w64': case(2 * t3 - 1, 8, 8, 512, 64, ops='fd'),
    }


_NAMES = list(cases(132))


def _get(name):
    return cases(cs_sweep._sm_count())[name]


@pytest.mark.parametrize('name', _NAMES)
def test_tier1_exact(name):
    cs_sweep.check_exact(_get(name), 'epilogue_' + name)


@pytest.mark.parametrize('name', _NAMES)
def test_tier2_rounding(name):
    cs_sweep.check_rounding(_get(name), 'epilogue_' + name)


def test_schedule_coverage(monkeypatch, capfd):
    """every case takes the staging schedule it is meant to test (per-launch debug line field epi_bufs)"""
    cs_sweep.enable_debug_lines(monkeypatch)
    sm = cs_sweep._sm_count()
    run = dict(cases(sm))
    run['stats_own_w128'] = cs_sweep.sweep(sm)['stats_own_w128']   # checked exactly by the sweep itself
    recs = cs_sweep.coverage_records(run, capfd)
    two = lambda r: r['kind'] == 'igemm' and r['epi_bufs'] == 2 and r['tma_store'] == 1
    req = {
        'two staging tiles, >= 5 tiles per CTA': lambda r: two(r) and r['max_tiles'] >= 5,
        'two staging tiles, odd tile count per CTA': lambda r: two(r) and r['max_tiles'] >= 3 and r['max_tiles'] % 2,
        'two staging tiles, owned n-tile': lambda r: two(r) and r['own'] == 1,
        'two staging tiles, M tail in a warpgroup-1 tile': lambda r: two(r) and cs_sweep._tail_in_wg1(r),
        'two staging tiles, dgrad residual': lambda r: two(r) and r['op'] == 'dgrad' and r['res'],
        'two staging tiles, fprop residual + ReLU': lambda r: two(r) and r['op'] == 'fprop' and r['res'] and r['act'] == 1,
        'two staging tiles, bias + ReLU6': lambda r: two(r) and r['bias'] and r['act'] == 2,
        'two staging tiles, statistics': lambda r: two(r) and r['stats'],
        'one staging tile on the TMA-store path (deep K)':
            lambda r: r['kind'] == 'igemm' and r['epi_bufs'] == 1 and r['tma_store'] == 1,
    }
    missing = [label for label, pred in req.items() if not any(pred(r) for r in recs)]
    assert not missing, 'staging schedules no longer reached (SMs=%d): %s' % (sm, missing)
