"""CPU tier of the device JPEG decode on streams Pillow's encoder never writes (tests/jpeg_writer.py): other component
ids, table slots, markers and segment orders, 16-bit DQT, fill bytes, restart intervals that do not divide the image,
Huffman codes past the decoders' lookahead, and coefficient blocks far outside what quantising real pixels gives.
The numpy restatement of the kernels (tests/jpeg_oracle.py) must equal Pillow on all of them, and each file must be
classified to the side that decodes it.

The bitwise contract names libjpeg-turbo's x86-64 SIMD ISLOW IDCT (SSE2 and AVX2 agree): on out-of-range blocks it
differs from libjpeg-turbo's C jpeg_idct_islow, which the contract does not follow, nor other architectures' SIMD."""
import os
import platform
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import jpeg_oracle  # noqa: E402
import jpeg_writer as W  # noqa: E402
from test_jpeg_cpu import encode, picture, pil_rgb  # noqa: E402
from convnet.pytorch_b200.utils import jpeg  # noqa: E402

YCC = [(1, 1, 1, 0, 0, 0), (2, 1, 1, 1, 1, 1), (3, 1, 1, 1, 1, 1)]


def _q(base, scale):
    """A quantisation table (natural order) growing with frequency: base + scale * (u + v), clamped to [1, 255]."""
    u, v = np.mgrid[0:8, 0:8]
    return np.clip(base + scale * (u + v), 1, 255).reshape(64)


def _blocks(planes, comps, width, height, qt):
    """Quantised coefficients of smooth seeded sample planes for a frame (comps as jpeg_writer.encode takes them)."""
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    if len(comps) == 1:
        hmax = vmax = 1
    mx, my = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    out = []
    for p, c in zip(planes, comps):
        h, v = (c[1], c[2]) if len(comps) > 1 else (1, 1)
        cw, ch = -(-width * h // hmax), -(-height * v // vmax)
        plane = W.pad_plane(p[:ch, :cw], 8 * my * v, 8 * mx * h)
        out.append(W.fdct(plane, qt[c[3]]))
    return out


def _frame(h, w, comps, seed, qt=None, **kw):
    """A writer file of a seeded picture: comps (id, h, v, tq, td, ta); qt {slot: table} (defaults: slot 0 luma-like,
    the other slots chroma-like); the Huffman tables default to annex K (slots 0 / 1, else the full tables)."""
    a = picture(h, w, seed)
    planes = [a[:, :, 0]] if len(comps) == 1 else [a[:, :, i] for i in range(3)]
    qt = qt or {s: _q(3 + 2 * s, 1 + s) for s in sorted({c[3] for c in comps})}
    dc = kw.pop('dc', None) or {c[4]: (W.K_DC_LUMA, W.K_DC_CHROMA, W.FULL_DC, W.FULL_DC)[c[4]] for c in comps}
    ac = kw.pop('ac', None) or {c[5]: (W.K_AC_LUMA, W.K_AC_CHROMA, W.FULL_AC, W.FULL_AC)[c[5]] for c in comps}
    blocks = kw.pop('blocks', None) or _blocks(planes, comps, w, h, qt)
    return W.encode(comps, blocks, w, h, qt, dc, ac, **kw)


def _gray(blocks, q, wide=False, **kw):
    R, C = blocks.shape[:2]
    return W.encode([(1, 1, 1, 0, 0, 0)], [blocks], 8 * C, 8 * R, {0: q}, {0: W.FULL_DC}, {0: W.FULL_AC},
                    wide_q=(0,) if wide else (), **kw)


def header_corpus():
    """(name, bytes, classifier reason) of files with the header and coding choices of other encoders."""
    long_dc = W.spread(W.DC_SYMBOLS, long=range(0, 16, 2))
    long_ac = W.spread(W.AC_SYMBOLS, long=[s for s in W.AC_SYMBOLS if s % 3 == 0 or s == 0x00])
    rgb = [(82, 1, 1, 0, 0, 0), (71, 1, 1, 0, 0, 0), (66, 1, 1, 0, 0, 0)]
    out = [
        ('ids 0/1/2 no JFIF', _frame(37, 51, [(0, 2, 2, 0, 0, 0), (1, 1, 1, 1, 1, 1), (2, 1, 1, 1, 1, 1)], 1,
                                     markers=()), 'baseline'),
        ('3 components no JFIF', _frame(24, 40, YCC, 2, markers=()), 'baseline'),
        ('Adobe transform 1', _frame(30, 42, [(1, 2, 1, 0, 0, 0)] + YCC[1:], 3, markers=(W.adobe(1),)), 'baseline'),
        ('Adobe transform 1 with JFIF', _frame(30, 42, YCC, 3, markers=(W.jfif(), W.adobe(1))), 'baseline'),
        ('SOF1 slots 2/3', _frame(35, 29, [(1, 2, 2, 2, 2, 3), (2, 1, 1, 3, 3, 2), (3, 1, 1, 3, 3, 2)], 4,
                                  sof=0xC1), 'baseline'),
        ('separate Cb and Cr tables', _frame(33, 47, [(1, 2, 1, 0, 0, 0), (2, 1, 1, 1, 1, 1), (3, 1, 1, 2, 1, 1)], 5,
                                             qt={0: _q(2, 1), 1: _q(5, 3), 2: _q(9, 7)}), 'baseline'),
        ('16-bit DQT', _frame(26, 34, YCC, 6, wide_q=(0, 1)), 'baseline'),
        ('16-bit DQT above 255', _frame(26, 34, YCC, 7, qt={0: _q(2, 1) * 300, 1: _q(4, 2) * 41}, wide_q=(0, 1)),
         'baseline'),
        ('tables after SOF, redefined', _frame(40, 40, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 8, tables_after_sof=True,
                                               redefine=True), 'baseline'),
        ('COM and APPn between tables', _frame(21, 27, YCC, 9, extra=[(1, W.COM, b'a comment'),
                                                                     (2, 0xE5, b'APP5 \xff data'),
                                                                     (3, 0xE1, b'Exif\0\0')]), 'baseline'),
        ('fill before markers', _frame(23, 31, [(1, 2, 1, 0, 0, 0)] + YCC[1:], 10, fill=3), 'baseline'),
        ('fill before RSTn', _frame(41, 37, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 11, restart=2, rst_fill=2, fill=1),
         'baseline'),
        ('restart 5 of 12 MCUs', _frame(24, 64, YCC, 12, restart=5), 'baseline'),
        ('restart 7 gray', _frame(40, 56, YCC[:1], 13, restart=7), 'baseline'),
        ('restart beyond the MCUs', _frame(17, 21, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 14, restart=1000), 'baseline'),
        ('restart 1 4:2:2', _frame(19, 45, [(1, 2, 1, 0, 0, 0)] + YCC[1:], 15, restart=1), 'baseline'),
        ('gray SOF 2x2', _frame(29, 35, [(1, 2, 2, 0, 0, 0)], 16), 'baseline'),
        ('gray SOF 2x2 restart 3', _frame(29, 35, [(1, 2, 2, 0, 0, 0)], 17, restart=3), 'baseline'),
        ('long DC and AC codes', _frame(45, 53, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 18, dc={0: long_dc, 1: long_dc},
                                        ac={0: long_ac, 1: long_ac}), 'baseline'),
        ('long codes 4:4:4 gray-like q1', _frame(24, 24, YCC, 19, qt={0: np.ones(64, int), 1: np.ones(64, int)},
                                                 dc={0: long_dc, 1: W.FULL_DC}, ac={0: long_ac, 1: long_ac}),
         'baseline'),
        ('Adobe transform 0', _frame(16, 16, YCC, 20, markers=(W.adobe(0),)), 'Adobe transform 0'),
        ('RGB ids', _frame(16, 16, rgb, 21, markers=()), 'RGB component ids'),
        ('4:1:1', _frame(16, 32, [(1, 4, 1, 0, 0, 0)] + YCC[1:], 22), 'sampling 4x1,1x1,1x1'),
        ('4:4:0', _frame(32, 16, [(1, 1, 2, 0, 0, 0)] + YCC[1:], 23), 'sampling 1x2,1x1,1x1'),
        ('16-bit DQT above 32767', _frame(16, 16, YCC[:1], 24, qt={0: np.full(64, 40000)}, wide_q=(0,)),
         'quantisation entries above 32767'),
    ]
    return out


def extreme_corpus(seed=0):
    """(name, bytes, 'baseline') of files whose dequantised coefficients leave 16 bits, or whose IDCT leaves the
    sample range: random blocks at 8-bit q = 1 ... 255 and at 16-bit q, DC-only blocks with |dq * 4| > 32767, blocks
    whose only AC sits in a few rows or columns, an AC coefficient that dequantises to 0 mod 65536, and a DC predictor
    that drifts past int16."""
    rng = np.random.default_rng(seed)
    out = []

    def rand(R, C, amp, density):
        b = rng.integers(-amp, amp + 1, (R, C, 64)) * (rng.random((R, C, 64)) < density)
        b[..., 0] = rng.integers(-2047, 2048, (R, C))
        return b
    for qv in (1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 144, 233, 255):
        for amp, dens in ((2047, 0.3), (32767, 0.05), (300, 1.0)):
            out.append(('random q%d amp %d' % (qv, amp), _gray(rand(3, 5, amp, dens), np.full(64, qv))))
    for qv in (256, 1000, 4097, 32767):
        out.append(('random 16-bit q%d' % qv, _gray(rand(3, 5, 200, 0.2), np.full(64, qv), wide=True)))
    b = np.zeros((4, 8, 64), np.int64)
    b[..., 0] = rng.integers(-2047, 2048, (4, 8))
    b[0, :, 1] = rng.integers(-3, 4, 8)                 # AC in row 0 only: still pass 1's shortcut
    b[1, :, 8] = 1                                      # AC in row 1: the full pass
    for qv in (9, 17, 33, 255):
        out.append(('DC-only q%d' % qv, _gray(b, np.full(64, qv))))
    for (r0, r1), (c0, c1) in (((1, 4), (4, 8)), ((4, 8), (0, 4)), ((1, 2), (7, 8)), ((7, 8), (0, 1))):
        b = np.zeros((2, 8, 64), np.int64)
        b[..., 0] = rng.integers(1000, 2048, (2, 8)) * rng.choice([-1, 1], (2, 8))
        m = np.zeros((8, 8), bool)
        m[r0:r1, c0:c1] = True
        b[..., m.reshape(-1)] = rng.integers(-3, 4, (2, 8, int(m.sum())))
        out.append(('AC rows %d-%d columns %d-%d' % (r0, r1 - 1, c0, c1 - 1), _gray(b, np.full(64, 40))))
    b = np.zeros((1, 4, 64), np.int64)
    b[..., 0] = [100, 3000, -3000, 9000]
    b[..., 8] = 256
    out.append(('AC dequantised to 0 mod 65536', _gray(b, np.full(64, 256), wide=True)))
    b = np.zeros((2, 16, 64), np.int64)
    b[..., 0] = np.cumsum(np.r_[np.full(16, 20000), np.full(16, -30000)]).reshape(2, 16)
    for qv in (1, 3):
        out.append(('DC predictor drift q%d' % qv, _gray(b, np.full(64, qv))))
    # colour: extreme luma and chroma through upsampling and the colour conversion
    for qv, comps in ((7, [(1, 2, 2, 0, 0, 0)] + YCC[1:]), (60, [(1, 2, 1, 0, 0, 0)] + YCC[1:]), (255, YCC)):
        h, w = 24, 40
        hmax, vmax = comps[0][1], comps[0][2]
        mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
        blocks = [rand(my * c[2], mx * c[1], 2047, 0.2) for c in comps]
        out.append(('colour %dx%d q%d' % (hmax, vmax, qv),
                    W.encode(comps, blocks, w, h, {0: np.full(64, qv), 1: np.full(64, qv)},
                             {0: W.FULL_DC, 1: W.FULL_DC}, {0: W.FULL_AC, 1: W.FULL_AC})))
    return [(n, d, 'baseline') for n, d in out]


def _patch_dqt(data, v):
    """Pillow's file with every 8-bit DQT entry set to v: the entropy data stay valid, the dequantised values grow."""
    b, pos = bytearray(data), 2
    while b[pos + 1] != 0xDA:
        length = (b[pos + 2] << 8) | b[pos + 3]
        if b[pos + 1] == 0xDB:
            i = pos + 4
            while i < pos + 2 + length:
                assert b[i] >> 4 == 0
                b[i + 1:i + 65] = bytes([v]) * 64
                i += 65
        pos += 2 + length
    return bytes(b)


def patched_dqt_corpus():
    out = []
    for q in (100, 95, 90, 75):
        for ss in (0, 1, 2):
            f = encode(picture(48, 64, q, noise=q == 100), quality=q, subsampling=ss)
            out += [('q%d ss%d DQT=%d' % (q, ss, v), _patch_dqt(f, v), 'baseline') for v in (1, 8, 32, 255)]
    return out


def stream_corpus():
    return header_corpus() + extreme_corpus() + patched_dqt_corpus()


def test_annex_k_tables_are_pillows_default_tables():
    info = jpeg.parse(encode(picture(16, 16, 0), quality=75))
    for got, want in ((info.dc[0], W.K_DC_LUMA), (info.dc[1], W.K_DC_CHROMA), (info.ac[0], W.K_AC_LUMA),
                      (info.ac[1], W.K_AC_CHROMA)):
        assert got.bits[1:] == want.bits and list(got.huffval[:len(want.vals)]) == want.vals


def test_writer_tables_reach_past_the_lookahead():
    """The 'long' tables give 10- to 16-bit codes to DC and AC symbols the corpus uses, and leave code space unused."""
    long_dc = W.spread(W.DC_SYMBOLS, long=range(0, 16, 2))
    long_ac = W.spread(W.AC_SYMBOLS, long=[s for s in W.AC_SYMBOLS if s % 3 == 0 or s == 0x00])
    for t in (long_dc, long_ac):
        lengths = {l for _, l in t.codes.values()}
        assert set(range(10, 17)) <= lengths and t.spare > 0
    assert long_ac.codes[0x00][1] > jpeg.LOOKAHEAD                   # EOB: in nearly every block


@pytest.mark.parametrize('part', ['header', 'extreme', 'patched-dqt'])
def test_classifier_sends_each_stream_to_its_side(part):
    corpus = {'header': header_corpus, 'extreme': extreme_corpus, 'patched-dqt': patched_dqt_corpus}[part]()
    for name, data, reason in corpus:
        info = jpeg.parse(data)
        assert info.reason == reason, (name, info.reason)
        assert info.device == (reason == 'baseline'), name
        if info.device:
            assert (info.height, info.width) == pil_rgb(data).shape[:2], name


@pytest.mark.parametrize('part', ['header', 'extreme', 'patched-dqt'])
def test_oracle_equals_pillow_on_streams_pillow_never_writes(part):
    corpus = {'header': header_corpus, 'extreme': extreme_corpus, 'patched-dqt': patched_dqt_corpus}[part]()
    bad = []
    for name, data, reason in corpus:
        if reason == 'baseline' and not np.array_equal(jpeg_oracle.decode(data), pil_rgb(data)):
            bad.append(name)
    assert not bad, bad


def test_idct_saturates_where_the_c_idct_wraps():
    """One block, by hand: DC 2047 at q 255 dequantises to s16(521985) = -2559; pass 1's shortcut wraps
    s16(-2559 * 4) = -10236, and the saturating store gives 0 where the C IDCT's range-limit table wraps."""
    b = np.zeros(64, np.int64)
    b[0] = 2047
    out = jpeg_oracle.idct(b[None], np.full(64, 255))
    assert (out == 0).all()
    b[8] = 1                                                     # no shortcut: -2559 << 2 saturates alike in pass 1
    assert (jpeg_oracle.idct(b[None], np.full(64, 255)) == 0).all()
    b = np.zeros(64, np.int64)
    b[0] = 1000                                                  # dq0 = 9000: << 2 wraps to -29536 in the shortcut
    assert (jpeg_oracle.idct(b[None], np.full(64, 9)) == 0).all()
    assert (pil_rgb(_gray(b.reshape(1, 1, 64), np.full(64, 9)))[..., 0] == 0).all()


_DECODE = """import hashlib, sys
from PIL import Image
h = hashlib.sha256()
for p in sys.argv[1:]:
    h.update(Image.open(p).convert('RGB').tobytes())
print(h.hexdigest())
"""


def test_the_contract_names_libjpeg_turbos_x86_simd_idct(tmp_path):
    """Pillow's SSE2 and AVX2 ISLOW paths decode the extreme corpus to the same bytes, which are the oracle's; the C
    path (JSIMD_FORCENONE) decodes them differently."""
    from PIL import features
    if not features.check_feature('libjpeg_turbo'):
        pytest.skip('Pillow does not report libjpeg_turbo: its IDCT is not the one the decode contract names')
    if platform.machine().lower() not in ('x86_64', 'amd64'):
        pytest.skip('the contract names libjpeg-turbo\'s x86-64 SIMD; this is %s' % platform.machine())
    paths = []
    for i, (_, data, _) in enumerate(extreme_corpus()):
        p = tmp_path / ('%03d.jpg' % i)
        p.write_bytes(data)
        paths.append(str(p))
    digests = {}
    for force in ('JSIMD_FORCESSE2', 'JSIMD_FORCEAVX2', 'JSIMD_FORCENONE'):
        env = {k: v for k, v in os.environ.items() if not k.startswith('JSIMD_')}
        env[force] = '1'
        r = subprocess.run([sys.executable, '-c', _DECODE] + paths, env=env, capture_output=True, text=True,
                           check=True)
        digests[force] = r.stdout.strip()
    import hashlib
    h = hashlib.sha256()
    for p in paths:
        h.update(jpeg_oracle.decode(open(p, 'rb').read()).tobytes())
    assert digests['JSIMD_FORCESSE2'] == digests['JSIMD_FORCEAVX2'] == h.hexdigest()
    assert digests['JSIMD_FORCENONE'] != digests['JSIMD_FORCESSE2']


def test_fill_bytes_before_markers_stay_inside_the_segment():
    data = _frame(41, 37, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 11, restart=2, rst_fill=2, fill=1)
    info = jpeg.parse(data)
    assert info.device and data[info.ecs[1]:info.ecs[1] + 2] == b'\xff\xd9'
    mx, my = info.mcus
    assert len(info.rst) == -(-mx * my // 2) - 1
    assert all(data[p - 2] == 0xFF and data[p - 1] == 0xD0 + (k & 7) for k, p in enumerate(info.rst))


def damaged(kind, mcu_row, h=128, w=80, seed=30):
    """A 4:2:0 file (MCU rows of 16 pixels) damaged in MCU 1 of its MCU row ``mcu_row`` (jpeg_writer.encode
    ``damage``); with one restart interval per MCU row for the 'restart' damage."""
    mx = -(-w // 16)
    return _frame(h, w, [(1, 2, 2, 0, 0, 0)] + YCC[1:], seed, restart=mx if kind == 'restart' else 0,
                  damage=(kind, mcu_row * mx + 1))


@pytest.mark.parametrize('kind', ['code', 'run', 'restart', 'short'])
def test_damaged_streams_keep_their_headers(kind):
    """The writer's damaged entropy data leave the headers intact, so the device takes the file and must report the
    damage (tests/test_gpu_jpeg_streams.py); the damage is where it was asked for."""
    data = damaged(kind, 3)
    info = jpeg.parse(data)
    assert info.device, info.reason
    nums = [data[p - 1] - 0xD0 for p in info.rst]
    if kind == 'code':
        with pytest.raises(ValueError, match='bad Huffman code'):
            jpeg_oracle.entropy_decode(data, info)
    elif kind == 'run':
        with pytest.raises(ValueError, match='past 63'):
            jpeg_oracle.entropy_decode(data, info)
    elif kind == 'restart':
        assert nums == [0, 1, 2, 4, 4, 5, 6]                        # the marker ending MCU row 3 is RST4
    else:
        whole = _frame(128, 80, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 30)
        assert data[info.ecs[1]:] == b'\xff\xd9' and len(data) < len(whole) * 3 // 4   # ends inside MCU row 3
