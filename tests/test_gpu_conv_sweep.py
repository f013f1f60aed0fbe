"""Generated sweep of the convolution kernels (implicit-GEMM fprop/dgrad, split-K wgrad, halo shift-GEMM fprop/dgrad
and wgrad) against fp64 torch, element by element.

The shapes are generated from the device's SM count, so that each intended schedule (one tile per CTA, warpgroup 1
computing tiles, five or more tiles per CTA, the M tail in a warpgroup-1 tile, owned-n-tile walks, ...) holds on any
H100 variant.  Every case runs in two tiers:

* tier 1 -- exact arithmetic: sparse integer operands in [-2, 2] (integer bias, residual and initial dw), so every
  product and partial sum is an integer far below 2^13 and representable in fp32, and |y| <= 256 is exact in bf16.  The
  kernel must equal the fp64 reference rounded once, bit for bit, and so must the fused BN statistics.
* tier 2 -- rounding-realistic: normal bf16 operands; every element must satisfy
  |y - ref| <= rt * |ref| + c * absref, where absref is the same convolution of |x| and |w| (plus |bias| and
  |residual|), rt = 2^-8 (one bf16 output rounding) for bf16 outputs and 0 for fp32 outputs.  The relative-L2 limits
  of test_gpu_ops.py are checked as well.

In both tiers outputs are written through out= into a NaN-filled view of a larger buffer whose guard regions must stay
intact, and each call is repeated on the same inputs and must give bitwise-identical results.  test_sweep_coverage
runs the sweep with the host's per-launch debug lines enabled and fails, naming the entry, when a configuration the
sweep is meant to reach is no longer reached.
"""
import math
import re
import zlib

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# tier-2 accumulation-error coefficients (|y - ref| beyond the output rounding, in units of absref).  Calibrated on an
# NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit): the worst ratios over the sweep were 8.5e-8 for bf16 outputs
# (halo dgrad, K = 256) and 1.4e-7 for fp32 outputs (fprop of a 64 -> 1000 fully connected layer), 5.6x and 6.9x
# below these bounds; test_tier2_calibration_report prints them again.
C_BF16 = 2.0 ** -21
C_FP32 = 2.0 ** -20
GUARD = 256               # elements before and after every output view (keeps TMA's 16-byte alignment)
SENTINEL = -1536.0        # exact in bf16 and fp32


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ the sweep
def _case(N, H, W, C, K, R=1, S=1, stride=1, pad=(0, 0), ops='fdw', bias=False, res=False, act=0, fp32=False,
          stats=False):
    pad = (pad, pad) if isinstance(pad, int) else tuple(pad)
    return dict(N=N, H=H, W=W, C=C, K=K, R=R, S=S, stride=stride, pad=pad, ops=ops, bias=bias, res=res, act=act,
                fp32=fp32, stats=stats)


def sweep(sm):
    """name -> case.  Most implicit-GEMM cases use 8x8 output maps (64 pixels per image), so N = 2T - 1 images give T
    m-tiles with a 64-row M tail.  T = S + S/2 gives two tiles to the busiest CTA with the tail in warpgroup 1's tile,
    2S + S/2 three tiles, 4S + S/2 five."""
    h = sm // 2
    t2, t3, t5 = sm + h, 2 * sm + h, 4 * sm + h
    n_rr = next(n for n in (5, 7, 9, 11, 3) if (2 * sm) % n)   # n-tiles that do not divide twice the grid
    m_rr = -(-t3 // n_rr)
    own_ctas = sm // 2
    m_own = 4 * own_ctas + own_ctas // 2
    return {
        # igemm widths 16..128 with warpgroup 1 computing tiles; A-side ck 16 / 32 / 64; schedules
        'w16_c8_deep': _case(2 * t5 - 1, 8, 8, 8, 16),                                  # >= 5 tiles per CTA
        'w32_c24_3x3s2': _case(2 * t3 - 1, 16, 16, 24, 32, 3, 3, 2, 1),                 # 3 per CTA, 9 k-iters
        'w48_c64_tail_wg1': _case(2 * t2 - 1, 8, 8, 64, 48),
        'w80_c16_3x3': _case(2 * t2, 8, 8, 16, 80, 3, 3, 1, 1),
        'w96_c32_1x3': _case(2 * t2 - 1, 8, 8, 32, 96, 1, 3, 1, (0, 1)),
        'w112_c16_1x7': _case(2 * t2 - 1, 8, 8, 16, 112, 1, 7, 1, (0, 3)),
        'bias_relu6_w128': _case(2 * t2 - 1, 8, 8, 64, 128, bias=True, act=2),         # bias on the TMA-store path
        'res_relu_w64_3x3s2': _case(2 * t3 - 1, 16, 16, 64, 64, 3, 3, 2, 1, res=True, act=1),
        'fc_fp32_bias_1000': _case(-(-t3 // 8) * 128 - 37, 1, 1, 64, 1000, bias=True, fp32=True),
        'fc_64_16': _case(64, 1, 1, 64, 16, bias=True, fp32=True),                      # one tile; unsplit wgrad
        # fused BN statistics: round-robin walks whose warpgroups change n-tile between tiles, and an owned-n-tile walk
        'stats_w64_rr': _case(2 * m_rr - 1, 8, 8, 64, 64 * n_rr, stats=True),
        'stats_w128_rr': _case(2 * m_rr - 1, 8, 8, 64, 128 * n_rr, stats=True),
        'stats_own_w128': _case(2 * m_own - 1, 8, 8, 64, 256, stats=True),
        # dgrad with empty residue classes; orphaned diagnostic shapes with 16 channels on the dy side
        'p1s2_64_128': _case(8, 16, 16, 64, 128, 1, 1, 2, 0),
        'c3_16_16': _case(4, 32, 32, 16, 16, 3, 3, 1, 1),
        'c3s2_16_32': _case(4, 32, 32, 16, 32, 3, 3, 2, 1),
        'p1s2_16_32': _case(4, 32, 32, 16, 32, 1, 1, 2, 0),
        # weight-gradient tile widths (NC = boxes per CTA x channels per box) with ragged K
        'nc32_p1': _case(4, 8, 8, 32, 32),
        'nc48_k24_1x3': _case(4, 8, 8, 16, 24, 1, 3, 1, (0, 1)),
        'nc80_k40_1x5': _case(4, 8, 8, 16, 40, 1, 5, 1, (0, 2)),
        'nc160_1x5': _case(8, 8, 8, 32, 64, 1, 5, 1, (0, 2)),
        'nc192_p1': _case(8, 8, 8, 192, 64),
        'nc224_k48_1x7': _case(4, 8, 8, 32, 48, 1, 7, 1, (0, 3)),
        # halo shift-GEMM kernels
        'halo3_w64_stats': _case(8, 28, 28, 64, 64, 3, 3, 1, 1, stats=True),
        'halo3_w128_res': _case(4, 28, 28, 64, 128, 3, 3, 1, 1, res=True, act=1),
        'halo3_w256_bias': _case(8, 14, 14, 64, 256, 3, 3, 1, 1, bias=True),
        'halo3_one_split': _case(1, 10, 10, 64, 64, 3, 3, 1, 1),
        'halo4_w64': _case(4, 32, 32, 16, 64, 4, 4, 1, 0, ops='fw'),
        'halo4_w128_stats': _case(3, 32, 32, 16, 128, 4, 4, 1, 0, ops='fw', stats=True),
    }


_NAMES = list(sweep(132))


def _get(name):
    return sweep(_sm_count())[name]


def _desc(cs):
    return _ops().make_desc(cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'], cs['S'], cs['stride'], cs['pad'])


def _gen(name, tier):
    return torch.Generator().manual_seed(zlib.crc32(('%s/%d' % (name, tier)).encode()))


# ------------------------------------------------------------------------------------------------ fp64 references
def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _w_kcrs(w, cs):
    return w.double().view(cs['K'], cs['R'], cs['S'], cs['C']).permute(0, 3, 1, 2)


def ref_fprop(x, w, cs):
    return _nhwc(F.conv2d(_nchw(x), _w_kcrs(w, cs), stride=cs['stride'], padding=cs['pad']))


def ref_dgrad(dy, w, cs):
    size = (cs['N'], cs['C'], cs['H'], cs['W'])
    return _nhwc(conv2d_input(size, _w_kcrs(w, cs), _nchw(dy), stride=cs['stride'], padding=cs['pad']))


def ref_wgrad(x, dy, cs):
    g = conv2d_weight(_nchw(x), (cs['K'], cs['C'], cs['R'], cs['S']), _nchw(dy), stride=cs['stride'],
                      padding=cs['pad'])
    return g.permute(0, 2, 3, 1).reshape(cs['K'], cs['R'] * cs['S'], cs['C'])


def _act(v, act):
    return v.relu() if act == 1 else (v.clamp(0, 6) if act == 2 else v)


# ------------------------------------------------------------------------------------------------ kernel calls
def _guarded(shape, dtype, fill):
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=dtype, device='cuda')
    view = buf[GUARD:GUARD + n].view(shape)
    view.fill_(fill)
    return buf, view


def _check_written(buf, view, what):
    n = view.numel()
    assert bool((buf[:GUARD] == SENTINEL).all()), '%s: wrote before its output' % what
    assert bool((buf[GUARD + n:] == SENTINEL).all()), '%s: wrote past its output' % what
    assert not bool(view.isnan().any()), '%s: %d output elements never written' % (what, int(view.isnan().sum()))


def _outshape(cs):
    d = _desc(cs)
    return d.P, d.Q


def call_fprop(cs, x, w, bias, res):
    """-> (y, per-channel [sum, sum of squares] from the fused statistics or None)"""
    ops = _ops()
    P, Q = _outshape(cs)
    buf, y = _guarded((cs['N'], P, Q, cs['K']), torch.float32 if cs['fp32'] else bf16, float('nan'))
    ws = torch.zeros(ops.bn_workspace_floats(cs['K']), device='cuda') if cs['stats'] else None
    ops.conv_fprop(x, w, _desc(cs), out=y, bias=bias, residual=res, act=cs['act'], out_fp32=cs['fp32'],
                   bn_stats_ws=ws)
    torch.cuda.synchronize()
    _check_written(buf, y, 'fprop')
    sums = None
    if ws is not None:
        K = cs['K']
        sums = ws[:16 * 2 * K * 2].view(torch.float64).view(16, 2, K).sum(0)   # kStatReplicas x {sum, sum^2} x K
    return y, sums


def call_dgrad(cs, dy, w, res):
    ops = _ops()
    wt = ops.weight_transpose(w)
    buf, dx = _guarded((cs['N'], cs['H'], cs['W'], cs['C']), bf16, float('nan'))
    ops.conv_dgrad(dy, wt, _desc(cs), out=dx, residual=res)
    torch.cuda.synchronize()
    _check_written(buf, dx, 'dgrad')
    return dx


def call_wgrad(cs, x, dy, dw0):
    buf, dw = _guarded(tuple(dw0.shape), torch.float32, 0.0)
    dw.copy_(dw0)
    _ops().conv_wgrad(x, dy, _desc(cs), dw)
    torch.cuda.synchronize()
    _check_written(buf, dw, 'wgrad')
    return dw


def _res_fprop(cs):
    return cs['res']


def _res_dgrad(cs):
    # the residual epilogue of dgrad is exercised where the stride-2 residue classes are all non-empty
    return cs['res'] and cs['R'] == 3


# ------------------------------------------------------------------------------------------------ tier 1
def _ints(shape, density, g, lo=-2, hi=2):
    v = torch.randint(lo, hi, shape, generator=g).float()
    v = torch.where(v >= 0, v + 1, v)                       # {lo..hi} without 0
    return torch.where(torch.rand(shape, generator=g) < density, v, torch.zeros(()))


def _density(n, target):
    """density of two sparse operands whose n-term products have a mean absolute sum near target"""
    return min(1.0, math.sqrt(target / (2.25 * n)))


def _exact_preconditions(absref, what, bf16_out):
    amax = float(absref.max())
    assert amax <= 2 ** 11, '%s: partial sums up to %g are not far below 2^13' % (what, amax)
    if bf16_out:
        assert amax <= 256, '%s: |y| up to %g is not exact in bf16' % (what, amax)


@pytest.mark.parametrize('name', _NAMES)
def test_tier1_exact(name):
    cs = _get(name)
    g = _gen(name, 1)
    N, H, W, C, K, RS = cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'] * cs['S']
    P, Q = _outshape(cs)
    dev = 'cuda'
    if 'f' in cs['ops']:
        d = _density(C * RS, 8 if cs['stats'] else 16)
        x, w = _ints((N, H, W, C), d, g), _ints((K, RS, C), d, g)
        bias = torch.randint(-4, 5, (K,), generator=g).float().to(dev) if cs['bias'] else None
        res = _ints((N, P, Q, K), 0.5, g).to(dev).to(bf16) if _res_fprop(cs) else None
        x, w = x.to(dev).to(bf16), w.to(dev).to(bf16)
        pre = ref_fprop(x, w, cs)
        absref = ref_fprop(x.abs(), w.abs(), cs)
        if bias is not None:
            pre, absref = pre + bias.double(), absref + bias.double().abs()
        if res is not None:
            pre, absref = pre + res.double(), absref + res.double().abs()
        _exact_preconditions(absref, 'fprop', not cs['fp32'])
        ref = _act(pre, cs['act'])
        y, sums = call_fprop(cs, x, w, bias, res)
        y2, sums2 = call_fprop(cs, x, w, bias, res)
        assert torch.equal(y, y2), 'fprop is not deterministic'
        want = ref.to(y.dtype)
        bad = (y != want)
        assert not bool(bad.any()), 'fprop: %d of %d elements differ, first at %s' % (
            int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
        if sums is not None:
            flat = ref.reshape(-1, K)
            assert float((flat * flat).sum(0).max()) < 2 ** 24, 'statistics partials would not be exact in fp32'
            assert torch.equal(sums, sums2), 'fused statistics are not deterministic'
            assert torch.equal(sums[0], flat.sum(0)), 'fused statistics: per-channel sum differs'
            assert torch.equal(sums[1], (flat * flat).sum(0)), 'fused statistics: per-channel sum of squares differs'
    if 'd' in cs['ops']:
        d = _density(K * RS, 16)
        dy, w = _ints((N, P, Q, K), d, g).to(dev).to(bf16), _ints((K, RS, C), d, g).to(dev).to(bf16)
        res = _ints((N, H, W, C), 0.5, g).to(dev).to(bf16) if _res_dgrad(cs) else None
        ref = ref_dgrad(dy, w, cs)
        absref = ref_dgrad(dy.abs(), w.abs(), cs)
        if res is not None:
            ref, absref = ref + res.double(), absref + res.double().abs()
        _exact_preconditions(absref, 'dgrad', True)
        dx = call_dgrad(cs, dy, w, res)
        assert torch.equal(dx, call_dgrad(cs, dy, w, res)), 'dgrad is not deterministic'
        bad = dx != ref.to(bf16)
        assert not bool(bad.any()), 'dgrad: %d of %d elements differ, first at %s' % (
            int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
    if 'w' in cs['ops']:
        d = _density(N * P * Q, 256)
        x, dy = _ints((N, H, W, C), d, g).to(dev).to(bf16), _ints((N, P, Q, K), d, g).to(dev).to(bf16)
        dw0 = torch.randint(-8, 9, (K, RS, C), generator=g).float().to(dev)
        ref = ref_wgrad(x, dy, cs)
        _exact_preconditions(ref_wgrad(x.abs(), dy.abs(), cs) + 8, 'wgrad', False)
        zero = torch.zeros_like(dw0)
        assert torch.equal(call_wgrad(cs, x, dy, zero), call_wgrad(cs, x, dy, zero)), 'wgrad is not deterministic'
        dw = call_wgrad(cs, x, dy, dw0)
        bad = dw.double() != ref + dw0.double()
        assert not bool(bad.any()), 'wgrad (dw += ...): %d of %d elements differ, first at %s' % (
            int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))


# ------------------------------------------------------------------------------------------------ tier 2
WORST = {}   # output type -> (worst (|y - ref| - rt |ref|) / absref, where)


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _check_bound(y, ref, absref, what):
    is_bf16 = y.dtype == bf16
    rt, c = (2.0 ** -8, C_BF16) if is_bf16 else (0.0, C_FP32)
    err = (y.double() - ref).abs()
    excess = err - rt * ref.abs()
    ratio = float((excess / absref.clamp_min(1e-300)).max())
    key = 'bf16' if is_bf16 else 'fp32'
    if ratio > WORST.get(key, (-math.inf, ''))[0]:
        WORST[key] = (ratio, what)
    bad = excess > c * absref
    assert not bool(bad.any()), '%s: %d elements outside |y-ref| <= %g |ref| + %g absref (worst ratio %.3g)' % (
        what, int(bad.sum()), rt, c, ratio)
    assert _rel_l2(y, ref) < (4e-3 if is_bf16 else 2e-5), what


@pytest.mark.parametrize('name', _NAMES)
def test_tier2_rounding(name):
    cs = _get(name)
    g = _gen(name, 2)
    N, H, W, C, K, RS = cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'] * cs['S']
    P, Q = _outshape(cs)
    dev = 'cuda'
    x = torch.randn(N, H, W, C, generator=g).to(dev).to(bf16)
    w = (torch.randn(K, RS, C, generator=g) / math.sqrt(RS * C)).to(dev).to(bf16)
    dy = torch.randn(N, P, Q, K, generator=g).to(dev).to(bf16)
    if 'f' in cs['ops']:
        bias = torch.randn(K, generator=g).to(dev) if cs['bias'] else None
        res = torch.randn(N, P, Q, K, generator=g).to(dev).to(bf16) if _res_fprop(cs) else None
        pre, absref = ref_fprop(x, w, cs), ref_fprop(x.abs(), w.abs(), cs)
        if bias is not None:
            pre, absref = pre + bias.double(), absref + bias.double().abs()
        if res is not None:
            pre, absref = pre + res.double(), absref + res.double().abs()
        y, _ = call_fprop(cs, x, w, bias, res)
        assert torch.equal(y, call_fprop(cs, x, w, bias, res)[0]), 'fprop is not deterministic'
        _check_bound(y, _act(pre, cs['act']), absref, '%s fprop' % name)
    if 'd' in cs['ops']:
        res = torch.randn(N, H, W, C, generator=g).to(dev).to(bf16) if _res_dgrad(cs) else None
        ref, absref = ref_dgrad(dy, w, cs), ref_dgrad(dy.abs(), w.abs(), cs)
        if res is not None:
            ref, absref = ref + res.double(), absref + res.double().abs()
        dx = call_dgrad(cs, dy, w, res)
        assert torch.equal(dx, call_dgrad(cs, dy, w, res)), 'dgrad is not deterministic'
        _check_bound(dx, ref, absref, '%s dgrad' % name)
    if 'w' in cs['ops']:
        zero = torch.zeros(K, RS, C, device=dev)
        dw = call_wgrad(cs, x, dy, zero)
        assert torch.equal(dw, call_wgrad(cs, x, dy, zero)), 'wgrad is not deterministic'
        _check_bound(dw, ref_wgrad(x, dy, cs), ref_wgrad(x.abs(), dy.abs(), cs), '%s wgrad' % name)


def test_tier2_calibration_report():
    """Prints the worst observed excess ratio next to each tier-2 coefficient (run after the tier-2 cases, e.g. with
    -s); the coefficients should stay within 8x of what the H100 shows."""
    if not WORST:
        pytest.skip('no tier-2 case ran in this session')
    for key, c in (('bf16', C_BF16), ('fp32', C_FP32)):
        if key in WORST:
            ratio, where = WORST[key]
            print('tier-2 %s outputs: worst (|y-ref| - rt|ref|)/absref = %.3e (%s), bound c = %.3e (%.1fx)' % (
                key, ratio, where, c, c / ratio if ratio > 0 else math.inf))


# ------------------------------------------------------------------------------------------------ coverage
_LINE = re.compile(r'^\[(igemm|wgrad|halo|halo_wgrad)\] (.*)$')


def _parse(text, case, op, cs):
    recs = []
    for line in text.splitlines():
        m = _LINE.match(line.strip())
        if m:
            r = {k: int(v) for k, v in (kv.split('=') for kv in m.group(2).split())}
            r.update(kind=m.group(1), case=case, op=op, filt=(cs['R'], cs['S']))
            recs.append(r)
    return recs


def _tail_in_wg1(r):
    """an igemm launch whose last (partial) m-tile is computed by warpgroup 1 of its CTA"""
    if r['M'] % 128 == 0:
        return False
    last = r['m_tiles'] - 1
    if r['own']:
        return (last // (r['grid'] // r['n_tiles'])) & 1 == 1
    return any(((last * r['n_tiles'] + n) // r['grid']) & 1 for n in range(r['n_tiles']))


def _requirements():
    ig = lambda r: r['kind'] == 'igemm'
    igf = lambda r: ig(r) and r['op'] == 'fprop'
    igd = lambda r: ig(r) and r['op'] == 'dgrad'
    wg = lambda r: r['kind'] == 'wgrad'
    ha = lambda r: r['kind'] == 'halo'
    hw = lambda r: r['kind'] == 'halo_wgrad'
    req = {}
    for bn in range(16, 129, 16):
        req['igemm fprop width %d, warpgroup 1 computing' % bn] = \
            lambda r, bn=bn: igf(r) and r['block_n'] == bn and r['max_tiles'] >= 2
    req.update({
        'igemm 1 tile per CTA': lambda r: ig(r) and r['max_tiles'] == 1,
        'igemm odd tile count per CTA': lambda r: ig(r) and r['max_tiles'] >= 3 and r['max_tiles'] % 2 == 1,
        'igemm >= 5 tiles per CTA': lambda r: ig(r) and r['max_tiles'] >= 5,
        'igemm ring wraps mid-tile': lambda r: ig(r) and r['max_tiles'] >= 2 and r['k_iters'] % r['stages'] != 0,
        'igemm M tail in a warpgroup-1 tile': lambda r: ig(r) and _tail_in_wg1(r),
        'igemm tma_store on': lambda r: ig(r) and r['tma_store'] == 1,
        'igemm tma_store off': lambda r: ig(r) and r['tma_store'] == 0,
        'igemm plain_a on': lambda r: ig(r) and r['plain_a'] == 1,
        'igemm plain_a off': lambda r: ig(r) and r['plain_a'] == 0,
        'igemm b_stationary': lambda r: ig(r) and r['bstat'] == 1,
        'igemm own_ntile': lambda r: ig(r) and r['own'] == 1,
        'igemm fprop ck 16 (C = 8)': lambda r: igf(r) and r['ck'] == 16 and r['C'] == 8,
        'igemm fprop ck 32 (C = 24)': lambda r: igf(r) and r['ck'] == 32 and r['C'] == 24,
        'igemm fprop ck 64': lambda r: igf(r) and r['ck'] == 64,
        'igemm bias, bf16 TMA-store output': lambda r: igf(r) and r['bias'] and r['tma_store'] and not r['out_fp32'],
        'igemm bias, fp32 output': lambda r: igf(r) and r['bias'] and r['out_fp32'],
        'igemm fprop residual': lambda r: igf(r) and r['res'],
        'igemm act 1': lambda r: igf(r) and r['act'] == 1,
        'igemm act 2': lambda r: igf(r) and r['act'] == 2,
        'igemm statistics, width 64': lambda r: ig(r) and r['stats'] and r['block_n'] == 64,
        'igemm statistics, width 128': lambda r: ig(r) and r['stats'] and r['block_n'] == 128,
        'igemm statistics, warpgroup changes n-tile, M tail':
            lambda r: ig(r) and r['stats'] and not r['own'] and (2 * r['grid']) % r['n_tiles'] != 0
            and r['max_tiles'] >= 3 and r['M'] % 128 != 0,
        'dgrad stride 1': lambda r: igd(r) and r['os'] == 1,
        'dgrad stride 2': lambda r: igd(r) and r['os'] == 2,
        'dgrad 1x1 stride 2 (empty residue classes)': lambda r: igd(r) and r['os'] == 2 and r['filt'] == (1, 1),
        'dgrad 3x3 stride 2': lambda r: igd(r) and r['os'] == 2 and r['filt'] == (3, 3),
        'dgrad residual': lambda r: igd(r) and r['res'],
        'dgrad dy-side ck 16': lambda r: igd(r) and r['ck'] == 16,
        'dgrad dy-side ck 32': lambda r: igd(r) and r['ck'] == 32,
        'dgrad dy-side ck 64': lambda r: igd(r) and r['ck'] == 64,
    })
    for nc in (16, 32, 48, 64, 80, 96, 112, 128, 160, 192, 224, 256):
        req['wgrad NC %d' % nc] = lambda r, nc=nc: wg(r) and r['nc'] == nc
    req.update({
        'wgrad split (partial tiles + reduce)': lambda r: wg(r) and r['partial'] == 1,
        'wgrad unsplit (direct red.add)': lambda r: wg(r) and r['partial'] == 0,
        'wgrad partial last column group': lambda r: wg(r) and r['nboxes_last'] < r['bpc'],
        'wgrad K % 128 <= 64': lambda r: wg(r) and r['K'] % 128 <= 64,
        'wgrad K % 128 > 64': lambda r: wg(r) and r['K'] % 128 > 64,
        'wgrad ckA 16': lambda r: wg(r) and r['ckA'] == 16,
        'wgrad ckA 32': lambda r: wg(r) and r['ckA'] == 32,
        'wgrad plain_x on': lambda r: wg(r) and r['plain_x'] == 1,
        'wgrad plain_x off': lambda r: wg(r) and r['plain_x'] == 0,
        'wgrad stride 2': lambda r: wg(r) and r['stride'] == 2,
    })
    for bn in (64, 128, 256):
        req['halo 3x3 block_n %d' % bn] = lambda r, bn=bn: ha(r) and r['taps'] == 9 and r['block_n'] == bn
    for bn in (64, 128):
        req['halo 4x4 stem block_n %d' % bn] = lambda r, bn=bn: ha(r) and r['taps'] == 16 and r['block_n'] == bn
    req.update({
        'halo 3x3 stationary weights': lambda r: ha(r) and r['taps'] == 9 and r['bstat'] == 1,
        'halo 3x3 streamed weights': lambda r: ha(r) and r['taps'] == 9 and r['bstat'] == 0,
        'halo dgrad': lambda r: ha(r) and r['dir'] == 1,
        'halo residual + ReLU': lambda r: ha(r) and r['res'] and r['act'] == 1,
        'halo bias': lambda r: ha(r) and r['bias'],
        'halo fused statistics': lambda r: ha(r) and r['stats'],
        'halo wgrad 3x3': lambda r: hw(r) and r['taps'] == 9,
        'halo wgrad 4x4': lambda r: hw(r) and r['taps'] == 16,
        'halo wgrad K % 128 == 64': lambda r: hw(r) and r['K'] % 128 == 64,
        'halo wgrad one split': lambda r: hw(r) and r['splits'] == 1,
        'halo wgrad many splits': lambda r: hw(r) and r['splits'] > 1,
    })
    return req


def test_sweep_coverage(monkeypatch, capfd):
    """Every configuration of the table in _requirements() is reached by some launch of the sweep."""
    for var in ('B200_IGEMM_DEBUG', 'B200_WGRAD_DEBUG', 'B200_HALO_DEBUG'):
        monkeypatch.setenv(var, '1')
    ops = _ops()
    recs = []
    capfd.readouterr()
    for name, cs in sweep(_sm_count()).items():
        N, H, W, C, K, RS = cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'] * cs['S']
        P, Q = _outshape(cs)
        x = torch.zeros(N, H, W, C, device='cuda', dtype=bf16)
        w = torch.zeros(K, RS, C, device='cuda', dtype=bf16)
        dy = torch.zeros(N, P, Q, K, device='cuda', dtype=bf16)
        if 'f' in cs['ops']:
            call_fprop(cs, x, w, torch.zeros(K, device='cuda') if cs['bias'] else None,
                       torch.zeros(N, P, Q, K, device='cuda', dtype=bf16) if _res_fprop(cs) else None)
            recs += _parse(capfd.readouterr().err, name, 'fprop', cs)
        if 'd' in cs['ops']:
            call_dgrad(cs, dy, w, torch.zeros(N, H, W, C, device='cuda', dtype=bf16) if _res_dgrad(cs) else None)
            recs += _parse(capfd.readouterr().err, name, 'dgrad', cs)
        if 'w' in cs['ops']:
            call_wgrad(cs, x, dy, torch.zeros(K, RS, C, device='cuda'))
            recs += _parse(capfd.readouterr().err, name, 'wgrad', cs)
    missing = []
    lines = []
    for label, pred in _requirements().items():
        hit = next((r for r in recs if pred(r)), None)
        if hit is None:
            missing.append(label)
        else:
            lines.append('covered: %-55s by %s %s' % (label, hit['case'], hit['op']))
    with capfd.disabled():
        print('\n' + '\n'.join(lines))
    assert not missing, 'configurations no longer reached by the sweep (SMs=%d): %s' % (_sm_count(), missing)
