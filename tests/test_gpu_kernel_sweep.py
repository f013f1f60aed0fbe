"""Generated sweep of the HBM-bound kernels -- BatchNorm (bn.cu), pooling (pool.cu), depthwise convolution (dwconv.cu),
squeeze-and-excitation and activation backward (se.cu), loss (loss.cu) and optimizer (optim.cu) -- against fp64 torch,
element by element.

The shapes are generated from the device's SM count, so that each intended launch regime (one block, fewer blocks than
accumulator replicas, grids at their caps, grid-stride loops that iterate, the unrolled loop of the BN backward final
reduction, ragged row chunks, ...) holds on any H100 variant.  Every case runs in two tiers:

* tier 1 -- exact arithmetic: small integer operands with dyadic scales (powers of two), so that every value the kernel
  forms is exactly representable: partial sums stay below 2^24 and bf16 outputs have at most 8 significant bits.  The
  result is then independent of summation order and FMA contraction and must equal the fp64 reference rounded once,
  bit for bit.  The tests assert these preconditions on the data they generate.
* tier 2 -- rounding-realistic: normal bf16 / fp32 operands; every element must satisfy
  |y - ref| <= rt * |ref| + c * absref, where absref is the same computation on absolute values, rt = 2^-8 (one bf16
  output rounding) for bf16 outputs and 0 for fp32 outputs.  Where a kernel's per-element arithmetic is a fixed short
  fp32 chain (bn_apply, act_bwd, avgpool_bwd, fused_sgd, grad_coef) the chain is restated and must hold to 1 ulp.

Outputs are written through out= into a NaN-filled view of a larger buffer whose guard regions must stay intact, and
every call is repeated on the same inputs and must give bitwise-identical results.  test_sweep_coverage runs the sweep
under torch.profiler and fails, naming the kernel, unless every kernel that the six source files compile into the
library (read from the library with cuobjdump) was launched.
"""
import math
import os
import re
import shutil
import subprocess
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, f64, u8 = torch.bfloat16, torch.float32, torch.float64, torch.uint8
DEV = 'cuda'

# tier-2 coefficients (|y - ref| beyond the output rounding, in units of absref), one per kernel family.  Calibrated on
# an NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit); the worst ratio observed over the sweep is given next to each
# (test_tier2_calibration_report prints them again).  The pool family showed no error beyond the bf16 rounding.
C_TIER2 = {
    'bn_stats': 2.0 ** -20,         # 1.7e-7 (5.7x): fp32 mean / invstd from one-pass fp32 partial sums of z and z^2
    'bn_sums': 2.0 ** -19,          # 2.1e-7 (9.1x): fp32 dgamma / dbeta (fp32 partials, fp64 across blocks)
    'bn_dz': 2.0 ** -21,            # 8.2e-8 (5.8x): bf16 dz = A*g + B*z + C with fp32 coefficients
    'bn_apply': 2.0 ** -22,         # ambiguity margin of the fp32 pre-activation (beyond 1 bf16 ulp, mask at 0 / 6)
    'bn_eval': 2.0 ** -20,          # 1.5e-7 (6.2x): rsqrtf (2 ulp) and one multiply-add
    'pool': 2.0 ** -22,             # 0: bf16 avgpool mean, max-pool backward sums of up to 4 terms
    'dw': 2.0 ** -24,               # 7.3e-9 (8.1x): bf16 depthwise fprop / dgrad (fp32 accumulation of <= 9 terms)
    'dw_wgrad': 2.0 ** -21,         # 6.5e-8 (7.4x): fp32 depthwise weight gradient
    'se': 2.0 ** -21,               # 5.7e-8 (8.4x): __expf-based sigmoid and fp32 reductions
    'ce': 2.0 ** -18,               # 4.3e-7 (8.9x): softmax cross-entropy, expf / logf of fp32 logits
    'sumsq': 2.0 ** -22,            # 3.7e-8 (6.4x): fp32 sum of squares
}
GUARD = 256               # elements before and after every output view
SENTINEL = -1536.0        # exact in bf16 and fp32
BYTE_SENTINEL = 0xA5
BN_ACCUM_FLOATS = 16 * 2 * 2048 * 2 + 64   # bn.cu: kReplicas x {sum, sum^2} x kBnMaxC doubles + ticket word
BN_TICKET_FLOAT = 16 * 2 * 2048 * 2        # index of the ticket counter (uint32) in the workspace
ACTS = (0, 1, 2)


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _gen(*key, device='cpu'):
    """the data generator of a case; on 'cuda' large draws cost no host time (other values)"""
    return torch.Generator(device=device).manual_seed(zlib.crc32('/'.join(str(k) for k in key).encode()))


# ------------------------------------------------------------------------------------------------ data
def _ints(shape, lo, hi, g, dtype=bf16, density=1.0):
    v = torch.randint(lo, hi + 1, shape, generator=g, device=g.device).to(f32)
    if density < 1.0:
        v = torch.where(torch.rand(shape, generator=g, device=g.device) < density, v, v.new_zeros(()))
    return v.to(DEV).to(dtype)


def _pick(shape, choices, g):
    t = torch.tensor(choices, dtype=f32)
    return t[torch.randint(0, len(choices), shape, generator=g, device=g.device).cpu()].to(DEV)


def _randn(shape, g, scale=1.0, shift=0.0, dtype=bf16):
    return (torch.randn(shape, generator=g, device=g.device) * scale + shift).to(DEV).to(dtype)


# ------------------------------------------------------------------------------------------------ guarded outputs
def _guarded(shape, dtype, fill=float('nan')):
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), BYTE_SENTINEL if dtype == u8 else SENTINEL, dtype=dtype, device=DEV)
    view = buf[GUARD:GUARD + n].view(shape)
    view.fill_(fill)
    return buf, view


def _bits(t):
    return t.view({bf16: torch.int16, f32: torch.int32, f64: torch.int64, u8: u8}[t.dtype])


def _same(a, b):
    return torch.equal(_bits(a), _bits(b))


def _check_guards(buf, n, what):
    sent = torch.tensor(BYTE_SENTINEL if buf.dtype == u8 else SENTINEL, dtype=buf.dtype, device=buf.device)
    assert _same(buf[:GUARD], sent.expand(GUARD)), '%s: wrote before its output' % what
    assert _same(buf[GUARD + n:], sent.expand(GUARD)), '%s: wrote past its output' % what


def _check_written(buf, view, what):
    _check_guards(buf, view.numel(), what)
    if view.dtype.is_floating_point:
        bad = view.isnan()
        assert not bool(bad.any()), '%s: %d of %d output elements never written' % (what, int(bad.sum()), bad.numel())


def _twice(fn, what):
    """run fn() twice on the same inputs: it returns a tuple of output tensors; both runs must agree bit for bit"""
    a = fn()
    b = fn()
    for i, (x, y) in enumerate(zip(a, b)):
        assert _same(x, y), '%s: output %d is not deterministic' % (what, i)
    return a


def _first_bad(bad):
    return tuple(bad.nonzero()[0].tolist())


def _exact(y, ref, what):
    """y must equal the fp64 reference rounded once to y's type"""
    want = ref.to(y.dtype)
    bad = _bits(y) != _bits(want)
    assert not bool(bad.any()), '%s: %d of %d elements differ, first at %s (got %r, want %r)' % (
        what, int(bad.sum()), bad.numel(), _first_bad(bad), float(y[bad][0]), float(want[bad][0]))


def _fits(x, dtype):
    return bool((x.to(dtype).double() == x).all())


def _exact_pre(values, dtype, what):
    for i, v in enumerate(values):
        assert _fits(v, dtype), '%s: precondition: intermediate %d is not exact in %s' % (what, i, dtype)


def _ulp(x, bits):
    """ulp of fp64 values in a binary format with `bits` significant bits (bf16: 8, fp32: 24); normal range"""
    _, e = torch.frexp(x.double().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x, dtype=f64), e - bits)


WORST = {}   # tier-2 family -> (worst (|y - ref| - rt |ref|) / absref, where)


def _bound(y, ref, absref, family, what):
    is_bf16 = y.dtype == bf16
    rt, c = (2.0 ** -8 if is_bf16 else 0.0), C_TIER2[family]
    yd = y.double()
    assert bool(torch.isfinite(yd).all()), '%s: non-finite output' % what
    excess = (yd - ref).abs() - rt * ref.abs()
    ratio = float((excess / absref.clamp_min(1e-300)).max()) if excess.numel() else -math.inf
    if ratio > WORST.get(family, (-math.inf, ''))[0]:
        WORST[family] = (ratio, what)
    bad = excess > c * absref
    assert not bool(bad.any()), '%s: %d of %d elements outside |y-ref| <= %g |ref| + %g absref (worst ratio %.3g), ' \
        'first at %s' % (what, int(bad.sum()), bad.numel(), rt, c, ratio, _first_bad(bad))


def _within_ulps(y, ref, n, bits, what):
    bad = (y.double() - ref).abs() > n * _ulp(ref, bits)
    assert not bool(bad.any()), '%s: %d elements beyond %d ulp, first at %s' % (what, int(bad.sum()), n, _first_bad(bad))


# ================================================================================================ BatchNorm
BN_CS = (8, 24, 64, 1000, 1024, 1032, 1280, 2048)


def _bn_geom(C):
    vec = 8 if C > 1024 else 4
    return dict(vec=vec, minb=3 if vec == 8 else 4, rpi_f=256 // (C // 8), rpi_b=256 // (C // vec))


def _reduce_blocks(M, C, sm):
    """bn.cu reduce_blocks: the bn_stats grid"""
    rpi = _bn_geom(C)['rpi_f']
    want = (-(-M // rpi) + 7) // 8
    cap = min(max(1200000 // (2 * C), sm), 6 * sm)
    return max(1, min(want, cap)), cap


def _partial_blocks(M, C, sm):
    """bn.cu partial_blocks: the bn_bwd_reduce grid (= the final kernel's block count)"""
    g = _bn_geom(C)
    want = (-(-M // g['rpi_b']) + 3) // 4
    cap = min(g['minb'] * sm, 6 * 148)
    return max(1, min(want, cap)), cap


def bn_sweep(sm):
    """name -> (M, C).  Per C: M = 7 (below rows_per_iter for C <= 256), ~10 backward blocks with M % 8 == 7, ~101
    blocks with M % 8 == 1, the reduce_blocks / partial_blocks caps with M % 8 == 7, and M = 4096 (dz exact)."""
    cases = {}
    for C in BN_CS:
        rb = _bn_geom(C)['rpi_b']
        _, cap_f = _reduce_blocks(1, C, sm)
        _, cap_b = _partial_blocks(1, C, sm)
        cases['c%d_m7' % C] = (7, C)
        cases['c%d_few' % C] = (40 * rb - 1, C)
        cases['c%d_mid' % C] = (400 * rb + 1, C)
        cases['c%d_cap' % C] = (max(cap_b * 4 * rb, cap_f * 8 * _bn_geom(C)['rpi_f']) + 7, C)
        cases['c%d_pow2' % C] = (4096, C)
    return cases


def _bn_regimes(sm):
    """the launch regimes bn_sweep is meant to reach, as a check on the generated shapes"""
    seen = set()
    for M, C in bn_sweep(sm).values():
        pb, capb = _partial_blocks(M, C, sm)
        rbk, capf = _reduce_blocks(M, C, sm)
        seen.add('final < 64' if pb < 64 else ('final 64..192' if pb <= 192 else ('final > 256' if pb > 256 else '')))
        seen.add('partial blocks < 16' if pb < 16 else '')
        seen.add('partial blocks at cap' if pb == capb else '')
        seen.add('stats blocks at cap' if rbk == capf else '')
        seen.add('stats one block' if rbk == 1 else '')
        seen.add('stats blocks < 16' if 1 < rbk < 16 else '')
        seen.add('M < rows_per_iter' if M < _bn_geom(C)['rpi_b'] else '')
        seen.add('idle threads' if 256 % (C // _bn_geom(C)['vec']) else '')
        seen.add('M %% 8 == %d' % (M % 8))
    return seen


_BN_NAMES = list(bn_sweep(132))


def _bn_case(name):
    return bn_sweep(_sm_count())[name]


def test_bn_sweep_regimes():
    want = {'final < 64', 'final 64..192', 'final > 256', 'partial blocks < 16', 'partial blocks at cap',
            'stats blocks at cap', 'stats one block', 'stats blocks < 16', 'M < rows_per_iter', 'idle threads',
            'M % 8 == 1', 'M % 8 == 7'}
    for sm in (_sm_count(), 132, 114):
        missing = want - _bn_regimes(sm)
        assert not missing, 'BN regimes not reached with %d SMs: %s' % (sm, sorted(missing))


def _bn_workspace(C):
    return torch.zeros(_ops().bn_workspace_floats(C), device=DEV)


def _check_ws_zero(ws, what):
    acc = ws[:BN_ACCUM_FLOATS]
    assert not bool(acc.ne(0).any()), '%s: %d accumulator / ticket words left nonzero' % (what, int(acc.ne(0).sum()))


def _stats_ref(s1, s2, M, eps):
    """bn.cu's finalisation formula on fp64 sums: (mean fp32, fp64 biased variance, invstd fp32)"""
    mu = s1 / M
    var = (s2 / M - mu * mu).clamp_min(0.0)
    istd = (1.0 / torch.sqrt(var + float(torch.tensor(eps, dtype=f32)))).float()
    return mu.float(), var, istd


def _check_coeffs(mean, invstd, scale, shift, s1, s2, M, eps, gamma, beta, what):
    mu32, var, istd = _stats_ref(s1, s2, M, eps)
    _exact(mean, mu32.double(), '%s mean' % what)
    _within_ulps(invstd, istd.double(), 1, 24, '%s invstd' % what)
    g = gamma if gamma is not None else torch.ones_like(mean)
    b = beta if beta is not None else torch.zeros_like(mean)
    assert _same(scale, g * invstd), '%s: scale != gamma * invstd' % what
    fused = (b.double() - mean.double() * scale.double()).float().double()
    split = (b - mean * scale).double()
    d = torch.minimum((shift.double() - fused).abs(), (shift.double() - split).abs())
    bad = d > _ulp(fused, 24)
    assert not bool(bad.any()), '%s shift: %d elements beyond 1 ulp of beta - mean*scale' % (what, int(bad.sum()))
    return var


def _running_ref(rm, rv, mean, var, M, f):
    unb = (var * M / (M - 1) if M > 1 else var).float().double()
    f = float(torch.tensor(f, dtype=f32))
    g = float(torch.tensor(1.0 - f, dtype=f32))
    return (g * rm.double() + f * mean.double(), g * rv.double() + f * unb,
            g * rm.double().abs() + f * mean.double().abs(), g * rv.double().abs() + f * unb.abs())


def _check_running(rm_new, rv_new, ref, what):
    rm_ref, rv_ref, rm_abs, rv_abs = ref
    for y, r, a, n in ((rm_new, rm_ref, rm_abs, 'running_mean'), (rv_new, rv_ref, rv_abs, 'running_var')):
        bad = (y.double() - r).abs() > 2.0 ** -20 * a
        assert not bool(bad.any()), '%s %s: %d elements off, first at %s' % (what, n, int(bad.sum()), _first_bad(bad))


def _stat_outputs(C):
    return [_guarded((C,), f32) for _ in range(4)]


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', _BN_NAMES)
def test_bn_stats(name, tier):
    check_bn_stats(*_bn_case(name), tier, name)


def check_bn_stats(M, C, tier, name, rng='cpu'):
    """bn_stats on an [M, C] z in the given tier; name seeds the data and names the case"""
    ops = _ops()
    g = _gen('bn_stats', name, tier, device=rng)
    eps = 1e-5
    if tier == 1:
        z = _ints((M, C), -4, 4, g)
        gamma, beta = _pick((C,), [-2, -1, -0.5, 0.5, 1, 2], g), _pick((C,), [-1, -0.25, 0, 0.5, 1.5], g)
        blocks, _ = _reduce_blocks(M, C, _sm_count())
        assert -(-M // blocks) * 16 < 2 ** 24, 'precondition: block partials of z^2 are not exact in fp32'
    else:
        z = _randn((M, C), g, 1.5, 0.3)
        gamma, beta = _randn((C,), g, 0.5, 1.0, f32), _randn((C,), g, 0.3, 0.0, f32)
    zd = z.double()
    s1, s2 = zd.sum(0), (zd * zd).sum(0)
    rm0, rv0 = _randn((C,), g, 1.0, 0.0, f32), _randn((C,), g, 0.2, 1.0, f32).abs()
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.zeros((), dtype=torch.int64, device=DEV)
    ws = _bn_workspace(C)

    def run(momentum, with_affine=True, with_running=True):
        outs = _stat_outputs(C)
        ops.bn_stats(z, gamma if with_affine else None, beta if with_affine else None, eps, momentum,
                     rm if with_running else None, rv if with_running else None, nbt if with_running else None,
                     *[v for _, v in outs], ws)
        torch.cuda.synchronize()
        for (buf, v), n in zip(outs, ('mean', 'invstd', 'scale', 'shift')):
            _check_written(buf, v, '%s bn_stats %s' % (name, n))
        _check_ws_zero(ws, '%s bn_stats' % name)
        return tuple(v for _, v in outs)

    mean, invstd, scale, shift = run(0.1)
    if tier == 1:
        var = _check_coeffs(mean, invstd, scale, shift, s1, s2, M, eps, gamma, beta, '%s bn_stats' % name)
    else:
        mu, var = s1 / M, (s2 / M - (s1 / M) ** 2).clamp_min(0)
        absz, sq = zd.abs().sum(0) / M, s2 / M
        _bound(mean, mu, absz, 'bn_stats', '%s mean' % name)
        istd = 1 / torch.sqrt(var + eps)
        _bound(invstd, istd, istd * sq / (var + eps), 'bn_stats', '%s invstd' % name)
        var = (1 / invstd.double() ** 2 - float(torch.tensor(eps, dtype=f32))).clamp_min(0)   # the kernel's variance
        assert _same(scale, gamma * invstd)
    assert int(nbt) == 1
    _check_running(rm, rv, _running_ref(rm0, rv0, mean, var, M, 0.1), '%s bn_stats momentum 0.1' % name)
    # the same z again: identical coefficients, the running statistics move once more, the counter counts
    rm1, rv1 = rm.clone(), rv.clone()
    again = run(0.1)
    for a, b in zip((mean, invstd, scale, shift), again):
        assert _same(a, b), '%s bn_stats: not deterministic' % name
    _check_running(rm, rv, _running_ref(rm1, rv1, mean, var, M, 0.1), '%s bn_stats second call' % name)
    assert int(nbt) == 2
    # cumulative moving average (momentum=None): factor 1 / (num_batches_tracked + 1)
    rm2, rv2 = rm.clone(), rv.clone()
    run(None)
    _check_running(rm, rv, _running_ref(rm2, rv2, mean, var, M, 1.0 / 3.0), '%s bn_stats momentum None' % name)
    assert int(nbt) == 3
    # NULL gamma / beta / running pointers: scale = invstd, shift = -mean * invstd; nothing else is touched
    rm3, rv3 = rm.clone(), rv.clone()
    m4, i4, s4, h4 = run(0.1, with_affine=False, with_running=False)
    assert _same(m4, mean) and _same(i4, invstd)
    if tier == 1:
        _check_coeffs(m4, i4, s4, h4, s1, s2, M, eps, None, None, '%s bn_stats without affine' % name)
    assert _same(rm, rm3) and _same(rv, rv3) and int(nbt) == 3


def test_bn_stats_shifted_mean():
    """|mean| = 16 std: the one-pass fp32 sums of z and z^2 cancel; invstd must still be within 2^-10"""
    ops = _ops()
    M, C = 65536, 64
    g = _gen('bn_shift')
    z = _randn((M, C), g, 1.0, 16.0)
    zd = z.double()
    var = zd.var(0, unbiased=False)
    outs = [torch.empty(C, device=DEV) for _ in range(4)]
    ops.bn_stats(z, None, None, 1e-5, 0.1, None, None, None, *outs, _bn_workspace(C))
    err = float(((outs[1].double() - 1 / torch.sqrt(var + 1e-5)).abs() * torch.sqrt(var + 1e-5)).max())
    assert err <= 2.0 ** -10, 'invstd relative error %.3g at |mean| = 16 std' % err
    WORST['bn_stats shifted 16 std (relative invstd error)'] = (err, 'M=%d C=%d' % (M, C))
    z64 = _randn((M, C), g, 1.0, 64.0)
    var64 = z64.double().var(0, unbiased=False)
    ops.bn_stats(z64, None, None, 1e-5, 0.1, None, None, None, *outs, _bn_workspace(C))
    err64 = float(((outs[1].double() - 1 / torch.sqrt(var64 + 1e-5)).abs() * torch.sqrt(var64 + 1e-5)).max())
    WORST['bn_stats shifted 64 std (relative invstd error, estimate only)'] = (err64, 'M=%d C=%d' % (M, C))


@pytest.mark.parametrize('C', [8, 24, 1000, 2048])
def test_bn_finalize(C):
    """bn_finalize on known fp64 sums in the documented [16 replicas][2][C] workspace layout (the layout the fused
    convolution statistics and SyncBatchNorm write), both momentum modes (momentum=None: separate counter bump)"""
    ops = _ops()
    g = _gen('bn_finalize', C)
    M = 3000 + C
    s1 = torch.randint(-4 * M, 4 * M, (C,), generator=g).double()
    s2 = (s1 * s1 / M + torch.randint(1, 8 * M, (C,), generator=g).double()).round()   # variance > 0
    parts1 = torch.randint(-1000, 1000, (16, C), generator=g).double()
    parts2 = torch.randint(0, 1000, (16, C), generator=g).double()
    parts1[0] += s1 - parts1.sum(0)
    parts2[0] += s2 - parts2.sum(0)
    s1, s2 = s1.to(DEV), s2.to(DEV)
    gamma, beta = _pick((C,), [-2, -1, 0.5, 1, 2], g), _pick((C,), [-1, 0, 0.25, 1], g)
    rm, rv = _randn((C,), g, 1.0, 0.0, f32), _randn((C,), g, 0.2, 1.0, f32).abs()
    nbt = torch.full((), 5, dtype=torch.int64, device=DEV)
    ws = _bn_workspace(C)
    for momentum, n_after in ((0.1, 6), (None, 7), (0.25, 8)):
        ws[:16 * 2 * C * 2].view(f64).view(16, 2, C).copy_(torch.stack([parts1, parts2], 1).to(DEV))
        rm0, rv0 = rm.clone(), rv.clone()
        f = 0.1 if momentum == 0.1 else (0.25 if momentum == 0.25 else 1.0 / (int(nbt) + 1))
        outs = _stat_outputs(C)
        ops.bn_finalize(M, C, gamma, beta, 1e-5, momentum, rm, rv, nbt, *[v for _, v in outs], ws)
        torch.cuda.synchronize()
        for (buf, v), n in zip(outs, ('mean', 'invstd', 'scale', 'shift')):
            _check_written(buf, v, 'bn_finalize %s' % n)
        _check_ws_zero(ws, 'bn_finalize')
        mean, invstd, scale, shift = [v for _, v in outs]
        var = _check_coeffs(mean, invstd, scale, shift, s1, s2, M, 1e-5, gamma, beta, 'bn_finalize C=%d' % C)
        _check_running(rm, rv, _running_ref(rm0, rv0, mean, var, M, f), 'bn_finalize momentum %s' % momentum)
        assert int(nbt) == n_after, 'num_batches_tracked %d, want %d' % (int(nbt), n_after)
    # no running buffers: nothing is bumped
    ws[:16 * 2 * C * 2].view(f64).view(16, 2, C).copy_(torch.stack([parts1, parts2], 1).to(DEV))
    outs = [torch.empty(C, device=DEV) for _ in range(4)]
    ops.bn_finalize(M, C, None, None, 1e-5, None, None, None, nbt, *outs, ws)
    torch.cuda.synchronize()
    assert int(nbt) == 8
    _check_ws_zero(ws, 'bn_finalize without running buffers')


@pytest.mark.parametrize('C', [8, 1000, 2048])
def test_bn_eval_coeffs(C):
    ops = _ops()
    g = _gen('bn_eval', C)
    gamma, beta = _randn((C,), g, 0.5, 1.0, f32), _randn((C,), g, 0.3, 0.0, f32)
    rm, rv = _randn((C,), g, 1.0, 0.0, f32), _randn((C,), g, 1.0, 0.0, f32).abs() + 1e-3
    for gm, bt in ((gamma, beta), (None, None)):
        (bs, sc), (bh, sh) = _guarded((C,), f32), _guarded((C,), f32)
        ops.bn_eval_coeffs(gm, bt, rm, rv, 1e-5, sc, sh)
        torch.cuda.synchronize()
        _check_written(bs, sc, 'bn_eval_coeffs scale')
        _check_written(bh, sh, 'bn_eval_coeffs shift')
        gd = gm.double() if gm is not None else torch.ones(C, dtype=f64, device=DEV)
        bd = bt.double() if bt is not None else torch.zeros(C, dtype=f64, device=DEV)
        istd = 1 / torch.sqrt(rv.double() + float(torch.tensor(1e-5, dtype=f32)))
        _bound(sc, gd * istd, (gd * istd).abs(), 'bn_eval', 'bn_eval_coeffs scale')
        _bound(sh, bd - rm.double() * gd * istd, bd.abs() + (rm.double() * gd * istd).abs(), 'bn_eval',
               'bn_eval_coeffs shift')


# ---- bn_apply
def _act(v, act):
    return v.clamp_min(0) if act == 1 else (v.clamp(0, 6) if act == 2 else v)


def _act_pass(pre, act):
    if act == 1:
        return pre > 0
    if act == 2:
        return (pre > 0) & (pre < 6)
    return torch.ones_like(pre, dtype=torch.bool)


def _unpack_mask(bits, M, C):
    """row-quad layout: byte (row % 4) of word (row // 4) * (C / 8) + v8, bit i = channel 8 v8 + i"""
    by_row = bits.view(-1, C // 8, 4).permute(0, 2, 1).reshape(-1, C // 8)
    shifts = torch.arange(8, device=bits.device, dtype=torch.int32)
    return ((by_row.to(torch.int32).unsqueeze(-1) >> shifts) & 1).view(-1, C).bool(), by_row[M:]


def _apply_mask_bytes(M, C):
    return (M + 7) // 8 * 8 * (C // 8)


def _bn_apply_call(z, sc, sh, act, mode, extra, with_mask, fill):
    """-> (y, mask buffer view); the mask view is pre-filled with `fill`"""
    ops = _ops()
    M, C = z.shape
    by, y = _guarded((M, C), bf16)
    bm, mask = _guarded((_apply_mask_bytes(M, C),), u8, fill) if with_mask else (None, None)
    kw = {}
    if mode == 1:
        kw = dict(residual=extra[0])
    elif mode == 2:
        kw = dict(z2=extra[0], scale2=extra[1], shift2=extra[2])
    ops.bn_apply(z, sc, sh, act, out=y, act_mask=mask, **kw)
    torch.cuda.synchronize()
    _check_written(by, y, 'bn_apply')
    if bm is not None:
        _check_guards(bm, mask.numel(), 'bn_apply mask')
        return y, mask
    return y, torch.zeros(0, dtype=u8, device=DEV)


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', _BN_NAMES)
def test_bn_apply(name, tier):
    check_bn_apply(*_bn_case(name), tier, name)


def check_bn_apply(M, C, tier, name, rng='cpu'):
    """bn_apply (three modes x three activations, with and without the mask) on [M, C] in the given tier"""
    g = _gen('bn_apply', name, tier, device=rng)
    if tier == 1:
        z, res, z2 = _ints((M, C), -8, 8, g), _ints((M, C), -8, 8, g), _ints((M, C), -8, 8, g)
        sc, sc2 = _pick((C,), [-2, -1, -0.5, 0.5, 1, 2], g), _pick((C,), [-1, -0.5, 0.5, 1], g)
        sh, sh2 = _pick((C,), [-4, -1.5, -0.5, 0, 0.5, 2, 6], g), _pick((C,), [-2, 0, 0.5, 1], g)
    else:
        z, res, z2 = _randn((M, C), g, 2.0), _randn((M, C), g, 2.0), _randn((M, C), g, 2.0)
        sc, sc2 = _randn((C,), g, 1.0, 0.0, f32), _randn((C,), g, 1.0, 0.0, f32)
        sh, sh2 = _randn((C,), g, 2.0, 1.0, f32), _randn((C,), g, 1.0, 0.0, f32)
    zd = z.double()
    base = zd * sc.double() + sh.double()
    babs = (zd * sc.double()).abs() + sh.double().abs()
    for mode in (0, 1, 2):
        if mode == 0:
            pre, absref, extra = base, babs, ()
        elif mode == 1:
            pre, absref, extra = base + res.double(), babs + res.double().abs(), (res,)
        else:
            t = z2.double() * sc2.double() + sh2.double()
            pre = base + t
            absref = babs + (z2.double() * sc2.double()).abs() + sh2.double().abs()
            extra = (z2, sc2, sh2)
        if tier == 1:
            _exact_pre([pre], bf16, '%s bn_apply mode %d' % (name, mode))
        for act in ACTS:
            what = '%s bn_apply mode %d act %d' % (name, mode, act)
            ref = _act(pre, act)
            y0, _ = _bn_apply_call(z, sc, sh, act, mode, extra, False, 0)
            y, m1 = _bn_apply_call(z, sc, sh, act, mode, extra, True, 0x5A)
            y2, m2 = _bn_apply_call(z, sc, sh, act, mode, extra, True, BYTE_SENTINEL)
            assert _same(y, y0) and _same(y, y2), '%s: output depends on the mask or is not deterministic' % what
            if tier == 1:
                _exact(y, ref, what)
            else:
                # restated chain: one bf16 rounding of an fp32 value (1 bf16 ulp), plus the fp32 intermediate's error
                bad = (y.double() - ref).abs() > _ulp(ref, 8) + C_TIER2['bn_apply'] * absref
                assert not bool(bad.any()), '%s: %d elements beyond 1 ulp, first at %s' % (what, int(bad.sum()),
                                                                                        _first_bad(bad))
            bits1, pad1 = _unpack_mask(m1, M, C)
            bits2, pad2 = _unpack_mask(m2, M, C)
            assert torch.equal(bits1[:M], bits2[:M]), '%s: mask bits of rows < M not all written' % what
            assert bool((pad1 == 0x5A).all()) and bool((pad2 == BYTE_SENTINEL).all()), \
                '%s: mask padding bytes of rows >= M were written' % what
            want = _act_pass(pre, act)
            bad = bits1[:M] != want
            if tier == 2:     # the fp32 pre-activation may sit on the other side of 0 / 6 within its rounding error
                amb = (pre.abs() <= C_TIER2['bn_apply'] * absref) | ((pre - 6).abs() <= C_TIER2['bn_apply'] * absref)
                bad &= ~amb
            assert not bool(bad.any()), '%s: %d mask bits differ from the fp64 pre-activation test, first at %s' % (
                what, int(bad.sum()), _first_bad(bad))


# ---- BatchNorm backward
def _bwd_call(dy, y, z, act, mean, invstd, gamma, beta, mask, dg0, db0, ws_fill):
    """bn_bwd_reduce + bn_bwd_dx -> (sums, dgamma_acc, dbeta_acc, dz, g_out); the workspace partial rows are filled with
    ws_fill beforehand (any content is allowed there)"""
    ops = _ops()
    M, C = z.shape
    ws = _bn_workspace(C)
    ws[BN_ACCUM_FLOATS:] = ws_fill
    bs, sums = _guarded((2 * C,), f32)
    dg, db = dg0.clone(), db0.clone()
    ops.bn_bwd_reduce(dy, y, z, act, mean, invstd, gamma, beta, sums, dg, db, ws, act_mask=mask)
    bz, dz = _guarded((M, C), bf16)
    bg, gout = _guarded((M, C), bf16)
    ops.bn_bwd_dx(dy, y, z, act, mean, invstd, gamma, beta, sums, dz=dz, g_out=gout, act_mask=mask)
    torch.cuda.synchronize()
    _check_written(bs, sums, 'bn_bwd_reduce sums')
    _check_written(bz, dz, 'bn_bwd_dx dz')
    _check_written(bg, gout, 'bn_bwd_dx g_out')
    _check_ws_zero(ws, 'bn_bwd_reduce')
    return sums, dg, db, dz, gout


def _mask_with_padding(mask, M, C, pad):
    """a copy of a row-quad mask with the bytes of rows >= M (the padding to 8 rows) set to `pad`"""
    m = mask.clone()
    rows = torch.arange(M, m.numel() // (C // 8), device=DEV)
    idx = ((rows // 4).view(-1, 1) * (C // 8) + torch.arange(C // 8, device=DEV)) * 4 + (rows % 4).view(-1, 1)
    m[idx.reshape(-1)] = pad
    return m


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', _BN_NAMES)
def test_bn_backward(name, tier):
    check_bn_backward(*_bn_case(name), tier, name, affine=not name.endswith('_few'))   # '_few': NULL gamma / beta


def check_bn_backward(M, C, tier, name, affine=True, rng='cpu'):
    """bn_bwd_reduce / bn_bwd_dx on [M, C]: every (VEC, ROWS, MINB) instantiation the shape selects x every activation
    x the three activation sources (0: recomputed from z, 1: y, 2: mask bits)"""
    ops = _ops()
    g = _gen('bn_bwd', name, tier, device=rng)
    if tier == 1:
        z = _ints((M, C), -4, 4, g)
        dy = _ints((M, C), -3, 3, g, density=min(1.0, 2.0 ** 19 / (M * 6)))
        mean = _pick((C,), [-1, -0.5, 0, 0.5, 1], g)
        invstd = _pick((C,), [0.5, 1, 2], g)
        gamma, beta = _pick((C,), [-2, -1, -0.5, 0.5, 1, 2], g), _pick((C,), [-1, -0.5, 0, 0.5, 1, 3], g)
        if not affine:
            gamma = beta = None
        gm = gamma if gamma is not None else torch.ones(C, device=DEV)
        bt = beta if beta is not None else torch.zeros(C, device=DEV)
        scale = gm * invstd
        shift = bt - mean * scale
        _exact_pre([scale.double(), shift.double(), z.double() * scale.double() + shift.double()], bf16,
                   '%s scale / shift / pre-activation' % name)
    else:
        z = _randn((M, C), g, 1.5, 0.3)
        dy = _randn((M, C), g)
        gamma, beta = _randn((C,), g, 0.5, 1.0, f32), _randn((C,), g, 0.3, 0.0, f32)
        gamma[::5] *= -1
        if not affine:
            gamma = beta = None
        mean, invstd, scale, shift = [torch.empty(C, device=DEV) for _ in range(4)]
        ops.bn_stats(z, gamma, beta, 1e-5, 0.1, None, None, None, mean, invstd, scale, shift, _bn_workspace(C))
        gm = gamma if gamma is not None else torch.ones(C, device=DEV)
    dg0 = _ints((C,), -8, 8, g, f32)
    db0 = _ints((C,), -8, 8, g, f32)
    zd, dyd = z.double(), dy.double()
    mu, isd, gmd = mean.double(), invstd.double(), gm.double()
    pre = zd * scale.double() + shift.double() if tier == 1 else None
    for act in ACTS:
        y, mask = _bn_apply_call(z, scale, shift, act, 0, (), True, 0)
        results = {}
        for src in (0, 1, 2):
            if act == 0 and src:
                continue
            what = '%s act %d src %d' % (name, act, src)
            yy = y if src == 1 else None
            mk = mask if src == 2 else None
            r1 = _bwd_call(dy, yy, z, act, mean, invstd, gamma, beta, mk, dg0, db0, 0.0)
            # repeat: partial-row region full of NaN, mask padding bytes 0xFF instead of 0x00
            mk2 = _mask_with_padding(mask, M, C, 0xFF) if src == 2 else None
            r2 = _bwd_call(dy, yy, z, act, mean, invstd, gamma, beta, mk2, dg0, db0, float('nan'))
            for i, (a, b) in enumerate(zip(r1, r2)):
                assert _same(a, b), '%s: output %d changed with NaN workspace / 0xFF mask padding or is not ' \
                    'deterministic' % (what, i)
            results[src] = r1
            sums, dgam, dbet, dz, gout = r1
            # g = dy * act'(.) is exact in both tiers
            if tier == 1:
                want_g = torch.where(_act_pass(pre, act), dyd, 0.0)
                _exact(gout, want_g, '%s g_out' % what)
            gd = gout.double()
            xm = zd - mu
            dgam_ref, dbet_ref = (gd * xm).sum(0) * isd, gd.sum(0)
            dgam_abs, dbet_abs = (gd.abs() * xm.abs()).sum(0) * isd, gd.abs().sum(0)
            if tier == 1:
                assert float(dgam_abs.max()) < 2 ** 24 and float(dbet_abs.max()) < 2 ** 24, 'precondition: sums'
                _exact(sums[:C], dgam_ref, '%s dgamma' % what)
                _exact(sums[C:], dbet_ref, '%s dbeta' % what)
            else:
                _bound(sums[:C], dgam_ref, dgam_abs, 'bn_sums', '%s dgamma' % what)
                _bound(sums[C:], dbet_ref, dbet_abs, 'bn_sums', '%s dbeta' % what)
            # dgamma_acc / dbeta_acc: += onto the initial values (one fp32 add of the returned sums)
            assert _same(dgam, dg0 + sums[:C]) and _same(dbet, db0 + sums[C:]), '%s: dgamma/dbeta accumulation' % what
            # dz from the kernel's own sums (checked above)
            dgk, dbk = sums[:C].double(), sums[C:].double()
            A = gmd * isd
            B = -gmd * isd * isd * dgk / M
            Cc = -A * dbk / M - B * mu
            dz_ref = A * gd + B * zd + Cc
            dz_abs = (A * gd).abs() + (B * zd).abs() + (A * dbk / M).abs() + (B * mu).abs()
            if tier == 2 or M & (M - 1):
                _bound(dz, dz_ref, dz_abs, 'bn_dz', '%s dz' % what)
            else:
                _exact_pre([A, B, Cc, A * gd, B * zd, A * gd + B * zd, B * zd + Cc, A * gd + Cc, dz_ref], f32,
                           '%s dz' % what)
                _exact(dz, dz_ref, '%s dz' % what)
        if act == 0:
            continue
        # the three sources agree: SRC 0 and SRC 2 both test the fp32 pre-activation, so g_out is identical; SRC 2
        # splits the rows between blocks in multiples of 8, so its fp32 sums (and dz) match only in the exact tier.
        # SRC 1 tests the bf16 output (same row split as SRC 0) and may differ only where a ReLU6 output rounds onto 6
        for i in (range(5) if tier == 1 else (4,)):
            assert _same(results[0][i], results[2][i]), '%s act %d: SRC 0 and SRC 2 differ (output %d)' % (name, act, i)
        diff = _bits(results[1][4]) != _bits(results[0][4])
        if tier == 1 or act == 1:
            assert not bool(diff.any()), '%s act %d: SRC 1 g_out differs from SRC 0' % (name, act)
            for i in range(5):
                assert _same(results[0][i], results[1][i]), '%s act %d: SRC 1 differs (output %d)' % (name, act, i)
        else:
            allowed = y.double() == 6
            assert not bool((diff & ~allowed).any()), '%s act 2: SRC 1 differs from SRC 0 off the clamp' % name


# ================================================================================================ pooling
def _pool_out(n):
    return (n - 1) // 2 + 1


def _maxpool_ref(x):
    """3x3 / stride 2 / pad 1 on [N,H,W,C] (fp64): the kernel's scan rule -- window positions in (r, s) order, the
    first valid one initialises, later ones win when strictly greater or NaN (ATen's rule)"""
    N, H, W, C = x.shape
    OH, OW = _pool_out(H), _pool_out(W)
    xd = x.double()
    best = torch.full((N, OH, OW, C), float('-inf'), dtype=f64, device=x.device)
    idx = torch.zeros((N, OH, OW, C), dtype=torch.int64, device=x.device)
    first = torch.ones((N, OH, OW, C), dtype=torch.bool, device=x.device)
    pad = torch.full((N, 2 * OH + 2, 2 * OW + 2, C), float('nan'), dtype=f64, device=x.device)
    pad[:, 1:H + 1, 1:W + 1] = xd
    valid = torch.zeros((2 * OH + 2, 2 * OW + 2), dtype=torch.bool, device=x.device)
    valid[1:H + 1, 1:W + 1] = True
    for r in range(3):
        for s in range(3):
            v = pad[:, r:r + 2 * OH:2, s:s + 2 * OW:2]
            ok = valid[r:r + 2 * OH:2, s:s + 2 * OW:2].view(1, OH, OW, 1)
            take = ok & (first | (v > best) | v.isnan())
            best = torch.where(take, v, best)
            idx = torch.where(take, torch.full_like(idx, r * 3 + s), idx)
            first = first & ~ok
    return best, idx.to(u8)


def _maxpool_bwd_ref(dy, am, in_shape):
    N, H, W, C = in_shape
    OH, OW = dy.shape[1], dy.shape[2]
    dx = torch.zeros((N, 2 * OH + 2, 2 * OW + 2, C), dtype=f64, device=dy.device)
    dxa = torch.zeros_like(dx)
    a = am.long()
    for k in range(9):
        r, s = divmod(k, 3)
        sel = (a == k).double()
        dx[:, r:r + 2 * OH:2, s:s + 2 * OW:2] += dy.double() * sel
        dxa[:, r:r + 2 * OH:2, s:s + 2 * OW:2] += dy.double().abs() * sel
    return dx[:, 1:H + 1, 1:W + 1], dxa[:, 1:H + 1, 1:W + 1]


def maxpool_sweep(sm):
    """name -> (N, H, W, C): H, W in {1, 2, odd, even}; J = ceil(H/2) above the 14-row chunk; C = 8 and 2048; the
    backward grid over its 16-per-SM cap (grid-stride loop) and the forward grid over its cap"""
    return {
        'h1w1_c8': (3, 1, 1, 8), 'h2w2_c8': (2, 2, 2, 8), 'h1w7_c16': (2, 1, 7, 16), 'h7w1_c8': (2, 7, 1, 8),
        'h5w6_c24': (3, 5, 6, 24), 'h31w30_c8': (2, 31, 30, 8), 'h60w33_c8': (1, 60, 33, 8),
        'h9w8_c2048': (2, 9, 8, 2048), 'h2w3_c2048': (2, 2, 3, 2048), 'stem_c64': (2, 112, 112, 64),
        'bwd_over_cap': (-(-3 * sm // 2), 2, 64, 256),
        'fwd_over_cap': (24 * sm, 2, 2, 2048),
    }


_POOL_NAMES = list(maxpool_sweep(132))


def _maxpool_call(x, fused=None):
    """-> (y, argmax) through guarded outputs (argmax bytes pre-filled with 0xEE, never a valid index)"""
    ops = _ops()
    N, H, W, C = x.shape
    shape = (N, _pool_out(H), _pool_out(W), C)
    by, y = _guarded(shape, bf16, 17408.0)
    ba, am = _guarded(shape, u8, 0xEE)
    if fused is None:
        ops.maxpool_fwd(x, out=y, argmax_out=am)
    else:
        ops.bn_apply_maxpool(x, fused[0], fused[1], fused[2], out=y, argmax_out=am)
    torch.cuda.synchronize()
    _check_guards(by, y.numel(), 'maxpool y')
    _check_guards(ba, am.numel(), 'maxpool argmax')
    assert not bool((am > 8).any()), 'maxpool: argmax bytes not written'
    assert not bool((y == 17408.0).any()), 'maxpool: outputs not written'
    return y, am


def _maxpool_bwd_call(dy, am, shape):
    b, dx = _guarded(shape, bf16)
    _ops().maxpool_bwd(dy, am, shape, out=dx)
    torch.cuda.synchronize()
    _check_written(b, dx, 'maxpool_bwd')
    return (dx,)


def _check_pool_values(y, ref, what):
    assert torch.equal(y.isnan(), ref.isnan()), '%s: NaN positions differ' % what
    ok = ~ref.isnan()
    _exact(y[ok], ref[ok], what)


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', _POOL_NAMES)
def test_maxpool(name, tier):
    N, H, W, C = maxpool_sweep(_sm_count())[name]
    g = _gen('maxpool', name, tier)
    x = _ints((N, H, W, C), -3, 3, g) if tier == 1 else _randn((N, H, W, C), g)
    y, am = _twice(lambda: _maxpool_call(x), name)
    ref, am_ref = _maxpool_ref(x)
    _check_pool_values(y, ref, '%s maxpool y' % name)
    bad = am != am_ref
    assert not bool(bad.any()), '%s: %d argmax bytes break the first-in-scan-order rule, first at %s' % (
        name, int(bad.sum()), _first_bad(bad))
    dy = _ints(y.shape, -3, 3, g) if tier == 1 else _randn(y.shape, g)
    dx, = _twice(lambda: _maxpool_bwd_call(dy, am, (N, H, W, C)), name)
    ref, absref = _maxpool_bwd_ref(dy, am, (N, H, W, C))
    if tier == 1:
        _exact(dx, ref, '%s maxpool_bwd' % name)
    else:
        _bound(dx, ref, absref, 'pool', '%s maxpool_bwd' % name)


def test_maxpool_nan_and_neg_inf():
    """windows holding NaN (the last NaN in scan order wins and propagates) and windows of -inf only (the first
    valid position), against the stated ATen rule"""
    g = _gen('maxpool_nan')
    N, H, W, C = 3, 13, 14, 16
    x = _ints((N, H, W, C), -3, 3, g).float()
    x[torch.rand(x.shape, generator=g).to(DEV) < 0.03] = float('nan')
    x[:, 4:9, 3:8] = float('-inf')
    x[1, :, :, :8] = float('-inf')
    x = x.to(bf16)
    y, am = _maxpool_call(x)
    ref, am_ref = _maxpool_ref(x)
    assert bool(ref.isnan().any()) and bool((ref == float('-inf')).any())
    _check_pool_values(y, ref, 'maxpool NaN / -inf')
    assert torch.equal(am, am_ref), 'maxpool NaN / -inf: argmax differs from the scan rule'


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', ['h1w1_c8', 'h5w6_c24', 'h31w30_c8', 'h9w8_c2048', 'stem_c64'])
def test_bn_apply_maxpool(name, tier):
    """maxpool(bf16(act(z*scale+shift))) in one pass: against fp64 and bit for bit against bn_apply + maxpool_fwd"""
    ops = _ops()
    N, H, W, C = maxpool_sweep(_sm_count())[name]
    g = _gen('bn_apply_maxpool', name, tier)
    if tier == 1:
        z = _ints((N, H, W, C), -8, 8, g)
        sc, sh = _pick((C,), [-2, -1, -0.5, 0.5, 1, 2], g), _pick((C,), [-4, -1.5, 0, 0.5, 2, 6], g)
    else:
        z = _randn((N, H, W, C), g, 2.0)
        sc, sh = _randn((C,), g, 1.0, 0.0, f32), _randn((C,), g, 2.0, 1.0, f32)
    for act in ACTS:
        what = '%s bn_apply_maxpool act %d' % (name, act)
        y, am = _twice(lambda: _maxpool_call(z, (sc, sh, act)), what)
        a = ops.bn_apply(z.view(-1, C), sc, sh, act).view(N, H, W, C)
        y2, am2 = _maxpool_call(a)
        assert _same(y, y2) and torch.equal(am, am2), '%s: differs from bn_apply + maxpool_fwd' % what
        pre = z.double() * sc.double() + sh.double()
        if tier == 1:
            _exact_pre([pre], bf16, what)
            ref, am_ref = _maxpool_ref(_act(pre, act).to(bf16))
            _exact(y, ref, what)
            assert torch.equal(am, am_ref), '%s: argmax differs from fp64' % what
        else:
            ref, _ = _maxpool_ref(_act(pre, act))
            bad = (y.double() - ref).abs() > _ulp(ref, 8)
            assert not bool(bad.any()), '%s: %d elements beyond 1 bf16 ulp of fp64' % (what, int(bad.sum()))


AVG_CASES = {'hw1_c8': (3, 1, 1, 8), 'hw49_c2048': (5, 7, 7, 2048), 'hw64_c24': (4, 8, 8, 24),
             'hw3136_c64': (4, 56, 56, 64), 'hw3136_bwd_over_cap': (8, 56, 56, 256)}


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', list(AVG_CASES))
def test_avgpool(name, tier):
    ops = _ops()
    N, H, W, C = AVG_CASES[name]
    HW = H * W
    g = _gen('avgpool', name, tier)
    x = _ints((N, H, W, C), -3, 3, g) if tier == 1 else _randn((N, H, W, C), g, 1.0, 0.5)

    def fwd():
        b, y = _guarded((N, 1, 1, C), bf16)
        ops.avgpool_fwd(x, out=y)
        torch.cuda.synchronize()
        _check_written(b, y, 'avgpool_fwd')
        return (y,)

    y, = _twice(fwd, name)
    inv = float(torch.tensor(1.0 / HW, dtype=f32))
    xd = x.double().view(N, HW, C)
    if tier == 1:
        s = xd.sum(1)
        assert float(xd.abs().sum(1).max()) < 2 ** 24
        _exact(y.view(N, C), (s.float() * inv).double(), '%s avgpool_fwd (fp32 sum times fp32 1/HW)' % name)
        if HW & (HW - 1) == 0:
            _exact(y.view(N, C), s / HW, '%s avgpool_fwd' % name)
    else:
        _bound(y.view(N, C), xd.mean(1), xd.abs().mean(1), 'pool', '%s avgpool_fwd' % name)
    dy = _ints((N, 1, 1, C), -3, 3, g) if tier == 1 else _randn((N, 1, 1, C), g)

    def bwd():
        b, dx = _guarded((N, H, W, C), bf16)
        ops.avgpool_bwd(dy, (N, H, W, C), out=dx)
        torch.cuda.synchronize()
        _check_written(b, dx, 'avgpool_bwd')
        return (dx,)

    dx, = _twice(bwd, name)
    want = (dy.float() * inv).to(bf16).expand(N, H, W, C)      # the fp32 chain: one multiply, one rounding
    assert _same(dx, want.contiguous()), '%s avgpool_bwd differs from bf16(dy * fp32(1/HW))' % name


# ================================================================================================ depthwise
def dw_sweep(sm):
    """name -> (N, H, W, C, R, S, stride, pad_h, pad_w).  3x3 / pad 1 cases run the sliding-window kernels (P in
    {1, 16, 17, 33}, odd / even W and W = 1, C = 8 and 2048, grids over the 16-per-SM cap, wgrad at the 592-block cap
    and on the b3 path); the rest are descriptors dw3_ok rejects (generic kernels)."""
    return {
        's1_p1_w1_c8': (3, 1, 1, 8, 3, 3, 1, 1, 1),
        's1_p16_c8': (2, 16, 15, 8, 3, 3, 1, 1, 1),
        's1_p17_c2048': (2, 17, 6, 2048, 3, 3, 1, 1, 1),
        's1_p33_c24': (2, 33, 9, 24, 3, 3, 1, 1, 1),
        's2_p1_w1_c8': (2, 2, 1, 8, 3, 3, 2, 1, 1),
        's2_p16_c64': (2, 31, 32, 64, 3, 3, 2, 1, 1),
        's2_p17_c2048': (2, 34, 7, 2048, 3, 3, 2, 1, 1),
        's2_p33_c16': (1, 65, 10, 16, 3, 3, 2, 1, 1),
        's1_over_cap': (-(-3 * sm // 2), 1, 64, 256, 3, 3, 1, 1, 1),
        's2_over_cap': (3 * sm, 2, 64, 256, 3, 3, 2, 1, 1),
        's1_wgrad_cap': (40, 4, 32, 2048, 3, 3, 1, 1, 1),
        'g_3x3_pad0': (2, 9, 10, 24, 3, 3, 1, 0, 0),
        'g_3x3_s3': (2, 11, 12, 16, 3, 3, 3, 1, 1),
        'g_1x1': (3, 5, 7, 8, 1, 1, 1, 0, 0),
        'g_2x2': (2, 8, 9, 64, 2, 2, 1, 0, 0),
        'g_1x9': (2, 6, 20, 32, 1, 9, 1, 0, 4),
        'g_1x1_s2_c2048': (2, 5, 6, 2048, 1, 1, 2, 0, 0),
    }


_DW_NAMES = list(dw_sweep(132))


def _dw_geom(cs):
    N, H, W, C, R, S, st, ph, pw = cs
    return (H + 2 * ph - R) // st + 1, (W + 2 * pw - S) // st + 1


def _dw_pad(x, cs, P, Q):
    N, H, W, C, R, S, st, ph, pw = cs
    Hp, Wp = max(H + 2 * ph, (P - 1) * st + R), max(W + 2 * pw, (Q - 1) * st + S)
    xp = torch.zeros((x.shape[0], Hp, Wp, C), dtype=f64, device=x.device)
    xp[:, ph:ph + H, pw:pw + W] = x.double()
    return xp


def _dw_taps(cs, P, Q):
    N, H, W, C, R, S, st, ph, pw = cs
    for r in range(R):
        for s in range(S):
            yield r * S + s, (slice(None), slice(r, r + st * (P - 1) + 1, st), slice(s, s + st * (Q - 1) + 1, st))


def ref_dw_fprop(x, w, cs):
    P, Q = _dw_geom(cs)
    xp = _dw_pad(x, cs, P, Q)
    y = torch.zeros((x.shape[0], P, Q, cs[3]), dtype=f64, device=x.device)
    for t, sl in _dw_taps(cs, P, Q):
        y += xp[sl] * w[t].double()
    return y


def ref_dw_dgrad(dy, w, cs):
    N, H, W, C, R, S, st, ph, pw = cs
    P, Q = _dw_geom(cs)
    dxp = _dw_pad(torch.zeros((N, H, W, C), device=dy.device), cs, P, Q)
    for t, sl in _dw_taps(cs, P, Q):
        dxp[sl] += dy.double() * w[t].double()
    return dxp[:, ph:ph + H, pw:pw + W]


def ref_dw_wgrad(x, dy, cs):
    P, Q = _dw_geom(cs)
    xp = _dw_pad(x, cs, P, Q)
    dw = torch.zeros((cs[4] * cs[5], cs[3]), dtype=f64, device=x.device)
    for t, sl in _dw_taps(cs, P, Q):
        dw[t] = (xp[sl] * dy.double()).sum((0, 1, 2))
    return dw


def _dw_desc(cs):
    N, H, W, C, R, S, st, ph, pw = cs
    return _ops().make_desc(N, H, W, C, C, R, S, st, (ph, pw))


def _dw_calls(cs, x, w, dy, dw0):
    ops = _ops()
    N, H, W, C, R, S = cs[:6]
    P, Q = _dw_geom(cs)
    d = _dw_desc(cs)

    def fprop():
        b, y = _guarded((N, P, Q, C), bf16)
        ops.dwconv_fprop(x, w, d, out=y)
        torch.cuda.synchronize()
        _check_written(b, y, 'dwconv_fprop')
        return (y,)

    def dgrad():
        b, dx = _guarded((N, H, W, C), bf16)
        ops.dwconv_dgrad(dy, w, d, out=dx)
        torch.cuda.synchronize()
        _check_written(b, dx, 'dwconv_dgrad')
        return (dx,)

    def wgrad():
        b, dw = _guarded((R * S, C), f32, 0.0)
        dw.copy_(dw0)
        ws = torch.full((592 * R * S * C,), float('nan'), device=DEV)     # any content is allowed
        ops.dwconv_wgrad(x, dy, d, dw, ws)
        torch.cuda.synchronize()
        _check_written(b, dw, 'dwconv_wgrad')
        return (dw,)

    return _twice(fprop, 'dw fprop')[0], _twice(dgrad, 'dw dgrad')[0], _twice(wgrad, 'dw wgrad')[0]


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', _DW_NAMES)
def test_depthwise(name, tier):
    cs = dw_sweep(_sm_count())[name]
    N, H, W, C, R, S = cs[:6]
    P, Q = _dw_geom(cs)
    g = _gen('dw', name, tier)
    if tier == 1:
        x, w, dy = _ints((N, H, W, C), -2, 2, g), _ints((R * S, C), -2, 2, g), _ints((N, P, Q, C), -2, 2, g)
        dw0 = _ints((R * S, C), -8, 8, g, f32)
    else:
        x, w, dy = _randn((N, H, W, C), g), _randn((R * S, C), g, 1 / 3), _randn((N, P, Q, C), g)
        dw0 = torch.zeros((R * S, C), device=DEV)
    y, dx, dw = _dw_calls(cs, x, w, dy, dw0)
    refs = ((y, ref_dw_fprop(x, w, cs), ref_dw_fprop(x.abs(), w.abs(), cs), 'dw', 'fprop'),
            (dx, ref_dw_dgrad(dy, w, cs), ref_dw_dgrad(dy.abs(), w.abs(), cs), 'dw', 'dgrad'),
            (dw, ref_dw_wgrad(x, dy, cs) + dw0.double(), ref_dw_wgrad(x.abs(), dy.abs(), cs) + dw0.double().abs(),
             'dw_wgrad', 'wgrad'))
    for out, ref, absref, fam, op in refs:
        if tier == 1:
            assert float(absref.max()) < (256 if out.dtype == bf16 else 2 ** 24), 'precondition: %s exact' % op
            _exact(out, ref, '%s dw %s' % (name, op))
        else:
            _bound(out, ref, absref, fam, '%s dw %s' % (name, op))


# ================================================================================================ SE and act_bwd
SE_CASES = {'n3_hw1_c72': (3, 1, 72), 'n5_hw7_c200': (5, 7, 200), 'n4_hw49_c8': (4, 49, 8),
            'n2_hw3136_c64': (2, 3136, 64), 'n300_hw49_c136': (300, 49, 136), 'n16_hw64_c2048': (16, 64, 2048)}


def _sigmoid(l):
    return torch.sigmoid(l.double())


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', list(SE_CASES))
def test_se(name, tier):
    ops = _ops()
    N, HW, C = SE_CASES[name]
    g = _gen('se', name, tier)
    if tier == 1:
        r, gr = _ints((N, HW, 1, C), -3, 3, g), _ints((N, HW, 1, C), -3, 3, g)
    else:
        r, gr = _randn((N, HW, 1, C), g, 1.0, 0.2), _randn((N, HW, 1, C), g)
    logit = (torch.rand((N, C), generator=g) * 40 - 20).to(DEV)
    dmean = _randn((N, 1, 1, C), g)
    inv = float(torch.tensor(1.0 / HW, dtype=f32))

    def call(fn, shape, *args):
        def run():
            b, o = _guarded(shape, bf16)
            fn(*args, out=o)
            torch.cuda.synchronize()
            _check_written(b, o, name)
            return (o,)
        return _twice(run, '%s %s' % (name, fn.__name__))[0]

    pooled = call(ops.se_pool, (N, 1, 1, C), r)
    rd, gd = r.double().view(N, HW, C), gr.double().view(N, HW, C)
    if tier == 1:     # exact integer sums, then the fp32 multiply by fp32(1/HW) and one bf16 rounding
        _exact(pooled.view(N, C), (rd.sum(1).float() * inv).double(), '%s se_pool' % name)
    else:
        _bound(pooled.view(N, C), rd.mean(1), rd.abs().mean(1), 'se', '%s se_pool' % name)
    sg = _sigmoid(logit).view(N, 1, C)
    y = call(ops.se_scale_fwd, (N, HW, 1, C), r, logit)
    _bound(y.view(N, HW, C), rd * sg, rd.abs() * sg, 'se', '%s se_scale_fwd' % name)
    dl = call(ops.se_bwd_reduce, (N, 1, 1, C), gr, r, logit)
    s = (gd * rd).sum(1)
    if tier == 1:
        assert float((gd * rd).abs().sum(1).max()) < 2 ** 24
    sgp = (sg * (1 - sg)).view(N, C)
    # sigma' = sg (1 - sg) cancels for large positive logits exactly as in torch's fp32 autograd: bounded by an
    # absolute term in sum |g r| rather than relative to sigma'
    _bound(dl.view(N, C), s * sgp, (gd * rd).abs().sum(1), 'se', '%s se_bwd_reduce' % name)
    dr = call(ops.se_bwd_dx, (N, HW, 1, C), gr, logit, dmean)
    dmd = dmean.double().view(N, 1, C)
    _bound(dr.view(N, HW, C), gd * sg + dmd / HW, gd.abs() * sg + dmd.abs() / HW, 'se', '%s se_bwd_dx' % name)


@pytest.mark.parametrize('n', [8, 8 * 1001, None])
def test_act_bwd(n):
    """dx = dy where act'(y) passes (ReLU: y > 0, ReLU6: 0 < y < 6, strict as torch's threshold / hardtanh backward),
    else +0; exact for y = +-0, 6, subnormals, +-inf and NaN"""
    ops = _ops()
    if n is None:                                   # grid over its 16-per-SM cap: the grid-stride loop iterates
        n = 8 * 16 * 256 * _sm_count() * 3 // 2
    g = _gen('act_bwd', n)
    special = torch.tensor([0.0, -0.0, 6.0, -6.0, 5.96875, 6.03125, 2.0 ** -130, -2.0 ** -130, 2.0 ** -126,
                            float('nan'), float('inf'), float('-inf'), 1e-30, 3.0], dtype=f32)
    yv = torch.randn(n, generator=g) * 4
    pick = torch.rand(n, generator=g) < 0.3
    yv[pick] = special[torch.randint(0, len(special), (int(pick.sum()),), generator=g)]
    y = yv.to(DEV).to(bf16)
    dy = _randn((n,), g)
    dy[:8] = torch.tensor([-0.0, 0.0, 1e-38, -1.5, 2.0, -3.0, 1.0, 7.0]).to(bf16)
    for act in ACTS:
        def run():
            b, dx = _guarded((n,), bf16)
            ops.act_bwd(dy, y, act, out=dx)
            torch.cuda.synchronize()
            _check_written(b, dx, 'act_bwd')
            return (dx,)
        dx, = _twice(run, 'act_bwd')
        yf = y.float()
        want = torch.where(_act_pass(yf, act), dy, torch.zeros((), dtype=bf16, device=DEV))
        bad = _bits(dx) != _bits(want)
        assert not bool(bad.any()), 'act_bwd act %d: %d elements differ, first at %s (y = %r)' % (
            act, int(bad.sum()), _first_bad(bad), float(y[bad][0]))


# ================================================================================================ loss
CE_CASES = {'b2560_k1000_eps': (2560, 1000, 1000, 0.1), 'b2560_k10_ld16': (2560, 10, 16, 0.0),
            'b37_k257_ld264_eps': (37, 257, 264, 0.1), 'b64_k1000_ld1008': (64, 1000, 1008, 0.0),
            'b1_k10': (1, 10, 10, 0.0)}


def _ce_call(logits, target, classes, eps, mix=None, gs=1.0, gs_dev=None):
    ops = _ops()
    B, ld = logits.shape
    bl, loss = _guarded((3,), f32)
    br, rows = _guarded((2 * B,), f32)
    bd, dl = _guarded((B, ld), bf16)
    if mix is None:
        ops.softmax_ce(logits, target, classes, eps, loss=loss, row_loss=rows, dlogits=dl, grad_scale=gs,
                       grad_scale_dev=gs_dev)
    else:
        ops.softmax_ce_mix(logits, target, mix, classes, loss=loss, row_loss=rows, dlogits=dl, grad_scale=gs,
                           grad_scale_dev=gs_dev)
    torch.cuda.synchronize()
    for b, v, n in ((bl, loss, 'loss'), (br, rows, 'row_loss'), (bd, dl, 'dlogits')):
        _check_written(b, v, 'softmax_ce %s' % n)
    return loss, rows, dl


def _f32(v):
    return float(torch.tensor(v, dtype=f32))


@pytest.mark.parametrize('mixed', [False, True])
@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('name', list(CE_CASES))
def test_softmax_ce(name, tier, mixed):
    """softmax_ce / softmax_ce_mix: per-row loss and every dlogits element in the rounding tier; the top-1 / top-5
    counts follow the 'strictly above the target' rule exactly, tier 1 with integer logits full of ties"""
    B, K, ld, eps = CE_CASES[name]
    if mixed:
        eps = 0.0
    g = _gen('ce', name, tier, mixed)
    logits = torch.zeros(B, ld)
    logits[:, :K] = torch.randint(-3, 4, (B, K), generator=g).float() if tier == 1 else torch.randn(B, K, generator=g) * 3
    logits = logits.to(DEV)
    target = torch.randint(0, K, (B,), generator=g).to(DEV)
    gs_dev = torch.full((1,), 0.5, device=DEV) if tier == 2 else None
    gscale = 4.0 if tier == 2 else 1.0
    mix = None
    lam = 1.0
    if mixed:
        ops = _ops()
        from convnet.pytorch_b200.lib import MIX_MIXUP
        perm = torch.randperm(B, generator=g).to(DEV)
        lam = _f32(0.37)
        params = torch.zeros(5, dtype=torch.int32, device=DEV)
        params[:1].view(f32).fill_(lam)
        mix = ops.Mix(perm, params, MIX_MIXUP)
    loss, rows, dl = _twice(lambda: _ce_call(logits, target, K, eps, mix, gscale, gs_dev), name)
    x = logits[:, :K].double()
    xt = x.gather(1, target.view(-1, 1)).view(-1)
    above = (logits[:, :K] > logits[:, :K].gather(1, target.view(-1, 1))).sum(1).float()
    assert _same(rows[B:], above), '%s: rank counts differ from the strictly-above rule' % name
    t1 = float((above < 0.5).sum())
    t5 = float((above < 4.5).sum())
    assert float(loss[1]) == _f32(_f32(100.0 * t1) / B) and float(loss[2]) == _f32(_f32(100.0 * t5) / B)
    mx = x.max(1).values
    lse = mx + torch.log(torch.exp(x - mx.view(-1, 1)).sum(1))
    sm = torch.exp(x - lse.view(-1, 1))
    onehot = torch.zeros_like(x).scatter_(1, target.view(-1, 1), 1.0)
    if mixed:
        oml = _f32(1.0 - lam)
        t2 = target[mix.perm]
        onehot2 = torch.zeros_like(x).scatter_(1, t2.view(-1, 1), 1.0)
        wsm = _f32(lam + oml)
        q = lam * onehot + oml * onehot2
        row_ref = -(lam * (xt - lse) + oml * (x.gather(1, t2.view(-1, 1)).view(-1) - lse))
        row_abs = lam * (xt.abs() + lse.abs()) + oml * (x.abs().max(1).values + lse.abs())
    else:
        eps_sum = _f32(_f32(eps) / K)
        eps_nll = _f32(_f32(1.0 - eps_sum) - _f32(eps))
        wsm = _f32(eps_nll + _f32(K * eps_sum))
        q = eps_nll * onehot + eps_sum
        row_ref = -(eps_nll * (xt - lse) + eps_sum * (x.sum(1) - K * lse))
        row_abs = eps_nll * (xt.abs() + lse.abs()) + eps_sum * (x.abs().sum(1) + K * lse.abs())
    _bound(rows[:B], row_ref, row_abs, 'ce', '%s row loss' % name)
    _bound(loss[:1], row_ref.mean().view(1), row_abs.mean().view(1), 'ce', '%s mean loss' % name)
    gs = _f32(_f32(gscale * (0.5 if gs_dev is not None else 1.0)) / B)
    ref = (wsm * sm - q) * gs
    absref = (abs(wsm) * sm + q) * abs(gs)
    _bound(dl[:, :K], ref, absref, 'ce', '%s dlogits' % name)
    assert not bool(_bits(dl[:, K:]).ne(0).any()), '%s: padding columns of dlogits are not +0' % name


@pytest.mark.parametrize('B,K', [(2560, 1000), (1, 10), (300, 4097)])
def test_colsum(B, K):
    g = _gen('colsum', B, K)
    m = _ints((B, K), -3, 3, g)
    init = _ints((K,), -100, 100, g, f32)
    b, out = _guarded((K,), f32)
    out.copy_(init)
    _ops().colsum_bf16(m, out)
    torch.cuda.synchronize()
    _check_written(b, out, 'colsum')
    _exact(out, init.double() + m.double().sum(0), 'colsum_bf16 (out +=)')


# ================================================================================================ optimizer
def _fma32(a, b, c):
    """fp32 fma emulated in fp64 (the product of two fp32 values is exact in fp64; one rounding of the sum, then
    one to fp32: within 1 fp32 ulp of the true fma)"""
    return (a.double() * b.double() + c.double()).float()


def _sgd_ref(p, g, m, n, wd_count, lr, momentum, damp, wd, inv_scale, clip, first):
    gs = torch.tensor(inv_scale, dtype=f32) * (clip.cpu() if clip is not None else torch.tensor(1.0))
    gs = gs.to(DEV).float()
    gg = g * gs
    dec = torch.arange(n, device=DEV) < wd_count
    gg = torch.where(dec, _fma32(torch.full_like(p, wd), p, gg), gg)
    step = gg
    m_new = None
    if momentum != 0.0:
        m_new = gg.clone() if first else _fma32(torch.full_like(p, momentum), m, _f32(1.0 - damp) * gg)
        step = m_new
    return _fma32(torch.full_like(p, -lr), step, p), m_new


def _sgd_cases(sm):
    big = sm * 8 * 256 * 4 * 3 + 5                     # grid at its 8-per-SM cap: the grid-stride loop iterates
    return [(1, 1), (3, 2), (4097, 0), (4097, 4097), (4097, 1), (4097, 2), (4097, 3), (4097, 1026), (4097, 2051),
            (4097, 4095), (big, big // 2)]


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('variant', ['momentum', 'dampening', 'no_momentum', 'clip', 'zero_grad'])
def test_fused_sgd(variant, tier):
    """fused_sgd element by element against the restated fp32 chain (unscale, weight decay on [0, wd_count), momentum
    with dampening, step, bf16 shadow): exact on dyadic data (tier 1), within 1 fp32 ulp otherwise"""
    ops = _ops()
    lr, mom, damp, wd, inv_scale = (0.125, 0.5, 0.0, 0.0625, 2.0 ** -7) if tier == 1 else (0.1, 0.9, 0.0, 1e-4,
                                                                                            1 / 128.0)
    if variant == 'dampening':
        damp = 0.25 if tier == 1 else 0.1
    if variant == 'no_momentum':
        mom = 0.0
    for n, wd_count in _sgd_cases(_sm_count()):
        g = _gen('sgd', variant, tier, n, wd_count)
        if tier == 1:
            p = _ints((n,), -64, 64, g, f32) * 0.25
            grads = [_ints((n,), -64, 64, g, f32) for _ in range(3)]
        else:
            p = _randn((n,), g, 1.0, 0.0, f32)
            grads = [_randn((n,), g, 128.0, 0.0, f32) for _ in range(3)]
        clip = torch.full((1,), 0.5 if tier == 1 else 0.37, device=DEV) if variant == 'clip' else None
        bp, p32 = _guarded((n,), f32)
        p32.copy_(p)
        bm, m32 = _guarded((n,), f32, 0.0) if mom != 0.0 else (None, None)
        b16, p16 = _guarded((n,), bf16)
        pr, mr = p.clone(), torch.zeros(n, device=DEV)
        for step, gr in enumerate(grads):
            bg, g32 = _guarded((n,), f32)
            g32.copy_(gr)
            ops.fused_sgd(p32, g32, m32, p16, n, wd_count, lr, mom, damp, wd, inv_scale, clip, step == 0,
                          zero_grad=variant == 'zero_grad')
            torch.cuda.synchronize()
            what = '%s tier %d n=%d wd_count=%d step %d' % (variant, tier, n, wd_count, step)
            pr, mn = _sgd_ref(pr, gr, mr, n, wd_count, lr, mom, damp, wd, inv_scale, clip, step == 0)
            if mn is not None:
                mr = mn
            for b, v, n_ in ((bp, p32, 'p32'), (b16, p16, 'p16')) + (((bm, m32, 'm32'),) if m32 is not None else ()):
                _check_written(b, v, '%s %s' % (what, n_))
            _check_guards(bg, n, '%s g32' % what)
            if variant == 'zero_grad':
                assert not bool(g32.ne(0).any()), '%s: gradient not cleared' % what
            else:
                assert _same(g32, gr), '%s: gradient modified' % what
            if tier == 1:
                _exact(p32, pr.double(), '%s p32' % what)
                if m32 is not None:
                    _exact(m32, mr.double(), '%s m32' % what)
            else:
                _within_ulps(p32, pr.double(), 1, 24, '%s p32' % what)
                if m32 is not None:
                    _within_ulps(m32, mr.double(), 1, 24, '%s m32' % what)
                pr = p32.clone()          # continue from the kernel's state: the 1-ulp slack must not compound
                if m32 is not None:
                    mr = m32.clone()
            assert _same(p16, p32.to(bf16)), '%s: bf16 shadow != bf16(p32)' % what


@pytest.mark.parametrize('tier', [1, 2])
@pytest.mark.parametrize('n', [1, 7, 1024, 3000001])
def test_sumsq_and_grad_coef(n, tier):
    ops = _ops()
    g = _gen('sumsq', n, tier)
    x = _ints((n,), -2, 2, g, f32) if tier == 1 else _randn((n,), g, 64.0, 0.0, f32)
    out = torch.full((8,), float('nan'), device=DEV)
    ws = torch.full((1024,), float('nan'), device=DEV)
    ops.sumsq(x, n, out[0:1], ws)
    s = out[0:1].clone()
    ops.sumsq(x, n, out[0:1], ws)
    assert _same(s, out[0:1])
    ref = (x.double() ** 2).sum().view(1)
    if tier == 1:
        assert float(ref) < 2 ** 24
        _exact(out[0:1], ref, 'sumsq')
    else:
        _bound(out[0:1], ref, ref, 'sumsq', 'sumsq n=%d' % n)
    # grad_coef, both modes, against the restated fp32 chain (sqrtf and the divisions are correctly rounded)
    inv = 1 / 64.0
    ops.grad_coef(out[0:1], inv, 0, 5.0, 0.0, None, out[1:2], out[2:3])
    norm = torch.sqrt(out[0:1]) * inv
    assert _same(out[2:3], norm)
    assert _same(out[1:2], torch.clamp_max(torch.tensor(5.0, device=DEV) / (norm + _f32(1e-6)), 1.0))
    state = torch.zeros(2, device=DEV)
    ops.grad_coef(out[0:1], inv, 1, 0.0, 0.9, state, out[1:2], out[2:3])
    assert float(out[1]) == 1.0 and _same(state[0:1], norm) and float(state[1]) == 1.0
    ops.grad_coef(out[0:1], inv, 1, 0.0, 0.9, state, out[1:2], None)
    run = (_f32(0.9) * norm.double() + _f32(0.1) * norm.double())
    _within_ulps(state[0:1], run, 1, 24, 'grad_coef smoothed norm')
    _within_ulps(out[1:2], (state[0:1] / (norm + _f32(1e-6))).double(), 0, 24, 'grad_coef coefficient')


# ================================================================================================ report / coverage
def test_tier2_calibration_report():
    """Prints the worst observed excess ratio next to each tier-2 coefficient (run after the tier-2 cases, e.g. with
    -s); the coefficients should stay 4-10x above what the H100 shows.  Also prints the invstd error of the shifted-mean
    BatchNorm statistics at 16 and 64 std (the latter an estimate of the one-pass formula's weakness, not a bound)."""
    if not WORST:
        pytest.skip('no tier-2 case ran in this session')
    for fam, (ratio, where) in sorted(WORST.items()):
        c = C_TIER2.get(fam)
        if c is None:
            print('%s: %.3e (%s)' % (fam, ratio, where))
        else:
            print('tier-2 %-9s worst (|y-ref| - rt|ref|)/absref = %.3e (%s), bound c = %.3e (%.1fx)' % (
                fam, ratio, where, c, c / ratio if ratio > 0 else math.inf))


SWEEP_FILES = ('bn.cu', 'pool.cu', 'dwconv.cu', 'se.cu', 'loss.cu', 'optim.cu')


def _kernel_key_mangled(sym):
    """Itanium name of a b200:: kernel -> (name, template arguments) for the int / bool arguments used here"""
    m = re.match(r'_ZN4b200(\d+)', sym)
    if not m:
        return None
    n = int(m.group(1))
    rest = sym[m.end():]
    name, rest = rest[:n], rest[n:]
    t = re.match(r'I((?:L[ib]\d+E)+)E', rest)
    return name, tuple(int(a) for a in re.findall(r'L[ib](\d+)E', t.group(1))) if t else ()


def _kernel_key_demangled(name):
    m = re.search(r'b200::(\w+)(?:<(.*?)>)?\(', name)
    if not m:
        return None
    args = []
    for a in (m.group(2) or '').split(','):
        a = re.sub(r'\((int|bool)\)', '', a).strip()
        if a:
            args.append({'true': 1, 'false': 0}[a] if a in ('true', 'false') else int(a))
    return m.group(1), tuple(args)


def _library_kernels():
    """kernels the six source files compiled into the library: cuobjdump lists every function per source identifier"""
    from convnet.pytorch_b200 import lib
    tool = shutil.which('cuobjdump') or os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
    assert os.path.exists(tool), 'cuobjdump not found (needed to list the kernels of the library)'
    text = subprocess.run([tool, '--dump-resource-usage', lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout
    kernels, src = {}, None
    for line in text.splitlines():
        m = re.match(r'\s*identifier\s*=\s*(\S+)', line)
        if m:
            src = os.path.basename(m.group(1))
            continue
        m = re.match(r'\s*Function\s+(\S+?):?\s*$', line)
        if m and src in SWEEP_FILES:
            key = _kernel_key_mangled(m.group(1))
            assert key is not None, 'unexpected kernel symbol %s' % m.group(1)
            kernels[key] = src
    return kernels


def _run_sweep_once():
    sm = _sm_count()
    for name in bn_sweep(sm):
        test_bn_stats(name, 1)
        test_bn_apply(name, 1)
        test_bn_backward(name, 1)
    for C in (8, 2048):
        test_bn_finalize(C)
        test_bn_eval_coeffs(C)
    for name in maxpool_sweep(sm):
        test_maxpool(name, 1)
    test_bn_apply_maxpool('h5w6_c24', 1)
    for name in AVG_CASES:
        test_avgpool(name, 1)
    for name in dw_sweep(sm):
        test_depthwise(name, 1)
    for name in SE_CASES:
        test_se(name, 1)
    test_act_bwd(8 * 1001)
    for mixed in (False, True):
        test_softmax_ce('b37_k257_ld264_eps', 1, mixed)
    test_colsum(300, 4097)
    test_fused_sgd('momentum', 1)
    test_sumsq_and_grad_coef(3000001, 1)


def test_sweep_coverage():
    """Every kernel of bn.cu, pool.cu, dwconv.cu, se.cu, loss.cu and optim.cu is launched by the sweep (a kernel added
    to these files fails this test until the sweep reaches it)"""
    want = _library_kernels()
    assert len(want) >= 47, 'only %d kernels found in the library for %s' % (len(want), SWEEP_FILES)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run_sweep_once()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert names, 'the profiler recorded no kernel events'
    seen = {_kernel_key_demangled(n) for n in names}
    missing = sorted('%s %s<%s>' % (src, k[0], ', '.join(map(str, k[1]))) for k, src in want.items() if k not in seen)
    print('\nsweep coverage: %d of %d kernels launched' % (len(want) - len(missing), len(want)))
    assert not missing, 'kernels never launched by the sweep: %s' % missing
