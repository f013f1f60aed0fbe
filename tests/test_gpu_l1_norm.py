"""L1 batch normalization on the Hopper kernel path (csrc/bn_l1.cu, ``resnet(bn_norm='L1')``).

Kernel sweep (the two-tier scheme of test_gpu_kernel_sweep.py): C in {8, 16, 24, 64, 1000, 2048} with row counts that
leave tails, every activation x activation source (recomputed from z, y, mask bits) x g_out.
  - Exact tier: small integers z = mu + (v_i - v_pi(i)) with an integer mean mu per channel (a fifth of the elements
    equal mu, so sign(0) = 0 is exercised).  mean, sign_sum, the running buffers and scale are compared bit for bit with
    the kernel's finalisation restated on the exact sums; invstd = s from the same fp64 expression; shift within 1 ulp
    (one fused multiply-add).
  - Rounding tier: realistic data against fp64, |y - ref| <= rt*|ref| + c*absref.
  - Outputs go into NaN-filled views with guard regions; every call is repeated and must be bitwise identical; the BN
    workspace accumulators must stay zero.
The input gradient is checked against fp64 on the kernel's own statistics and sums (which isolates the kernel), and its
masked gradient g must equal bn_bwd_dx's bit for bit for every source.  A coverage test launches every kernel cuobjdump
lists for bn_l1.cu.
Units: plain / residual / downsample-join conv-free units against fp64 autograd of the L1 formula.  Networks: ResNet-20
and ResNet-18 against the bf16 L1 oracle of tests/l1_oracle.py (T2 with the self-sensitivity bounds of
test_gpu_engine.py), CUDA-graph replay bitwise against eager, folded eval against unfolded, and a profiler trace of one
train_step.
"""
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_kernel_sweep import (BN_ACCUM_FLOATS, _guarded, _check_written, _same, _gen,
                                   _kernel_key_mangled, _kernel_key_demangled)
from test_gpu_engine import _pair, _rel, _cos, _global, _setup

pytestmark = pytest.mark.gpu
bf16, f32, f64, u8 = torch.bfloat16, torch.float32, torch.float64, torch.uint8
DEV = 'cuda'
L1_FIX = 1.2533141373155003           # sqrt(pi/2), as bn_l1.cu
EPS = 1e-5
MOMENTUM = 0.1
RT = 2.0 ** -8                        # bf16 output rounding (plus margin)
RT32 = 2.0 ** -23                     # fp32 output rounding (plus margin)
C_STATS = 2.0 ** -18                  # fp32 partial sums of z and |z - mean| (fp64 across blocks)
C_DZ = 2.0 ** -17                     # bf16 dz = A*g + B*sign + C with fp32 coefficients
C_SUMS = 2.0 ** -16                   # fp32 dgamma / dbeta partials of bn_bwd_reduce

# (C, M): row counts leave tails of the 4-row unroll, of the row-quad mask words and of the block split
CASES = {'c8_m1': (8, 1), 'c8_m70001': (8, 70001), 'c16_m333': (16, 333), 'c24_m4099': (24, 4099),
         'c64_m20007': (64, 20007), 'c64_m8': (64, 8), 'c1000_m61': (1000, 61), 'c2048_m517': (2048, 517)}


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def _data(name, tier):
    """z [M, C] bf16 and, for the exact tier, the integer channel means"""
    C, M = CASES[name]
    g = _gen('l1', name, tier)
    if tier == 'exact':
        v = torch.randint(0, 5, (M, C), generator=g)
        perm = torch.argsort(torch.rand(M, C, generator=g), dim=0)
        mu = torch.randint(-3, 4, (C,), generator=g)
        z = (mu + v - torch.gather(v, 0, perm)).to(f32)
        return z.to(DEV).to(bf16), mu.to(f64)
    shift = torch.randn(C, generator=g) * 2
    scale = torch.rand(C, generator=g) * 3 + 0.1
    return (torch.randn(M, C, generator=g) * scale + shift).to(DEV).to(bf16), None


def _affine(C, g, exact):
    if exact:
        gamma = torch.randint(-4, 5, (C,), generator=g).to(f32) / 4
        beta = torch.zeros(C)
    else:
        gamma = torch.rand(C, generator=g) + 0.5
        beta = torch.randn(C, generator=g) * 0.5
    rm, rv = torch.randn(C, generator=g), torch.rand(C, generator=g) + 0.5
    return [t.to(DEV) for t in (gamma, beta, rm, rv)]


def _ws():
    return torch.zeros(_ops().bn_workspace_floats(2048), device=DEV, dtype=f32)


def _stats(z, gamma, beta, rm, rv, ws):
    """one bn_l1_stats call into guarded outputs -> (dict of views, list of (buf, view, name))"""
    C = z.shape[-1]
    outs = {k: _guarded((C,), f32) for k in ('mean', 'invstd', 'sign_sum', 'scale', 'shift')}
    _ops().bn_l1_stats(z, gamma, beta, EPS, MOMENTUM, rm, rv, outs['mean'][1], outs['invstd'][1], outs['sign_sum'][1],
                       outs['scale'][1], outs['shift'][1], ws)
    return {k: v[1] for k, v in outs.items()}, [(b, v, k) for k, (b, v) in outs.items()]


def _f32(x):
    return np.asarray(x, dtype=np.float32)


def _check_tier(got, ref, absref, c, what, rt=RT):
    """|got - ref| <= rt*|ref| + c*absref element-wise (rt: the output's own rounding)"""
    got, ref, absref = got.double().cpu(), ref.double().cpu(), absref.double().cpu()
    bound = rt * ref.abs() + c * absref
    bad = (got - ref).abs() > bound
    assert not bool(bad.any()), '%s: %d elements out of bound, worst excess %.3e' % (
        what, int(bad.sum()), float(((got - ref).abs() - bound).max()))


@pytest.mark.parametrize('tier', ['exact', 'rounding'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_l1_stats(name, tier):
    C, M = CASES[name]
    z, mu_int = _data(name, tier)
    gamma, beta, rm0, rv0 = _affine(C, _gen('l1aff', name, tier), tier == 'exact')
    ws = _ws()
    rm, rv = rm0.clone(), rv0.clone()
    st, bufs = _stats(z, gamma, beta, rm, rv, ws)
    for b, v, k in bufs:
        _check_written(b, v, '%s %s' % (name, k))
    assert bool((ws[:BN_ACCUM_FLOATS] == 0).all()), 'BN workspace accumulators touched'
    # repeat on the same inputs (running buffers restarted): bitwise identical
    rm2, rv2 = rm0.clone(), rv0.clone()
    st2, _ = _stats(z, gamma, beta, rm2, rv2, ws)
    for k in st:
        assert _same(st[k], st2[k]), '%s: %s differs on repeat' % (name, k)
    assert _same(rm, rm2) and _same(rv, rv2)

    zd = z.double().cpu()
    mean = st['mean'].double().cpu()
    if tier == 'exact':
        assert torch.equal(mean, mu_int), '%s: mean not exact' % name
    else:
        _check_tier(mean, zd.mean(0), zd.abs().mean(0), C_STATS, name + ' mean', rt=RT32)
    d = zd - mean                                              # the kernel subtracts its own (fp32) mean
    sgn = torch.sign(d).sum(0)
    assert torch.equal(st['sign_sum'].double().cpu(), sgn), '%s: sign_sum' % name
    lsum = d.abs().sum(0)
    s_ref = (1.0 / (lsum / M * L1_FIX + float(np.float32(EPS)))).float()
    if tier == 'exact':
        assert _same(st['invstd'].cpu(), s_ref), '%s: invstd' % name
    else:
        s64 = 1.0 / (d.abs().mean(0) * L1_FIX + EPS)
        _check_tier(st['invstd'], s64, s64, C_STATS * 8, name + ' invstd', rt=RT32)
    s = st['invstd'].cpu().numpy()
    g_, b_ = gamma.cpu().numpy(), beta.cpu().numpy()
    sc = _f32(g_) * _f32(s)
    assert np.array_equal(st['scale'].cpu().numpy(), sc), '%s: scale' % name
    sh_ref = b_.astype(np.float64) - mean.numpy() * sc.astype(np.float64)
    sh = st['shift'].cpu().numpy()
    assert np.all(np.abs(sh - sh_ref) <= np.spacing(np.abs(sh_ref).astype(np.float32))), '%s: shift' % name
    keep = np.float32(1) - np.float32(MOMENTUM)
    m = np.float32(MOMENTUM)
    rm_ref = _f32(rm0.cpu().numpy()) * m + _f32(mean.numpy()) * keep
    rv_ref = _f32(rv0.cpu().numpy()) * m + _f32(s) * keep
    assert np.array_equal(rm.cpu().numpy(), rm_ref) and np.array_equal(rv.cpu().numpy(), rv_ref), '%s: running' % name


def test_l1_eval_coeffs():
    g = _gen('l1eval')
    for C in (8, 1000, 2048):
        gamma, beta, rm, rv = _affine(C, g, False)
        sb, sc = _guarded((C,), f32)
        hb, sh = _guarded((C,), f32)
        _ops().bn_l1_eval_coeffs(gamma, beta, rm, rv, sc, sh)
        _check_written(sb, sc, 'eval scale')
        _check_written(hb, sh, 'eval shift')
        ref_sc = _f32(gamma.cpu().numpy()) * _f32(rv.cpu().numpy())
        assert np.array_equal(sc.cpu().numpy(), ref_sc)
        ref_sh = beta.cpu().double().numpy() - rm.cpu().double().numpy() * ref_sc.astype(np.float64)
        assert np.all(np.abs(sh.cpu().numpy() - ref_sh) <= np.spacing(np.abs(ref_sh).astype(np.float32)))


def _backward_case(name, tier, act):
    """runs stats, apply and the backward of every source / g_out combination; returns the checks' inputs"""
    ops = _ops()
    C, M = CASES[name]
    z, _ = _data(name, tier)
    g = _gen('l1bwd', name, tier, act)
    gamma, beta, rm, rv = _affine(C, g, tier == 'exact')
    if tier == 'exact':
        dy = torch.randint(-4, 5, (M, C), generator=g).to(f32).to(DEV).to(bf16)
    else:
        dy = torch.randn(M, C, generator=g).to(DEV).to(bf16)
    ws = _ws()
    st, _ = _stats(z, gamma, beta, rm, rv, ws)
    mask = torch.zeros(ops.bn_act_mask_bytes(M, C), device=DEV, dtype=u8)
    y = ops.bn_apply(z, st['scale'], st['shift'], act, act_mask=mask)
    return ops, z, dy, y, mask, gamma, beta, st, ws


@pytest.mark.parametrize('act', [0, 1, 2])
@pytest.mark.parametrize('tier', ['exact', 'rounding'])
@pytest.mark.parametrize('name', sorted(CASES))
def test_l1_backward(name, tier, act):
    C, M = CASES[name]
    ops, z, dy, y, mask, gamma, beta, st, ws = _backward_case(name, tier, act)
    sources = {'z': (None, None)} if act == 0 else {'z': (None, None), 'y': (y, None), 'mask': (y, mask)}
    zd = z.double().cpu()
    mu, s, S = (st[k].double().cpu() for k in ('mean', 'invstd', 'sign_sum'))
    gm = gamma.double().cpu()
    for src, (y_arg, m_arg) in sources.items():
        for want_g in (False, True):
            what = '%s/%s act %d src %s g_out %d' % (name, tier, act, src, want_g)
            sums = torch.full((2 * C,), float('nan'), device=DEV)
            dga, dba = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
            ops.bn_bwd_reduce(dy, y_arg, z, act, st['mean'], st['invstd'], gamma, beta, sums, dga, dba, ws,
                              act_mask=m_arg)
            assert torch.equal(dga, sums[:C]) and torch.equal(dba, sums[C:]), what + ': arena accumulation'
            outs = []
            for rep in range(2):
                dzb, dz = _guarded((M, C), bf16)
                gb, gv = _guarded((M, C), bf16) if want_g else (None, None)
                ops.bn_l1_bwd_dx(dy, y_arg, z, act, st['mean'], st['invstd'], st['sign_sum'], gamma, beta, sums,
                                 dz=dz, g_out=gv, act_mask=m_arg)
                _check_written(dzb, dz, what + ' dz')
                if want_g:
                    _check_written(gb, gv, what + ' g_out')
                outs.append((dz, gv))
            assert _same(outs[0][0], outs[1][0]), what + ': dz differs on repeat'
            g_bn = torch.empty_like(dy)
            ops.bn_bwd_dx(dy, y_arg, z, act, st['mean'], st['invstd'], gamma, beta, sums, g_out=g_bn, act_mask=m_arg)
            if want_g:
                assert _same(outs[0][1], outs[1][1]), what + ': g_out differs on repeat'
                assert _same(outs[0][1], g_bn), what + ': masked gradient differs from bn_bwd_dx'
            assert bool((ws[:BN_ACCUM_FLOATS] == 0).all()), what + ': BN workspace accumulators touched'
            gd = g_bn.double().cpu()
            # sums against fp64 (bn_bwd_reduce with invstd = s)
            t = gd * (zd - mu) * s
            _check_tier(sums[:C], t.sum(0), t.abs().sum(0), C_SUMS, what + ' dgamma', rt=RT32)
            _check_tier(sums[C:], gd.sum(0), gd.abs().sum(0), C_SUMS, what + ' dbeta', rt=RT32)
            # dz against fp64 on the kernel's statistics and sums
            dg, db = sums[:C].double().cpu(), sums[C:].double().cpu()
            A = gm * s
            B = -A * L1_FIX * dg / M
            Cc = -A * db / M - B * S / M
            ref = A * gd + B * torch.sign(zd - mu) + Cc
            absref = (A * gd).abs() + B.abs() + Cc.abs()
            _check_tier(outs[0][0], ref, absref, C_DZ, what + ' dz')


def test_l1_coverage():
    """every kernel of bn_l1.cu is launched by the sweep"""
    from convnet.pytorch_b200 import lib
    tool = shutil.which('cuobjdump') or os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
    text = subprocess.run([tool, '--dump-resource-usage', lib.LIB_PATH], check=True, capture_output=True,
                          text=True).stdout
    want, src = set(), None
    for line in text.splitlines():
        m = re.match(r'\s*identifier\s*=\s*(\S+)', line)
        if m:
            src = os.path.basename(m.group(1))
            continue
        m = re.match(r'\s*Function\s+(\S+?):?\s*$', line)
        if m and src == 'bn_l1.cu':
            want.add(_kernel_key_mangled(m.group(1)))
    assert len(want) >= 11, 'only %d kernels found for bn_l1.cu' % len(want)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name in ('c64_m20007', 'c2048_m517'):
            test_l1_backward(name, 'rounding', 1)
        test_l1_eval_coeffs()
        torch.cuda.synchronize()
    seen = {_kernel_key_demangled(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    missing = sorted('%s<%s>' % (k[0], ', '.join(map(str, k[1]))) for k in want if k not in seen)
    print('\nbn_l1.cu coverage: %d of %d kernels launched' % (len(want) - len(missing), len(want)))
    assert not missing, 'kernels never launched: %s' % missing


# ---------------------------------------------------------------------------------------------- conv-free units
def _l1_ref(z, gamma, beta):
    mean = z.mean(0)
    s = 1.0 / ((z - mean).abs().mean(0) * L1_FIX + EPS)
    return (z - mean) * s * gamma + beta


@pytest.mark.parametrize('kind', ['plain', 'residual', 'join'])
def test_l1_unit_teacher_forced(kind):
    """one BN unit the way the engine runs it (plain: ReLU recomputed from z; residual: y = relu(L1(z) + r), mask bits,
    g for the skip; join: y = relu(L1a(z) + L1b(z2)), the downsample branch's backward fed g) against fp64 autograd of
    the L1 formula on the same bf16 inputs"""
    ops = _ops()
    g = _gen('l1unit', kind)
    M, C = 4 * 28 * 28, 128
    z = (torch.randn(M, C, generator=g) * 1.5 + 0.3).to(DEV).to(bf16)
    z2 = (torch.randn(M, C, generator=g) * 0.7 - 0.2).to(DEV).to(bf16)
    r = torch.randn(M, C, generator=g).to(DEV).to(bf16)
    dy = torch.randn(M, C, generator=g).to(DEV).to(bf16)
    ga, ba, gb, bb = (torch.rand(C, generator=g) + 0.5).to(DEV), (torch.randn(C, generator=g) * 0.3).to(DEV), \
        (torch.rand(C, generator=g) + 0.5).to(DEV), (torch.randn(C, generator=g) * 0.3).to(DEV)
    ws = _ws()
    zero = torch.zeros(C, device=DEV)
    sa, _ = _stats(z, ga, ba, zero.clone(), zero.clone(), ws)
    sb, _ = _stats(z2, gb, bb, zero.clone(), zero.clone(), ws)
    mask = torch.empty(ops.bn_act_mask_bytes(M, C), device=DEV, dtype=u8)
    grads = {k: torch.zeros(C, device=DEV) for k in ('dga', 'dba', 'dgb', 'dbb')}
    sums_a, sums_b = torch.empty(2 * C, device=DEV), torch.empty(2 * C, device=DEV)
    if kind == 'plain':
        y = ops.bn_apply(z, sa['scale'], sa['shift'], 1)
        ops.bn_bwd_reduce(dy, None, z, 1, sa['mean'], sa['invstd'], ga, ba, sums_a, grads['dga'], grads['dba'], ws)
        dz = ops.bn_l1_bwd_dx(dy, None, z, 1, sa['mean'], sa['invstd'], sa['sign_sum'], ga, ba, sums_a)
    else:
        if kind == 'residual':
            y = ops.bn_apply(z, sa['scale'], sa['shift'], 1, residual=r, act_mask=mask)
        else:
            y = ops.bn_apply(z, sa['scale'], sa['shift'], 1, z2=z2, scale2=sb['scale'], shift2=sb['shift'], act_mask=mask)
        ops.bn_bwd_reduce(dy, y, z, 1, sa['mean'], sa['invstd'], ga, ba, sums_a, grads['dga'], grads['dba'], ws,
                          act_mask=mask)
        gk = torch.empty_like(dy)
        dz = ops.bn_l1_bwd_dx(dy, y, z, 1, sa['mean'], sa['invstd'], sa['sign_sum'], ga, ba, sums_a, g_out=gk,
                              act_mask=mask)
        if kind == 'join':
            ops.bn_bwd_reduce(gk, None, z2, 0, sb['mean'], sb['invstd'], gb, bb, sums_b, grads['dgb'], grads['dbb'], ws)
            dz2 = ops.bn_l1_bwd_dx(gk, None, z2, 0, sb['mean'], sb['invstd'], sb['sign_sum'], gb, bb, sums_b)
    torch.cuda.synchronize()
    # fp64 autograd of the formula
    leaf = {k: v.double().cpu().requires_grad_(True) for k, v in (('z', z), ('z2', z2), ('ga', ga), ('ba', ba),
                                                                  ('gb', gb), ('bb', bb))}
    pre = _l1_ref(leaf['z'], leaf['ga'], leaf['ba'])
    if kind == 'residual':
        pre = pre + r.double().cpu()
    elif kind == 'join':
        pre = pre + _l1_ref(leaf['z2'], leaf['gb'], leaf['bb'])
    yr = F.relu(pre)
    yr.backward(dy.double().cpu())
    assert _rel(y.double().cpu(), yr.detach()) < 4e-3, '%s: y' % kind
    assert _rel(dz.double().cpu(), leaf['z'].grad) < 5e-3, '%s: dz %.3e' % (kind, _rel(dz.double().cpu(),
                                                                                       leaf['z'].grad))
    assert _rel(grads['dga'].double().cpu(), leaf['ga'].grad) < 1e-3, '%s: dgamma' % kind
    assert _rel(grads['dba'].double().cpu(), leaf['ba'].grad) < 1e-3, '%s: dbeta' % kind
    if kind == 'residual':
        g_ref = dy.double().cpu() * (pre > 0).double()
        assert _rel(gk.double().cpu(), g_ref.detach()) < 1e-3, 'residual: skip gradient'
    if kind == 'join':
        assert _rel(dz2.double().cpu(), leaf['z2'].grad) < 5e-3, 'join: dz2 %.3e' % _rel(dz2.double().cpu(),
                                                                                        leaf['z2'].grad)
        assert _rel(grads['dgb'].double().cpu(), leaf['gb'].grad) < 1e-3, 'join: dgamma2'
        assert _rel(grads['dbb'].double().cpu(), leaf['bb'].grad) < 1e-3, 'join: dbeta2'


# ---------------------------------------------------------------------------------------------- networks
def _check_against_l1_oracle(mine, ref, x, y, logit_tol=1e-3, grad_tol=1e-2, cos_min=0.999):
    """T2 of test_gpu_engine._check_against_bf16_oracle, against the L1 oracle (tests/l1_oracle.py, the bf16 storage
    points of oracle.ref_model): logits / loss / every gradient / running buffers, each bound max(survey bound,
    1.5 x the oracle's self-sensitivity to nudging 0.1 % of the input pixels by one bf16 ulp)"""
    import l1_oracle
    assert x.shape[0] >= 32
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    mine.train()
    mine._b200.arena.zero_grad()
    lo = mine(x)
    loss = F.cross_entropy(lo, y)
    loss.backward()
    torch.cuda.synchronize()
    names = [n for n, _ in mine.named_parameters()]
    xc, yc = x.cpu(), y.cpu()
    o_logits, o_loss, o_grads, o_bufs = l1_oracle.loss_and_grads(sd, xc, yc, quant=True)
    gq = torch.Generator().manual_seed(99)
    xb = xc.to(torch.bfloat16)
    nudge = torch.rand(xc.shape, generator=gq) < 1e-3
    xp = torch.where(nudge, (xb.float() * (1 + 2 ** -8)).to(torch.bfloat16), xb).float()
    p_logits, _, p_grads, _ = l1_oracle.loss_and_grads(sd, xp, yc, quant=True)
    gm = _global({n: p.grad for n, p in mine.named_parameters()}, names)
    go, gp = _global(o_grads, names), _global(p_grads, names)
    per = sorted((_cos(p.grad.cpu(), o_grads[n]), n) for n, p in mine.named_parameters() if float(o_grads[n].norm()) > 0)
    self_worst = min(_cos(p_grads[n], o_grads[n]) for n in names if float(o_grads[n].norm()) > 0)
    s_log, s_grad = _rel(p_logits, o_logits), _rel(gp, go)
    print('T2 logits rel %.3e  dloss %.3e  grad rel %.3e  worst tensors %s | oracle self-sensitivity: logits %.3e '
          'grad rel %.3e worst tensor cos %.5f' % (_rel(lo.cpu(), o_logits), abs(float(loss) - float(o_loss)),
                                                   _rel(gm, go), per[:3], s_log, s_grad, self_worst))
    assert _rel(lo.cpu(), o_logits) < max(logit_tol, 1.5 * s_log), 'logits vs bf16 oracle %.3e' % _rel(lo.cpu(), o_logits)
    assert abs(float(loss) - float(o_loss)) < 5e-3
    assert _rel(gm, go) < max(grad_tol, 1.5 * s_grad), 'global grad rel vs bf16 oracle %.3e (self %.3e)' % (
        _rel(gm, go), s_grad)
    assert 1.0 - per[0][0] < max(1.0 - cos_min, 1.5 * (1.0 - self_worst)), 'grad cos of %s vs bf16 oracle = %.5f' % (
        per[0][1], per[0][0])
    for n, b in mine.named_buffers():
        if 'running' in n:
            assert _rel(b.cpu(), o_bufs[n]) < 1e-3, n


def test_resnet20_l1_against_bf16_oracle():
    """per-tensor cos floor 0.997 instead of 0.999: the self-sensitivity below is measured with one nudge seed, and on
    this network the oracle's own worst tensor (a 64-entry BN bias of layer2) moves between cos 0.9979 and 0.9992 from
    one nudge seed to the next -- with the variance BN as well (measured on the CPU oracle, seeds 99-101)"""
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20, bn_norm='L1'), (3, 64, 64), 10, batch=32)
    _check_against_l1_oracle(mine, ref, x, y, cos_min=0.997)


def test_resnet18_l1_against_bf16_oracle():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=18, bn_norm='L1'), (3, 96, 96), 1000, batch=32)
    _check_against_l1_oracle(mine, ref, x, y)


def test_resnet18_l1_graph_replay_bitwise():
    """Trainer.train with captured graphs (two eager steps, then replays) against graphs disabled: parameters, running
    buffers and losses bit for bit after 6 steps"""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    _setup()
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(16, 3, 64, 64, generator=g), torch.randint(0, 1000, (16,), generator=g))
               for _ in range(6)]
    results = []
    for use_graphs in (False, True):
        torch.manual_seed(123)
        model = resnet(dataset='imagenet', depth=18, bn_norm='L1')
        convert_b200(model, 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9)
        tr.use_graphs = use_graphs
        res = tr.train(batches)
        assert (tr.graph_replays > 0) == use_graphs
        if use_graphs:
            assert tr.graph_replays == len(batches) - 2
        results.append((res, {k: v.detach().clone() for k, v in model.state_dict().items()}))
    (r0, s0), (r1, s1) = results
    assert r0['loss'] == r1['loss'], (r0['loss'], r1['loss'])
    diff = [k for k in s0 if not torch.equal(s0[k], s1[k])]
    assert not diff, 'graph replay differs from eager in %s' % diff[:5]
    assert float(s1['bn1.running_var'].abs().sum()) > 0


def test_resnet18_l1_folded_eval():
    """inference with the L1 BN folded into the convolution (w * gamma*running_var, beta - running_mean*gamma*
    running_var) against the unfolded kernels and torch eval"""
    from convnet.pytorch_b200 import engine
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=18, bn_norm='L1'), (3, 64, 64), 1000, steps=3,
                            batch=8)
    saved = engine.FOLD_BN_EVAL
    try:
        ref.eval(); mine.eval()
        with torch.no_grad():
            engine.FOLD_BN_EVAL = False
            a0 = mine(x)
            engine.FOLD_BN_EVAL = True
            a1 = mine(x)
            b = ref(x.to(torch.bfloat16).float())
        assert _rel(a1, a0) < 2e-2, 'folded vs unfolded %.3e' % _rel(a1, a0)
        assert _rel(a0, b) < 3e-2, 'unfolded vs torch eval %.3e' % _rel(a0, b)
        assert _rel(a1, b) < 3e-2, 'folded vs torch eval %.3e' % _rel(a1, b)
    finally:
        engine.FOLD_BN_EVAL = saved


def test_l1_train_step_runs_only_library_kernels():
    """a profiler trace of one L1 train_step: every GPU kernel is the library's, apart from memsets and the zero fill
    of the stem's weight-gradient scratch (torch.zeros)"""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    _setup()
    torch.manual_seed(123)
    model = convert_b200(resnet(dataset='imagenet', depth=18, bn_norm='L1'), 'cuda')
    model.train()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 64, 64, generator=g).cuda()
    y = torch.randint(0, 1000, (16,), generator=g).cuda()
    rt = model._b200
    rt.train_step(x, y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rt.train_step(x, y)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    lib_k = [n for n in names if 'b200::' in n]
    other = sorted({n for n in names if 'b200::' not in n and 'memset' not in n.lower() and 'FillFunctor' not in n})
    print('\nL1 train_step: %d library kernels, other GPU work: %s' % (len(lib_k), sorted(set(names) - set(lib_k))))
    assert any('bn_l1_partial_kernel' in n for n in lib_k) and any('bn_l1_bwd_dx_kernel' in n for n in lib_k)
    assert not other, 'kernels outside the library: %s' % other
