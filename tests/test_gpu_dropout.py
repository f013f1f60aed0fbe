"""In-block dropout on the Hopper kernel path (csrc/dropout.cu, ``resnet(dropout=p)`` on CIFAR BasicBlocks).

Kernels, C in {8, 16, 24, 64, 160, 320, 640, 1024, 2048} with row counts that leave tails of the 2-row unroll, the
row-quad mask words and the block split (the larger M from the SM count, as the kernel sweep):
  - apply: outputs go into NaN-filled views with guard regions and repeated calls must be bitwise equal; the mask bits
    equal the numpy Philox of tests/dropout_oracle.py and (pre > 0) bit for bit, y equals the fp32 restatement
    bf16(fma(z, scale, shift) * c) bit for bit, the mask's padding rows stay untouched; the keep rate is within 5 sigma
    of T/65536 and other keys / layers give other masks.
  - backward: exact tier (integer data, c = 2: the sums are exact), rounding tier against fp64 on the kernel's
    statistics and against fp64 autograd of dropout(relu(bn(z))) with the same mask, and with an all-ones mask and
    c = 1 bit for bit bn_bwd_reduce / bn_bwd_dx.  A coverage test launches every kernel cuobjdump lists for dropout.cu.
Networks: WRN-16-4 and ResNet-20 with p = 0.3 against the bf16 dropout oracle (masks regenerated from the key read back
from the runtime; the T2 bounds of test_gpu_l1_norm.py), CUDA-graph replay bitwise against eager, MixUp and device
augmentation, the launch list of one train_step, and a dropout=0 model's launch list against the plain model's.
"""
import collections
import copy
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dropout_oracle
from test_gpu_kernel_sweep import (BN_ACCUM_FLOATS, BYTE_SENTINEL, GUARD, _guarded, _check_written, _same, _gen,
                                   _sm_count, _kernel_key_mangled, _kernel_key_demangled)
from test_gpu_engine import _pair, _rel, _cos, _global, _setup

pytestmark = pytest.mark.gpu
bf16, f32, f64, u8 = torch.bfloat16, torch.float32, torch.float64, torch.uint8
DEV = 'cuda'
CS = (8, 16, 24, 64, 160, 320, 640, 1024, 2048)
PS = (0.1, 0.3, 0.5, 0.9)
RT32 = 2.0 ** -23
C_SUMS = 2.0 ** -16                   # fp32 dgamma / dbeta partials
C_DZ = 2.0 ** -17                     # bf16 dz with fp32 coefficients
PAD = 0x5A                            # initial content of the mask view (its padding rows must keep it)


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def _ms(C):
    """row counts: below one row iteration, a tail of every unroll, and ~8 blocks per SM of the apply grid"""
    rpi = 256 // (C // 8)
    return {'small': 7, 'mid': 37 * rpi + 5, 'large': (_sm_count() * 8 * 16 * rpi // 2) | 3}


CASES = ['c%d_%s' % (C, k) for C in CS for k in ('small', 'mid', 'large')]


def _case(name):
    c, k = name.split('_')
    C = int(c[1:])
    return C, _ms(C)[k]


def _key(g):
    return torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), generator=g, dtype=torch.int64)


def _unpack_mask(mask, M, C):
    """row-quad mask bytes -> bool [M, C]"""
    cv = C // 8
    Mp = (M + 7) // 8 * 8
    b = mask[:Mp * cv].view(Mp // 4, cv, 4).permute(0, 2, 1).reshape(Mp, cv).cpu().numpy()
    return np.unpackbits(b[:, :, None], axis=2, bitorder='little').reshape(Mp, C)[:M].astype(bool)


def _apply_inputs(C, M, g, positive=False):
    z = (torch.randn(M, C, generator=g) * 2 + 0.3).to(bf16)
    # bf16-valued coefficients: z*scale + shift is exact in fp64, so its fp32 rounding restates the kernel's fma
    scale = (torch.rand(C, generator=g) * 3 + 0.1).to(bf16).float()
    shift = (torch.randn(C, generator=g) * 2 + (20.0 if positive else 0.0)).to(bf16).float()
    return z.to(DEV), scale.to(DEV), shift.to(DEV)


def _apply(z, scale, shift, key, layer, p):
    M, C = z.shape
    nb = _ops().bn_act_mask_bytes(M, C)
    yb, y = _guarded((M, C), bf16)
    mb, mask = _guarded((nb,), u8, fill=PAD)
    _ops().bn_apply_dropout(z, scale, shift, key.to(DEV), layer, p, mask, out=y)
    return yb, y, mb, mask


@pytest.mark.parametrize('p', PS)
@pytest.mark.parametrize('name', CASES)
def test_apply(name, p):
    C, M = _case(name)
    g = _gen('dropout_apply', name, p)
    z, scale, shift = _apply_inputs(C, M, g)
    key, layer = _key(g), int(torch.randint(0, 40, (1,), generator=g))
    yb, y, mb, mask = _apply(z, scale, shift, key, layer, p)
    _check_written(yb, y, name + ' y')
    nb = mask.numel()
    sent = torch.full((GUARD,), BYTE_SENTINEL, dtype=u8, device=DEV)
    assert _same(mb[:GUARD], sent) and _same(mb[GUARD + nb:], sent), name + ': mask guard overwritten'
    cv = C // 8
    rows = np.arange((M + 7) // 8 * 8)
    pad_idx = [((r >> 2) * cv + v) * 4 + (r & 3) for r in rows[M:] for v in range(cv)]
    if pad_idx:
        assert bool((mask[torch.tensor(pad_idx, device=DEV)] == PAD).all()), name + ': mask padding rows written'
    _, y2, _, mask2 = _apply(z, scale, shift, key, layer, p)
    assert _same(y, y2) and _same(mask, mask2), name + ': not repeatable'
    # restatement
    T, c = dropout_oracle.threshold(p)
    keep = dropout_oracle.keep_mask(int(key), layer, M, C, T)
    pre = (z.double().cpu() * scale.double().cpu() + shift.double().cpu()).float()
    bit = keep & (pre > 0).numpy()
    got = _unpack_mask(mask, M, C)
    assert np.array_equal(got, bit), '%s: %d mask bits differ' % (name, int((got != bit).sum()))
    ref = torch.where(torch.from_numpy(bit), pre * torch.tensor(c, dtype=f32), torch.zeros(()))
    assert _same(y.cpu(), ref.to(bf16)), name + ': y differs from bf16(fma(z, scale, shift) * c)'


@pytest.mark.parametrize('p', PS)
def test_keep_rate_keys_and_layers(p):
    C, M = 64, 100003
    g = _gen('dropout_rate', p)
    z, scale, shift = _apply_inputs(C, M, g, positive=True)     # pre > 0 everywhere: the mask is the keep draw
    key = _key(g)
    masks = {}
    for k, layer in ((key, 0), (key, 1), (key + 1, 0)):
        _, _, _, mask = _apply(z, scale, shift, k, layer, p)
        masks[(int(k), layer)] = _unpack_mask(mask, M, C)
    T, _ = dropout_oracle.threshold(p)
    q, n = T / 65536.0, M * C
    a = masks[(int(key), 0)]
    assert abs(a.sum() - n * q) <= 5 * np.sqrt(n * q * (1 - q)), 'keep rate %.6f vs %.6f' % (a.mean(), q)
    for other in ((int(key), 1), (int(key) + 1, 0)):
        b = masks[other]
        same = float((a == b).mean())
        assert abs(same - (q * q + (1 - q) * (1 - q))) < 0.01, 'masks of %s not independent: agreement %.4f' % (other, same)


def _bwd_case(name, tier, p):
    ops = _ops()
    C, M = _case(name)
    g = _gen('dropout_bwd', name, tier, p)
    if tier == 'exact':
        z = torch.randint(-3, 4, (M, C), generator=g).to(f32)
        dy = torch.randint(-4, 5, (M, C), generator=g).to(f32)
        mean = torch.randint(-2, 3, (C,), generator=g).to(f32)
        invstd = torch.ones(C)
        gamma = torch.randint(-4, 5, (C,), generator=g).to(f32) / 4
    else:
        z = torch.randn(M, C, generator=g) * 1.5 + 0.2
        dy = torch.randn(M, C, generator=g)
        mean = z.mean(0) + torch.randn(C, generator=g) * 0.01
        invstd = 1.0 / (z.std(0) + 0.1)
        gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g) * 0.3
    z, dy = z.to(bf16).to(DEV), dy.to(bf16).to(DEV)
    mean, invstd, gamma, beta = (t.to(DEV) for t in (mean, invstd, gamma, beta))
    scale = gamma * invstd
    shift = beta - mean * scale
    key = _key(g)
    mask = torch.empty(ops.bn_act_mask_bytes(M, C), device=DEV, dtype=u8)
    ops.bn_apply_dropout(z, scale, shift, key.to(DEV), 3, p, mask)
    return ops, C, M, z, dy, mean, invstd, gamma, beta, mask


# exact tier on the mid row counts only: there every fp32 partial sum of the integer data stays below 2^24
@pytest.mark.parametrize('name,tier', [('c%d_mid' % C, 'exact') for C in CS] +
                         [('c%d_%s' % (C, k), 'rounding') for C in CS for k in ('mid', 'large')])
def test_backward(name, tier):
    p = 0.5 if tier == 'exact' else 0.3
    ops, C, M, z, dy, mean, invstd, gamma, beta, mask = _bwd_case(name, tier, p)
    ws = torch.zeros(ops.bn_workspace_floats(2048), device=DEV, dtype=f32)
    _, c = dropout_oracle.threshold(p)
    outs = []
    for rep in range(2):
        sums = torch.full((2 * C,), float('nan'), device=DEV)
        dga, dba = torch.ones(C, device=DEV), torch.ones(C, device=DEV)
        ops.bn_bwd_reduce_dropout(dy, z, mask, p, mean, invstd, sums, dga, dba, ws)
        assert torch.equal(dga, sums[:C] + 1) and torch.equal(dba, sums[C:] + 1), name + ': arena accumulation'
        dzb, dz = _guarded((M, C), bf16)
        ops.bn_bwd_dx_dropout(dy, z, mask, p, mean, invstd, gamma, sums, dz=dz)
        _check_written(dzb, dz, name + ' dz')
        outs.append((sums, dz))
    assert _same(outs[0][0], outs[1][0]) and _same(outs[0][1], outs[1][1]), name + ': not repeatable'
    assert bool((ws[:BN_ACCUM_FLOATS] == 0).all()), name + ': BN workspace accumulators touched'
    sums, dz = outs[0]
    bit = torch.from_numpy(_unpack_mask(mask, M, C)).double()
    gd = dy.double().cpu() * bit * c
    xhat = (z.double().cpu() - mean.double().cpu()) * invstd.double().cpu()
    t = gd * xhat
    if tier == 'exact':
        assert torch.equal(sums.double().cpu(), torch.cat([t.sum(0), gd.sum(0)])), name + ': sums not exact'
    else:
        from test_gpu_l1_norm import _check_tier
        _check_tier(sums[:C], t.sum(0), t.abs().sum(0), C_SUMS, name + ' dgamma', rt=RT32)
        _check_tier(sums[C:], gd.sum(0), gd.abs().sum(0), C_SUMS, name + ' dbeta', rt=RT32)
    from test_gpu_l1_norm import _check_tier
    dg, db = sums[:C].double().cpu(), sums[C:].double().cpu()
    A = gamma.double().cpu() * invstd.double().cpu()
    ref = A * (gd - db / M - xhat * dg / M)
    absref = (A * gd).abs() + (A * db / M).abs() + (A * xhat * dg / M).abs()
    _check_tier(dz, ref, absref, C_DZ, name + ' dz', rt=2.0 ** -8)


@pytest.mark.parametrize('C', CS)
def test_backward_against_autograd(C):
    """dz, dgamma, dbeta of the dropout unit against fp64 autograd of dropout(relu(bn(z))) with the kernel's mask"""
    ops = _ops()
    M = 4 * 16 * 16 if C <= 640 else 2 * 8 * 8 * 5
    g = _gen('dropout_autograd', C)
    z = (torch.randn(M, C, generator=g) * 1.5 + 0.3).to(bf16).to(DEV)
    dy = torch.randn(M, C, generator=g).to(bf16).to(DEV)
    gamma, beta = (torch.rand(C, generator=g) + 0.5).to(DEV), (torch.randn(C, generator=g) * 0.3).to(DEV)
    ws = torch.zeros(ops.bn_workspace_floats(2048), device=DEV, dtype=f32)
    coef = torch.empty(6 * C, device=DEV)
    mean, invstd, scale, shift = coef[:C], coef[C:2 * C], coef[2 * C:3 * C], coef[3 * C:4 * C]
    ops.bn_stats(z, gamma, beta, 1e-5, 0.1, None, None, None, mean, invstd, scale, shift, ws)
    key = _key(g).to(DEV)
    mask = torch.empty(ops.bn_act_mask_bytes(M, C), device=DEV, dtype=u8)
    y = ops.bn_apply_dropout(z, scale, shift, key, 5, 0.3, mask)
    sums = torch.empty(2 * C, device=DEV)
    dga, dba = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    ops.bn_bwd_reduce_dropout(dy, z, mask, 0.3, mean, invstd, sums, dga, dba, ws)
    dz = ops.bn_bwd_dx_dropout(dy, z, mask, 0.3, mean, invstd, gamma, sums)
    keep = torch.from_numpy(dropout_oracle.keep_mask(int(key), 5, M, C, dropout_oracle.threshold(0.3)[0])).double()
    leaf = {k: v.double().cpu().requires_grad_(True) for k, v in (('z', z), ('ga', gamma), ('ba', beta))}
    zz = leaf['z']
    mu, var = zz.mean(0), zz.var(0, unbiased=False)
    pre = (zz - mu) / torch.sqrt(var + 1e-5) * leaf['ga'] + leaf['ba']
    out = F.relu(pre) * keep / 0.7
    out.backward(dy.double().cpu())
    assert _rel(y.double().cpu(), out.detach()) < 4e-3, 'y'
    assert _rel(dz.double().cpu(), zz.grad) < 5e-3, 'dz %.3e' % _rel(dz.double().cpu(), zz.grad)
    assert _rel(dga.double().cpu(), leaf['ga'].grad) < 1e-3, 'dgamma'
    assert _rel(dba.double().cpu(), leaf['ba'].grad) < 1e-3, 'dbeta'


@pytest.mark.parametrize('C', CS)
def test_all_ones_mask_equals_bn_backward(C):
    """p = 0 (T = 65536, c = 1) on an all-ones mask: bit for bit bn_bwd_reduce / bn_bwd_dx with that mask"""
    ops, _, M, z, dy, mean, invstd, gamma, beta, _ = _bwd_case('c%d_mid' % C, 'rounding', 0.3)
    ones = torch.full((ops.bn_act_mask_bytes(M, C),), 0xFF, device=DEV, dtype=u8)
    ws = torch.zeros(ops.bn_workspace_floats(2048), device=DEV, dtype=f32)
    s1, s2 = torch.empty(2 * C, device=DEV), torch.empty(2 * C, device=DEV)
    ops.bn_bwd_reduce_dropout(dy, z, ones, 0.0, mean, invstd, s1, None, None, ws)
    y = torch.empty_like(z)
    ops.bn_bwd_reduce(dy, y, z, 1, mean, invstd, gamma, beta, s2, None, None, ws, act_mask=ones)
    assert _same(s1, s2), 'sums differ from bn_bwd_reduce'
    d1 = ops.bn_bwd_dx_dropout(dy, z, ones, 0.0, mean, invstd, gamma, s2)
    d2 = ops.bn_bwd_dx(dy, y, z, 1, mean, invstd, gamma, beta, s2, act_mask=ones)
    assert _same(d1, d2), 'dz differs from bn_bwd_dx'


def test_dropout_coverage():
    """every kernel of dropout.cu is launched by the tests above"""
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
        if m and src == 'dropout.cu':
            want.add(_kernel_key_mangled(m.group(1)))
    assert len(want) >= 5, 'only %d kernels found for dropout.cu' % len(want)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for C in (64, 2048):
            test_backward('c%d_mid' % C, 'rounding')
        torch.cuda.synchronize()
    seen = {_kernel_key_demangled(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    missing = sorted('%s<%s>' % (k[0], ', '.join(map(str, k[1]))) for k in want if k not in seen)
    print('\ndropout.cu coverage: %d of %d kernels launched' % (len(want) - len(missing), len(want)))
    assert not missing, 'kernels never launched: %s' % missing


# ---------------------------------------------------------------------------------------------- networks
WRN = dict(dataset='cifar10', depth=16, width=[64, 128, 256], dropout=0.3)
R20 = dict(dataset='cifar10', depth=20, dropout=0.3)


def _check_against_dropout_oracle(mine, ref, x, y, logit_tol=1e-3, grad_tol=1e-2, cos_min=0.999):
    """T2 of test_gpu_l1_norm._check_against_l1_oracle against the dropout oracle, whose masks are regenerated from the
    key the runtime drew for this step"""
    assert x.shape[0] >= 32
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    mine.train()
    mine._b200.arena.zero_grad()
    lo = mine(x)
    loss = F.cross_entropy(lo, y)
    loss.backward()
    torch.cuda.synchronize()
    key = int(mine._b200.dropout_key.item())
    masks = dropout_oracle.network_masks(key, dropout_oracle.block_spec(ref, x.shape[0], *x.shape[2:]), x.shape[0])
    names = [n for n, _ in mine.named_parameters()]
    xc, yc = x.cpu(), y.cpu()
    o_logits, o_loss, o_grads, o_bufs = dropout_oracle.loss_and_grads(sd, xc, yc, masks, 0.3, quant=True)
    gq = torch.Generator().manual_seed(99)
    xb = xc.to(torch.bfloat16)
    nudge = torch.rand(xc.shape, generator=gq) < 1e-3
    xp = torch.where(nudge, (xb.float() * (1 + 2 ** -8)).to(torch.bfloat16), xb).float()
    p_logits, _, p_grads, _ = dropout_oracle.loss_and_grads(sd, xp, yc, masks, 0.3, quant=True)
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


@pytest.mark.parametrize('cfg', [WRN, R20], ids=['wrn16_4', 'resnet20'])
def test_network_against_bf16_oracle(cfg):
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, cfg, (3, 32, 32), 10, batch=32)
    _check_against_dropout_oracle(mine, ref, x, y)
    # eval mode ignores dropout: the converted model's eval logits equal those of the same model without dropout
    plain = resnet(**dict(cfg, dropout=0))
    plain.load_state_dict(mine.state_dict())
    from convnet.pytorch_b200.engine import convert_b200
    convert_b200(plain)
    mine.eval(); plain.eval()
    with torch.no_grad():
        assert _same(mine(x), plain(x))


def _trainer(model, mix=False):
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    opt = OptimRegime(model, copy.deepcopy(model.regime))
    kw = dict(mixup=1.0) if mix else {}
    return Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9, **kw)


def test_graph_replay_matches_eager():
    """Trainer.train with captured graphs against graphs disabled under the same torch.manual_seed: parameters, running
    buffers and losses bit for bit after 6 steps (each replay draws a fresh key)"""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    _setup()
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(32, 3, 32, 32, generator=g), torch.randint(0, 10, (32,), generator=g)) for _ in range(6)]
    results = []
    for use_graphs in (False, True):
        torch.manual_seed(123)
        model = convert_b200(resnet(**R20), 'cuda')
        tr = _trainer(model)
        tr.use_graphs = use_graphs
        keys = []
        res = tr.train(batches)
        assert (tr.graph_replays > 0) == use_graphs
        if use_graphs:
            assert tr.graph_replays == len(batches) - 2
        keys.append(int(model._b200.dropout_key.item()))
        results.append((res, keys, {k: v.detach().clone() for k, v in model.state_dict().items()}))
    (r0, k0, s0), (r1, k1, s1) = results
    assert k0 == k1, 'the last step drew another key'
    assert r0['loss'] == r1['loss'], (r0['loss'], r1['loss'])
    diff = [k for k in s0 if not torch.equal(s0[k], s1[k])]
    assert not diff, 'graph replay differs from eager in %s' % diff[:5]


def test_mobilenet_v2_head_dropout_graph_replay_matches_eager():
    """MobileNet-v2 with its head Dropout(0.2): Trainer.train with captured graphs against graphs disabled under the same
    torch.manual_seed, parameters, running buffers and losses bit for bit after 6 steps -- the head's keep mask comes
    from torch's CUDA generator, whose Philox offset a captured graph advances on every replay, so each replayed step
    draws the mask the eager step draws"""
    from convnet.pytorch_b200.models import mobilenet_v2
    from convnet.pytorch_b200.engine import convert_b200
    _setup()
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(32, 3, 64, 64, generator=g), torch.randint(0, 1000, (32,), generator=g)) for _ in range(6)]
    results = []
    for use_graphs in (False, True):
        torch.manual_seed(123)
        model = convert_b200(mobilenet_v2(dataset='imagenet'), 'cuda')
        assert model._b200.dropout_p == 0.2
        tr = _trainer(model)
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


@pytest.mark.parametrize('kind', ['mixup', 'device_augment'])
def test_combines_with_mixup_and_device_augment(kind):
    """a dropout WRN-16-4 trains through Trainer.train with MixUp, or on uint8 batches augmented on the device: finite
    losses, parameters move, and the step still launches the dropout kernels"""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from torch.profiler import ProfilerActivity, profile
    _setup()
    torch.manual_seed(123)
    model = convert_b200(resnet(**WRN), 'cuda')
    g = torch.Generator().manual_seed(1)
    if kind == 'mixup':
        tr = _trainer(model, mix=True)
        batches = [(torch.randn(32, 3, 32, 32, generator=g), torch.randint(0, 10, (32,), generator=g))
                   for _ in range(4)]
    else:
        from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment
        tr = _trainer(model)
        spec = BatchAugment(padding=4, duplicates=2)
        batches = []
        for _ in range(4):
            img = torch.randint(0, 256, (16, 32, 32, 3), generator=g, dtype=torch.uint8)
            batches.append((AugmentedBatch(img, spec.sample(16, 32, 32), spec),
                            torch.randint(0, 10, (16,), generator=g).repeat_interleave(2)))
    w0 = model.layer1[0].conv2.weight.detach().clone()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = tr.train(batches)
        torch.cuda.synchronize()
    assert np.isfinite(res['loss'])
    assert not torch.equal(w0, model.layer1[0].conv2.weight)
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    assert any('bn_apply_dropout_kernel' in n for n in names) and any('bn_bwd_dx_dropout_kernel' in n for n in names)


def _step_launches(cfg):
    """GPU kernel names of one train_step (the second) of a freshly converted CIFAR ResNet, B = 32"""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    _setup()
    torch.manual_seed(123)
    model = convert_b200(resnet(**cfg), 'cuda')
    g = torch.Generator().manual_seed(1)
    x = torch.randn(32, 3, 32, 32, generator=g).cuda()
    y = torch.randint(0, 10, (32,), generator=g).cuda()
    rt = model._b200
    model.train()
    rt.train_step(x, y)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rt.train_step(x, y)
        torch.cuda.synchronize()
    return model, collections.Counter(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def test_train_step_runs_only_library_kernels():
    """a profiler trace of one dropout train_step: besides library kernels and memsets it runs the plain model's torch
    work (the 3-channel CIFAR stem's weight pad-cast and gradient add) and one more kernel, the key draw"""
    _, drop = _step_launches(WRN)
    _, plain = _step_launches(dict(WRN, dropout=0))

    def other(c):
        return collections.Counter({n: k for n, k in c.items() if 'b200::' not in n and 'memset' not in n.lower()})
    extra = other(drop) - other(plain)
    print('\ndropout train_step: %d kernels, outside the library and the plain step: %s' % (sum(drop.values()),
                                                                                          list(extra)))
    assert not other(plain) - other(drop)
    assert sum(extra.values()) == 1 and 'random_full_64_bits_range' in next(iter(extra)), extra
    assert sum(k for n, k in drop.items() if 'bn_apply_dropout_kernel' in n) == 6
    assert sum(k for n, k in drop.items() if 'bn_bwd_dx_dropout_kernel' in n) == 6


def test_zero_dropout_takes_the_plain_path():
    """dropout=0 / None builds exactly the plain model's step: the same kernel launches and no key"""
    lists = []
    for cfg in (dict(WRN, dropout=0), dict(WRN, dropout=None), {k: v for k, v in WRN.items() if k != 'dropout'}):
        model, names = _step_launches(cfg)
        assert model._b200.dropout_key is None
        lists.append(names)
    assert lists[0] == lists[2] and lists[1] == lists[2]


def test_out_of_range_rates_raise():
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.lib import B200Error
    model = resnet(dataset='cifar10', depth=8, dropout=0.3)
    model.layer1[0].dropout.p = 1.0
    with pytest.raises(B200Error):
        convert_b200(model, 'cuda')
    with pytest.raises(B200Error):
        convert_b200(resnet(dataset='cifar10', depth=8, dropout=0.3, bn_norm='L1'), 'cuda')
