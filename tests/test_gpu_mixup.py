"""MixUp / CutMix on the kernel path: the mixing input relayout (b200_input_prep_mix / _u8_mix) exactly, the soft-target
cross-entropy (b200_softmax_ce_mix) against fp64, whole Trainer steps against the bf16 oracle fed with the same
draws, and CUDA-graph replays that must follow each step's draws."""
import copy
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_ops import close_bf16
from test_gpu_engine import _pair, _rel, _cos, _global, _setup
from test_mixup_cpu import oracle_soft_loss_and_grads, soft_cross_entropy, soft_target

pytestmark = pytest.mark.gpu

N, C, H, W = 6, 3, 14, 14
BOXES = [(0, 0, 0, 0),            # empty
         (0, H, 0, W),            # whole image
         (0, 5, 3, 9), (9, H, 3, 9), (4, 8, 0, 5), (4, 8, 10, W),      # touching the top, bottom, left, right edge
         (3, 9, 5, 11), (1, 2, 13, 14)]                                 # odd edges: split 2x2 space-to-depth cells
PERMS = [list(range(N)), [2, 1, 0, 3, 5, 4]]                           # identity; 1 and 3 are fixed points
LAYOUTS = [(8, False, False), (16, True, False), (16, True, True)]      # modes 0, 1, 2


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def _mix(perm, lam, box, kind):
    ops = _ops()
    blk = torch.zeros(5, dtype=torch.int32)
    blk[:1].view(torch.float32)[0] = float(np.float32(lam))
    blk[1:] = torch.tensor(box, dtype=torch.int32)
    return ops.Mix(torch.tensor(perm, dtype=torch.int64).cuda(), blk.cuda(), kind)


def _ref_mix(x, perm, lam, box, kind):
    """the reference's fp32 mixing of an NCHW batch (utils/mixup.py:19-26 / 84-90)."""
    from convnet.pytorch_b200.lib import MIX_MIXUP
    p = torch.tensor(perm)
    if kind == MIX_MIXUP:
        lam_t = torch.tensor([np.float32(lam)]).view(-1, 1, 1, 1)
        return lam_t * x + (1. - lam_t) * x[p]
    r0, r1, c0, c1 = box
    out = x.clone()
    out[..., r0:r1, c0:c1] = x[p][..., r0:r1, c0:c1]
    return out


def _nan_out(cpad, s2d, border):
    shape = (N, H // 2 + 3, W // 2 + 3, cpad) if (s2d and border) else ((N, H // 2, W // 2, cpad) if s2d else (N, H, W, cpad))
    return torch.full(shape, float('nan'), dtype=torch.bfloat16, device='cuda')


def _u8_batch():
    g = torch.Generator().manual_seed(3)
    return torch.randint(0, 256, (N, H, W, C), generator=g, dtype=torch.uint8)


def _u8_reference(x_u8, mean, std):
    """fp64 u8*scale + bias with the kernel's fp32 coefficients, rounded to fp32 once (== fmaf: both operations are
    exact in fp64) -> NCHW."""
    scale, bias = _ops().u8_norm_coeffs(mean, std)
    s = torch.tensor(np.float32(scale), dtype=torch.float64)
    b = torch.tensor(np.float32(bias), dtype=torch.float64)
    return (x_u8.double() * s + b).float().permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize('cpad,s2d,border', LAYOUTS)
@pytest.mark.parametrize('src', ['fp32', 'u8'])
def test_input_prep_mix_is_exact(cpad, s2d, border, src):
    """mixup == input_prep(reference_mix(x)) and cutmix == input_prep(x with the box pasted), bit for bit, written into
    NaN-filled buffers (an element left unwritten fails); every box and permutation case."""
    from convnet.pytorch_b200.lib import MIX_MIXUP, MIX_CUTMIX
    ops = _ops()
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    if src == 'fp32':
        x = torch.randn(N, C, H, W, generator=torch.Generator().manual_seed(2))
        x_ref = x
        run = lambda mix, out: ops.input_prep(x.cuda(), cpad, s2d=s2d, border=border, mix=mix, out=out)  # noqa: E731
    else:
        xu = _u8_batch()
        x_ref = _u8_reference(xu, mean, std)
        run = lambda mix, out: ops.input_prep_u8(xu.cuda(), cpad, mean, std, s2d=s2d, border=border, mix=mix,  # noqa: E731
                                                 out=out)
        # the unmixed uint8 relayout equals the relayout of its fp32 normalisation
        plain = run(None, _nan_out(cpad, s2d, border))
        assert torch.equal(plain.view(torch.int16), ops.input_prep(x_ref.cuda(), cpad, s2d=s2d, border=border).view(torch.int16))
    cases = [(MIX_MIXUP, lam, (0, 0, 0, 0)) for lam in (0.37, 0.9)] + [(MIX_CUTMIX, 0.5, b) for b in BOXES]
    for perm in PERMS:
        for kind, lam, box in cases:
            got = run(_mix(perm, lam, box, kind), _nan_out(cpad, s2d, border))
            want = ops.input_prep(_ref_mix(x_ref, perm, lam, box, kind).cuda(), cpad, s2d=s2d, border=border)
            torch.cuda.synchronize()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (kind, lam, box, perm)


@pytest.mark.parametrize('B,classes,ld', [(37, 10, 16), (64, 1000, 1000), (20, 100, 104)])
def test_softmax_ce_mix_against_fp64(B, classes, ld):
    """loss within 1e-5 relative of the fp64 soft-target cross-entropy, dlogits within bf16 rounding, top-1 / top-5 of
    the ORIGINAL target, padding columns zero; lambda = 1 with the identity permutation is b200_softmax_ce at eps = 0
    bit for bit."""
    from convnet.pytorch_b200.lib import MIX_MIXUP
    from convnet.pytorch_b200.utils.meters import accuracy
    ops = _ops()
    g = torch.Generator().manual_seed(B + classes)
    logits = (torch.randn(B, ld, generator=g) * 3).cuda()
    t = torch.randint(0, classes, (B,), generator=g)
    perm = torch.randperm(B, generator=g)
    perm[:3] = torch.arange(3)                       # fixed points: t2 == t on those rows
    up = torch.tensor([0.5], device='cuda')
    for lam in (0.0, 0.37, 1.0):
        mix = _mix(perm.tolist(), lam, (0, 0, 0, 0), MIX_MIXUP)
        stats = torch.empty(3, device='cuda')
        rows = torch.empty(2 * B, device='cuda')
        dl = torch.full((B, ld), float('nan'), dtype=torch.bfloat16, device='cuda')
        ops.softmax_ce_mix(logits, t.cuda(), mix, classes, loss=stats, row_loss=rows, dlogits=dl, grad_scale_dev=up)
        torch.cuda.synchronize()
        lg = logits[:, :classes].double().cpu()
        q = soft_target(t, classes, (t[perm], lam)).double()
        lsm = F.log_softmax(lg, -1)
        loss_ref = float((-(q * lsm).sum(-1)).mean())
        assert abs(float(stats[0]) - loss_ref) <= 1e-5 * abs(loss_ref), (lam, float(stats[0]), loss_ref)
        grad_ref = 0.5 * (lsm.exp() - q) / B
        assert close_bf16(dl[:, :classes].cpu(), grad_ref), lam
        if ld > classes:
            assert float(dl[:, classes:].float().abs().max()) == 0.0
        p1, p5 = accuracy(logits[:, :classes], t.cuda(), topk=(1, 5))
        assert abs(float(stats[1]) - float(p1)) < 1e-4 and abs(float(stats[2]) - float(p5)) < 1e-4
    ident = _mix(list(range(B)), 1.0, (0, 0, 0, 0), MIX_MIXUP)
    outs = []
    for fn in (lambda s, r, d: ops.softmax_ce_mix(logits, t.cuda(), ident, classes, loss=s, row_loss=r, dlogits=d,
                                                  grad_scale_dev=up),
               lambda s, r, d: ops.softmax_ce(logits, t.cuda(), classes, 0.0, loss=s, row_loss=r, dlogits=d,
                                              grad_scale_dev=up)):
        s, r = torch.empty(3, device='cuda'), torch.empty(2 * B, device='cuda')
        d = torch.empty((B, ld), dtype=torch.bfloat16, device='cuda')
        fn(s, r, d)
        outs.append((s, r, d))
    (s0, r0, d0), (s1, r1, d1) = outs
    assert torch.equal(s0, s1) and torch.equal(r0, r1) and torch.equal(d0.view(torch.int16), d1.view(torch.int16))


class _NoStep(object):
    """Optimizer stand-in: the Trainer's step runs completely, the gradients stay in the arena for inspection."""

    def __init__(self, model):
        self.model = model

    def zero_grad(self):
        self.model._b200.arena.zero_grad_force()

    def update(self, epoch, steps):
        pass

    pre_forward = pre_backward = step = lambda self, *a, **k: None

    def set_grad_unscale(self, *a):
        pass


def _trainer_step(model, x, y, seed, **flags):
    """one Trainer._step on the fused kernel path with the draws of ``seed``; -> (logits, stats, mixing module)."""
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    tr = Trainer(model, CrossEntropyLoss(), _NoStep(model), device='cuda', print_freq=10 ** 9, **flags)
    tr.use_graphs = False
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    out, stats, _ = tr._step(x, y, training=True)
    torch.cuda.synchronize()
    assert torch.is_tensor(stats), 'the fused kernel path was not taken'
    return out, stats, tr.last_mix


def _mixed_cpu(x, m):
    from convnet.pytorch_b200.utils.mixup import CutMix
    from convnet.pytorch_b200.lib import MIX_MIXUP, MIX_CUTMIX
    kind = MIX_CUTMIX if isinstance(m, CutMix) else MIX_MIXUP
    return _ref_mix(x, m.mix_index.tolist(), float(m.mix_values), getattr(m, 'box', None), kind)


def _check_mixed_step_against_bf16_oracle(mine, ref, x, y, seed, logit_tol=1e-3, grad_tol=1e-2, cos_min=0.999, **flags):
    """The bounds of test_gpu_engine._check_against_bf16_oracle (with the oracle's self-sensitivity to one-ulp input
    nudges) for a mixed step: the oracle sees the reference-mixed batch and the soft target of the same draws."""
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    mine.train()
    lo, stats, m = _trainer_step(mine, x, y, seed, **flags)
    assert 0.0 < float(m.mix_values) < 1.0, 'a trivial draw would not test the mixing'
    names = [n for n, _ in mine.named_parameters()]
    yc = y.cpu()
    soft = (yc[m.mix_index], float(m.mix_values))
    xm = _mixed_cpu(x.cpu(), m)
    o_logits, o_loss, o_grads, o_bufs = oracle_soft_loss_and_grads(sd, xm, yc, soft, quant=True)
    gq = torch.Generator().manual_seed(99)
    xb = xm.to(torch.bfloat16)
    nudge = torch.rand(xm.shape, generator=gq) < 1e-3
    xp = torch.where(nudge, (xb.float() * (1 + 2 ** -8)).to(torch.bfloat16), xb).float()
    p_logits, _, p_grads, _ = oracle_soft_loss_and_grads(sd, xp, yc, soft, quant=True)
    gm = _global({n: p.grad for n, p in mine.named_parameters()}, names)
    go, gp = _global(o_grads, names), _global(p_grads, names)
    per = sorted((_cos(p.grad.cpu(), o_grads[n]), n) for n, p in mine.named_parameters() if float(o_grads[n].norm()) > 0)
    self_worst = min(_cos(p_grads[n], o_grads[n]) for n in names if float(o_grads[n].norm()) > 0)
    s_log, s_grad = _rel(p_logits, o_logits), _rel(gp, go)
    print('mixed step (lambda %.4f) vs bf16 oracle: logits rel %.3e  dloss %.3e  grad rel %.3e  worst %s | self %.3e %.3e '
          '%.5f' % (float(m.mix_values), _rel(lo.cpu(), o_logits), abs(float(stats[0]) - float(o_loss)), _rel(gm, go),
                    per[:2], s_log, s_grad, self_worst))
    assert _rel(lo.cpu(), o_logits) < max(logit_tol, 1.5 * s_log)
    assert abs(float(stats[0]) - float(o_loss)) < 5e-3
    assert _rel(gm, go) < max(grad_tol, 1.5 * s_grad)
    assert 1.0 - per[0][0] < max(1.0 - cos_min, 1.5 * (1.0 - self_worst)), per[0]
    for n, b in mine.named_buffers():
        if 'running' in n:
            assert _rel(b.cpu(), o_bufs[n]) < 1e-3, n
    # the meters count against the original target
    from convnet.pytorch_b200.utils.meters import accuracy
    p1, p5 = accuracy(lo, y, topk=(1, 5))
    assert abs(float(stats[1]) - float(p1)) < 1e-3 and abs(float(stats[2]) - float(p5)) < 1e-3


def test_resnet18_imagenet_mixup_step_against_bf16_oracle():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=18), (3, 64, 64), 1000, batch=32)
    _check_mixed_step_against_bf16_oracle(mine, ref, x, y, seed=0, mixup=0.2)


def test_resnet20_cifar_cutmix_step_against_bf16_oracle():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, batch=32)
    _check_mixed_step_against_bf16_oracle(mine, ref, x, y, seed=1, cutmix=1.0)


@pytest.mark.parametrize('flags', [dict(mixup=0.2), dict(cutmix=1.0)])
def test_uint8_mixed_step_matches_normalised_fp32(flags):
    """A uint8 NHWC batch mixed in the relayout kernel gives the step of its fp32 normalisation with the same draws."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200, Runtime
    _setup()
    g = torch.Generator().manual_seed(4)
    xu = torch.randint(0, 256, (32, 32, 32, 3), generator=g, dtype=torch.uint8)
    y = torch.randint(0, 10, (32,), generator=g).cuda()
    xf = _u8_reference(xu, Runtime.input_mean, Runtime.input_std)
    res = []
    for x in (xu.cuda(), xf.cuda()):
        torch.manual_seed(123)
        model = convert_b200(resnet(dataset='cifar10', depth=20), 'cuda')
        lo, stats, m = _trainer_step(model, x, y, 0, **flags)
        res.append((lo.cpu(), stats.cpu(), m.mix_index.clone(), float(m.mix_values)))
    (l0, s0, p0, m0), (l1, s1, p1, m1) = res
    assert torch.equal(p0, p1) and m0 == m1
    assert _rel(l0, l1) < 1e-6 and abs(float(s0[0]) - float(s1[0])) < 1e-6


@pytest.mark.parametrize('flags', [dict(mixup=0.2), dict(cutmix=1.0)])
def test_trainer_cuda_graph_replay_with_mixing_matches_eager(flags):
    """test_trainer_cuda_graph_replay_matches_eager with mixing: 6 steps, 4 of them replayed.  Parameters and meters
    agree with the eager run, and every replayed step's loss equals the loss recomputed on the host from its logits
    and THAT step's draws -- the graph read the new permutation, lambda and box, not the captured ones."""
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
        model = resnet(dataset='imagenet', depth=18)
        convert_b200(model, 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9, **flags)
        tr.use_graphs = use_graphs
        rec, step = [], tr._step

        def recording_step(inputs, target, **kw):
            n0 = tr.graph_replays
            out, loss, grad = step(inputs, target, **kw)
            m = tr.last_mix
            rec.append((out.detach().clone(), loss.detach().clone(), target.clone(), m.mix_index.clone(),
                        m.mix_values.clone(), tr.graph_replays > n0))
            return out, loss, grad
        tr._step = recording_step
        random.seed(7)
        np.random.seed(7)
        torch.manual_seed(7)
        res = tr.train(batches)
        torch.cuda.synchronize()
        assert (tr.graph_replays > 0) == use_graphs
        if use_graphs:
            assert tr.graph_replays == len(batches) - 2 and tr.graph_replayed_launches > 100
            replayed = [r for r in rec if r[5]]
            assert len(replayed) == 4
            lams = set()
            for out, stats, target, perm, lam, _ in replayed:
                t = target.cpu()
                want = float(soft_cross_entropy(out.cpu().double(), t, (t[perm], float(lam))))
                assert abs(float(stats[0]) - want) < 1e-5 * max(1.0, abs(want)), (float(stats[0]), want)
                lams.add(float(lam))
            assert len(lams) > 1, 'the replayed steps should have drawn different lambdas'
        results.append((res, {k: v.detach().float().clone() for k, v in model.state_dict().items()}))
    (r0, s0), (r1, s1) = results
    assert abs(r0['loss'] - r1['loss']) < 2e-3 * max(1.0, abs(r0['loss']))
    for k in ('prec1', 'prec5'):                      # at most one sample of the 96 may flip
        assert abs(r0[k] - r1[k]) <= 100.0 / 96 + 1e-6, k
    for k in s0:
        assert _rel(s1[k], s0[k]) < 2e-3, '%s: %.3e' % (k, _rel(s1[k], s0[k]))
