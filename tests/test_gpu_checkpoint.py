"""Activation checkpointing (``checkpoint_segments``) on the kernel path: ResNetRuntime keeps only the input and the BN
coefficient vectors of a checkpointed segment, and its backward pass reruns the segment's forward launches just before
the segment's backward.

Each checkpointed model is compared with the same weights built without checkpointing:
  * one train_step: logits, loss and the whole gradient arena bit for bit; the recomputed z / y / masks bit for bit
    against the forward's; running buffers bit for bit outside the checkpointed segments, and inside them two
    sequential momentum updates (the reference's reentrant recompute updates them again) with num_batches_tracked +2;
  * 6 Trainer steps (4 CUDA-graph replays): losses and the final parameter arena bit for bit;
  * eval logits, BN folded and unfolded, bit for bit;
  * the library calls of one train_step: those of the plain model, plus, in recompute windows, exactly the
    checkpointed blocks' forward calls; a profiler trace shows only library kernels and memsets;
  * the eager-step peak memory of ResNet-101 at batch 64, 224 px, which falls by at least what the segments no longer
    keep.
"""
import copy
import inspect

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

CONFIGS = {
    'resnet50_128': ('resnet', dict(dataset='imagenet', depth=50), 128),
    'resnet18_l1_64': ('resnet', dict(dataset='imagenet', depth=18, bn_norm='L1'), 64),
    'resnet_se50_64': ('resnet_se', dict(dataset='imagenet', depth=50), 64),
    'resnext50_64': ('resnext', dict(dataset='imagenet', depth=50), 64),
}
BATCH = 32


def _bn_state(name, C):
    """deterministic BN state: no zero gamma (the init zeroes each block's last one) and a visible momentum update"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name.replace('.module', ''))) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def _build(factory, cfg, s):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.models.modules.lp_norm import L1BatchNorm2d
    torch.manual_seed(123)
    model = models.__dict__[factory](**dict(cfg, checkpoint_segments=s))
    with torch.no_grad():
        for n, m in model.named_modules():
            if isinstance(m, (nn.BatchNorm2d, L1BatchNorm2d)):
                for k, v in _bn_state(n, m.num_features).items():
                    getattr(m, k).copy_(v)
    return convert_b200(model, 'cuda')


def _pair(name, s):
    factory, cfg, px = CONFIGS[name]
    plain, ckpt = _build(factory, cfg, 0), _build(factory, cfg, s)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(BATCH, 3, px, px, generator=g).cuda()
    y = torch.randint(0, 1000, (BATCH,), generator=g).cuda()
    return plain, ckpt, x, y


def _plain_key(k):
    return k.replace('.module.', '.')


def _checkpointed_bn_names(ckpt):
    """state_dict prefixes of the BN layers inside checkpointed segments"""
    from convnet.pytorch_b200.models.modules.checkpoint import CheckpointModule
    from convnet.pytorch_b200.models.modules.lp_norm import L1BatchNorm2d
    names = set()
    for lname, layer in ckpt.named_children():
        if not isinstance(layer, CheckpointModule):
            continue
        for a, b in layer.segments():
            for j in range(a, b):
                for n, m in layer.module[j].named_modules():
                    if isinstance(m, (nn.BatchNorm2d, L1BatchNorm2d)):
                        names.add('%s.module.%d.%s' % (lname, j, n))
    return names


@pytest.mark.parametrize('s', [1, 2, 4])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_train_step_bitwise_and_running_buffers(name, s):
    plain, ckpt, x, y = _pair(name, s)
    before = {_plain_key(k): v.clone() for k, v in ckpt.state_dict().items()}
    rp, rc = plain._b200, ckpt._b200
    assert rc.segments and not rp.segments
    lp, sp = rp.train_step(x, y)
    lc, sc = rc.train_step(x, y)
    torch.cuda.synchronize()
    assert torch.equal(lp, lc) and torch.equal(sp, sc)
    assert torch.equal(rp.arena.g32, rc.arena.g32), 'gradient arena differs'
    inside = _checkpointed_bn_names(ckpt)
    assert inside
    sd_p = plain.state_dict()
    l1 = 'bn_norm' in CONFIGS[name][1]
    for k, v in ckpt.state_dict().items():
        pk = _plain_key(k)
        layer = k.rsplit('.', 1)[0]
        if layer not in inside or not ('running' in k or 'num_batches_tracked' in k):
            assert torch.equal(v, sd_p[pk]), k
        elif 'num_batches_tracked' in k:
            assert int(v) == int(before[pk]) + 2, k
        else:
            # r1 = a r0 + c b (plain, one update) -> r2 = a r1 + c b' with b' the recomputed statistic of the same
            # batch: expected a r1 + (r1 - a r0).  a = 1 - momentum (BatchNorm2d), momentum (L1: weights the old value)
            a = 0.1 if l1 else 0.9
            r0, r1 = before[pk].double(), sd_p[pk].double()
            expect = a * r1 + (r1 - a * r0)
            err = float(((v.double() - expect).abs() / (expect.abs() + 1e-3)).max())
            assert err < 2e-5, (k, err)


@pytest.mark.parametrize('s', [1, 2, 4])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_recomputed_activations_bitwise(name, s):
    """the tensors the recompute rebuilds are the forward's: z, y and the mask bits of every unit"""
    plain, ckpt, x, y = _pair(name, s)
    rp, rc = plain._b200, ckpt._b200
    _, tp = rp.run_forward(x, True, True)
    _, tc = rc.run_forward(x, True, True)
    n_seg = 0
    for i, seg in enumerate(tc['blocks']):
        if seg is None or 'segment' not in seg:
            continue
        a, b = seg['segment']
        assert a == i
        for j, rec in zip(range(a, b), rc._recompute(seg)):
            ref = tp['blocks'][j]
            units = [(u, v) for u, v in zip(ref['units'], rec['units'])]
            if ref['down'] is not None:
                units.append((ref['down'], rec['down']))
            for u, v in units:
                for f in ('z', 'y', 'mask'):
                    p, q = getattr(u, f, None), getattr(v, f, None)     # _stats_only units have no mask
                    assert (p is None) == (q is None) and (p is None or torch.equal(p, q)), (j, f)
                for f in ('mean', 'invstd', 'scale', 'shift'):
                    assert torch.equal(getattr(u, f), getattr(v, f)), (j, f)
        n_seg += 1
    assert n_seg == len(rc.segments)
    torch.cuda.synchronize()


@pytest.mark.parametrize('s', [1, 2])
def test_graph_replays_bitwise(s):
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    factory, cfg, _ = CONFIGS['resnet50_128']
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(16, 3, 64, 64, generator=g), torch.randint(0, 1000, (16,), generator=g))
               for _ in range(6)]
    out = []
    for seg in (0, s):
        model = _build(factory, cfg, seg)
        tr = Trainer(model, CrossEntropyLoss().cuda(), OptimRegime(model, copy.deepcopy(model.regime)),
                     device='cuda', print_freq=10 ** 9)
        res = tr.train(batches)
        assert tr.graph_replays == len(batches) - 2
        out.append((res['loss'], model._b200.arena.p32.clone()))
    assert out[0][0] == out[1][0]
    assert torch.equal(out[0][1], out[1][1]), 'parameters differ after 6 steps'


@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_eval_logits_equal(name):
    from convnet.pytorch_b200 import engine
    plain, ckpt, x, _ = _pair(name, 2)
    saved = engine.FOLD_BN_EVAL
    try:
        plain.eval(); ckpt.eval()
        with torch.no_grad():
            for fold in (False, True):
                engine.FOLD_BN_EVAL = fold
                assert torch.equal(plain(x), ckpt(x)), 'fold=%s' % fold
    finally:
        engine.FOLD_BN_EVAL = saved


def _record_ops(rt, fn):
    """names of the ops calls of fn(), each tagged 'recompute' inside Runtime._recompute and with the block index
    inside _block_fwd"""
    from convnet.pytorch_b200 import ops
    calls, tag = [], {'recompute': False, 'block': None}
    saved = {}
    for n, f in vars(ops).items():
        if not n.startswith('_') and inspect.isfunction(f) and f.__module__ == ops.__name__:
            def wrap(*a, _n=n, _f=f, **k):
                calls.append((_n, tag['recompute'], tag['block']))
                return _f(*a, **k)
            saved[n] = f
            setattr(ops, n, wrap)
    block_fwd, recompute = rt._block_fwd, rt._recompute

    def blk(spec, h, training):
        tag['block'] = rt.blocks.index(spec)
        try:
            return block_fwd(spec, h, training)
        finally:
            tag['block'] = None

    def rec(seg):
        tag['recompute'] = True
        try:
            return recompute(seg)
        finally:
            tag['recompute'] = False
    rt._block_fwd, rt._recompute = blk, rec
    try:
        fn()
    finally:
        for n, f in saved.items():
            setattr(ops, n, f)
        del rt._block_fwd, rt._recompute
    return calls


@pytest.mark.parametrize('name', ['resnet50_128', 'resnet18_l1_64'])
def test_train_step_library_calls(name):
    plain, ckpt, x, y = _pair(name, 2)
    rp, rc = plain._b200, ckpt._b200
    rp.train_step(x, y)
    rc.train_step(x, y)
    cp = _record_ops(rp, lambda: rp.train_step(x, y))
    cc = _record_ops(rc, lambda: rc.train_step(x, y))
    assert not any(r for _, r, _ in cp)
    # outside the recompute windows: the plain model's calls, in order
    assert [c[0] for c in cc if not c[1]] == [c[0] for c in cp]
    # inside: the forward calls of the checkpointed blocks, block by block
    ckpt_blocks = [i for a, b in rc.segments for i in range(a, b)]
    for i in ckpt_blocks:
        fwd = [c[0] for c in cp if c[2] == i and not c[1]]
        again = [c[0] for c in cc if c[2] == i and c[1]]
        assert fwd and again == fwd, i
    assert sum(c[1] for c in cc) == sum(c[2] in ckpt_blocks for c in cp)


_PROFILE_CHILD = r"""
import sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import test_gpu_checkpoint as t
_, ckpt, x, y = t._pair('resnet50_128', 1)
rt = ckpt._b200
rt.train_step(x, y)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    rt.train_step(x, y)
    torch.cuda.synchronize()
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        print('KERNEL', e.name)
"""


def test_checkpointed_train_step_runs_only_library_kernels():
    """a profiler trace of one checkpointed train_step: library kernels, memsets and torch.zeros fills only.  It runs in
    a child process so that this profiler session cannot change what later sessions of the test process record."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    out = subprocess.run([sys.executable, '-c', _PROFILE_CHILD, os.path.dirname(here), here], check=True,
                         capture_output=True, text=True).stdout
    names = [line[len('KERNEL '):] for line in out.splitlines() if line.startswith('KERNEL ')]
    lib_k = [n for n in names if 'b200::' in n]
    other = sorted({n for n in names if 'b200::' not in n and 'memset' not in n.lower() and 'FillFunctor' not in n})
    assert lib_k and not other, 'kernels outside the library: %s' % other


def _tape_bytes(blocks):
    n = 0
    for saved in blocks:
        units = list(saved['units']) + ([saved['down']] if saved['down'] is not None else [])
        for u in units:
            for t in (u.z, u.y, getattr(u, 'mask', None)):
                n += t.numel() * t.element_size() if t is not None else 0
    return n


def test_peak_memory_falls():
    """ResNet-101, batch 64, 224 px, s = 2: the eager-step peak falls at least by the z / y / mask bytes of the
    checkpointed blocks, less the largest segment's (rebuilt during its backward), halved for allocator rounding"""
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    g = torch.Generator().manual_seed(2)
    x = torch.randn(64, 3, 224, 224, generator=g).cuda()
    y = torch.randint(0, 1000, (64,), generator=g).cuda()
    peaks, segments = [], None
    for s in (0, 2):
        torch.manual_seed(123)
        model = convert_b200(models.resnet(dataset='imagenet', depth=101, checkpoint_segments=s), 'cuda')
        rt = model._b200
        rt.train_step(x, y)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        rt.train_step(x, y)
        torch.cuda.synchronize()
        peaks.append(torch.cuda.max_memory_allocated() - base)
        if s:
            segments = rt.segments
        else:
            _, tape = rt.run_forward(x, True, True)
            plain_tape = tape['blocks']
        del model, rt
    per_seg = [_tape_bytes(plain_tape[a:b]) for a, b in segments]
    bound = (sum(per_seg) - max(per_seg)) // 2
    print('\nResNet-101 b64 224px eager step peak: plain %.2f GB, s=2 %.2f GB, bound %.2f GB'
          % (peaks[0] / 2 ** 30, peaks[1] / 2 ** 30, bound / 2 ** 30))
    assert peaks[0] - peaks[1] >= bound > 0
