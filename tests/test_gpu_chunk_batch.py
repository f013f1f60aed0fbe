"""Gradient accumulation (``chunk_batch``) on the fused kernel path: Trainer._step splits the batch with torch.chunk,
runs one fused train_step per chunk with the loss gradient scaled by 1 / chunk_batch, and takes one optimizer step.

  * one chunked Trainer step against N eager train_steps on the same chunks (upstream / N, reduce=False) in the same
    arena: logits, the combined statistics, every arena gradient and the running buffers bit for bit; against the
    generic autograd path (an unfused criterion) to fp32 accumulation-order tolerance;
  * each chunk's device relayout (batch augmentation with D = 4, resized crop with D = 2, chunk boundaries inside one
    image's copies) bit for bit the matching rows of the whole batch's relayout; Trainer runs on those batches bit for
    bit the runs on the applied fp32 batch, graph replays included;
  * MixUp / CutMix with N = 2: per-chunk draws, against the host mixing of the generic path;
  * 6 chunked steps replayed from captured graphs bit for bit the eager steps;
  * the library launches of a chunked step: N times a chunk's train_step plus one optimizer step, no host apply().
"""
import copy
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CONFIGS = {
    'resnet20_32': (dict(dataset='cifar10', depth=20), 32, 10),
    'resnet18_l1_64': (dict(dataset='imagenet', depth=18, bn_norm='L1'), 64, 1000),
    'resnet50_ckpt2_64': (dict(dataset='imagenet', depth=50, checkpoint_segments=2), 64, 1000),
    'wrn16_4_dropout_32': (dict(dataset='cifar10', depth=16, width=[64, 128, 256], dropout=0.3), 32, 10),
}
BATCH = 32


class _NoStep(object):
    """optimizer stand-in: zero_grad clears the arena, step leaves the accumulated gradients in place"""

    def __init__(self, model):
        self.model = model

    def zero_grad(self):
        self.model._b200.arena.zero_grad_force()

    def update(self, epoch, steps):
        pass

    pre_forward = pre_backward = step = lambda self, *a, **k: None

    def set_grad_unscale(self, *a):
        pass


def _unfused():
    """the plain criterion under another type: Trainer takes the generic autograd path with it"""
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss

    class Unfused(CrossEntropyLoss):
        pass
    return Unfused()


def _model(name):
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    torch.manual_seed(123)
    return convert_b200(resnet(**CONFIGS[name][0]), 'cuda')


def _data(name, seed=1):
    _, px, classes = CONFIGS[name]
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(BATCH, 3, px, px, generator=g).cuda(),
            torch.randint(0, classes, (BATCH,), generator=g).cuda())


def _trainer(model, criterion=None, opt=None):
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    return Trainer(model, criterion if criterion is not None else CrossEntropyLoss(),
                   opt if opt is not None else _NoStep(model), device='cuda', print_freq=10 ** 9)


def _buffers(model):
    return {k: v.clone() for k, v in model.named_buffers()}


@pytest.mark.parametrize('N', [2, 3, 4])
@pytest.mark.parametrize('name', sorted(CONFIGS))
def test_chunked_step_equals_eager_chunks(name, N):
    from convnet.pytorch_b200 import ops
    x, y = _data(name)
    ranges = ops.chunk_rows(BATCH, N)

    # the Trainer's chunked step (eager: graphs off)
    model = _model(name)
    tr = _trainer(model)
    tr.use_graphs = False
    torch.manual_seed(7)
    out, stats, _ = tr._step(x, y, training=True, chunk_batch=N)
    torch.cuda.synchronize()
    assert torch.is_tensor(stats), 'the fused path was not taken'

    # N eager train_steps on the same chunks, upstream / N, accumulated in the same arena
    ref = _model(name)
    rt = ref._b200
    rt.arena.zero_grad_force()
    up = (torch.ones((), dtype=torch.float32) / N).cuda()
    torch.manual_seed(7)
    logits, chunk_stats = [], []
    for r0, r1 in ranges:
        lo, st = rt.train_step(x[r0:r1], y[r0:r1], 0.0, up, reduce=False)
        logits.append(lo)
        chunk_stats.append(st)
    torch.cuda.synchronize()
    assert torch.equal(out, torch.cat(logits))
    w = torch.tensor([[1.0 / N, (r1 - r0) / BATCH, (r1 - r0) / BATCH] for r0, r1 in ranges]).cuda()
    assert torch.equal(stats, (torch.stack(chunk_stats) * w).sum(0))
    assert torch.equal(model._b200.arena.g32, rt.arena.g32), 'gradient arena differs'
    mine, theirs = _buffers(model), _buffers(ref)
    for k, v in mine.items():
        assert torch.equal(v, theirs[k]), k

    # the generic autograd path of the parent (unfused criterion): same sums in another order
    gen = _model(name)
    tg = _trainer(gen, _unfused())
    tg.use_graphs = False
    torch.manual_seed(7)
    out_g, loss_g, _ = tg._step(x, y, training=True, chunk_batch=N)
    torch.cuda.synchronize()
    assert not torch.is_tensor(loss_g)
    assert torch.allclose(out, out_g, rtol=1e-5, atol=1e-5)
    assert abs(float(stats[0]) - loss_g) < 1e-5 * max(1.0, abs(loss_g))
    g0, g1 = model._b200.arena.g32, gen._b200.arena.g32
    assert float((g0 - g1).norm()) <= 1e-5 * float(g1.norm()) + 1e-12
    for k, v in _buffers(gen).items():
        assert torch.allclose(mine[k].double(), v.double(), rtol=1e-5, atol=1e-6), k


def test_num_batches_tracked_grows_by_chunks():
    from convnet.pytorch_b200 import ops
    model = _model('resnet20_32')
    x, y = _data('resnet20_32')
    tr = _trainer(model)
    before = {k: int(v) for k, v in model.named_buffers() if k.endswith('num_batches_tracked')}
    tr._step(x, y, training=True, chunk_batch=3)
    for k, v in model.named_buffers():
        if k.endswith('num_batches_tracked'):
            assert int(v) == before[k] + len(ops.chunk_rows(BATCH, 3)), k


def _aug_batch(B, D, H, W, seed, resize=None):
    from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment
    spec = BatchAugment(padding=4, cutout={'holes': 1, 'length': 8}, duplicates=D, resize=resize)
    g = torch.Generator().manual_seed(seed)
    images = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    return AugmentedBatch(images, spec.sample(B, H, W), spec), \
        torch.randint(0, 10, (B,), generator=g).repeat_interleave(D)


def _rrc_batches(steps, B, D, size, seed):
    from PIL import Image
    from convnet.pytorch_b200.utils.augment import ResizedCrop, ResizedCropCollate
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    spec = ResizedCrop(size, duplicates=D)
    collate = ResizedCropCollate(spec)
    out = []
    for _ in range(steps):
        samples = []
        for _ in range(B):
            h, w = (int(v) for v in torch.randint(size // 2, 3 * size, (2,), generator=g))
            img = Image.fromarray(torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy(), 'RGB')
            samples.append((spec(img), int(torch.randint(0, 1000, (1,), generator=g))))
        out.append(collate(samples))
    return out


@pytest.mark.parametrize('resize', [None, (24, 24)])
def test_augment_chunk_relayout_is_rows_of_the_whole(resize):
    """B = 7, D = 4, N = 3: chunks of 10, 10 and 8 rows, both boundaries inside an image's copies"""
    from convnet.pytorch_b200 import ops
    batch, _ = _aug_batch(7, 4, 32, 32, seed=3, resize=resize)
    spec = batch.spec
    aug = ops.Aug(batch.params.cuda().reshape(28, -1), spec.lut(3).cuda(), 4, spec.padding,
                  resize if resize is not None else None)
    images = batch.images.cuda()
    whole = ops.input_prep_u8_aug(images, 16, aug)
    ranges = ops.chunk_rows(28, 3)
    assert any(r0 % 4 for r0, _ in ranges)
    for r0, r1 in ranges:
        a, b0, b1 = aug.row_range(r0, r1)
        got = ops.input_prep_u8_aug(images[b0:b1], 16, a)
        assert got.shape[0] == r1 - r0 and got.is_contiguous()
        assert torch.equal(got.view(torch.int16), whole[r0:r1].view(torch.int16)), (r0, r1)


@pytest.mark.parametrize('s2d', [False, True])
def test_resized_crop_chunk_relayout_is_rows_of_the_whole(s2d):
    """B = 7, D = 2, N = 3: chunks of 5, 5 and 4 rows, both boundaries inside an image's copies"""
    from convnet.pytorch_b200 import ops
    batch, _ = _rrc_batches(1, 7, 2, 64, seed=4)[0]
    regions = batch.regions.cuda()
    rrc = ops.Rrc(batch.index.cuda(), batch.draws.cuda(), batch.spec.lut(3).cuda(), 2, batch.spec.size,
                  batch.host + (batch.nbytes,))
    whole = ops.input_prep_u8_rrc(regions, 16, rrc, s2d=s2d, border=s2d)
    ranges = ops.chunk_rows(14, 3)
    assert any(r0 % 2 for r0, _ in ranges)
    for r0, r1 in ranges:
        a, _, _ = rrc.row_range(r0, r1)
        got = ops.input_prep_u8_rrc(regions, 16, a, s2d=s2d, border=s2d)
        assert got.shape[0] == r1 - r0 and got.is_contiguous()
        assert torch.equal(got.view(torch.int16), whole[r0:r1].view(torch.int16)), (r0, r1)


def _run(model_fn, data, chunk_batch, use_graphs=True, criterion=None):
    """Trainer.train over ``data`` with the real optimizer -> (per-step stats or losses, final parameters, trainer)"""
    from convnet.pytorch_b200.utils.optim import OptimRegime
    torch.manual_seed(123)
    model = model_fn()
    tr = _trainer(model, criterion, OptimRegime(model, copy.deepcopy(model.regime)))
    tr.use_graphs = use_graphs
    losses, step = [], tr._step

    def recording_step(inputs, target, **kw):
        out, loss, grad = step(inputs, target, **kw)
        losses.append(loss.detach().clone() if torch.is_tensor(loss) else torch.tensor([loss]))
        return out, loss, grad
    tr._step = recording_step
    tr.train(data, chunk_batch=chunk_batch)
    torch.cuda.synchronize()
    return torch.stack([l.reshape(-1).cpu() for l in losses]), model._b200.arena.p32.detach().clone().cpu(), tr


def test_trainer_device_augment_chunks_match_applied_batch():
    """ResNet-20, B = 8, D = 4, N = 3 (boundaries inside copies), 6 steps: losses and parameters bit for bit those of
    the fp32 batch of apply(), and no apply() on the device-augmented run"""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.utils import augment
    data = [_aug_batch(8, 4, 32, 32, seed=10 + i) for i in range(6)]
    fn = lambda: convert_b200(resnet(dataset='cifar10', depth=20), 'cuda')     # noqa: E731
    applied = [(b.apply(), t) for b, t in data]
    real = augment.AugmentedBatch.apply
    augment.AugmentedBatch.apply = lambda self: pytest.fail('host apply() on the fused chunked path')
    try:
        l0, p0, tr = _run(fn, data, 3)
    finally:
        augment.AugmentedBatch.apply = real
    assert tr.graph_replays > 0
    l1, p1, _ = _run(fn, applied, 3)
    assert torch.equal(l0, l1), (l0, l1)
    assert torch.equal(p0, p1)


def test_trainer_resized_crop_chunks_match_applied_batch():
    """ResNet-18 (space-to-depth stem), 64 px, B = 5, D = 2, N = 3: chunks of 4, 4, 2 rows (one boundary inside an
    image's copies), 5 steps"""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    data = _rrc_batches(5, 5, 2, 64, seed=5)
    fn = lambda: convert_b200(resnet(dataset='imagenet', depth=18), 'cuda')     # noqa: E731
    l0, p0, tr = _run(fn, data, 3)
    assert tr.graph_replays > 0
    l1, p1, _ = _run(fn, [(b.apply(), t) for b, t in data], 3)
    assert torch.equal(l0, l1), (l0, l1)
    assert torch.equal(p0, p1)


@pytest.mark.parametrize('flags', [{'mixup': 0.4}, {'cutmix': 1.0}])
def test_mixing_draws_per_chunk(flags):
    """ResNet-20, N = 2: each chunk draws its own mixing (the reference's order, the chunk's size); the fused step
    matches the generic path, which mixes the fp32 chunk on the host side with torch"""
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    x, y = _data('resnet20_32')
    runs = []
    for crit in (CrossEntropyLoss(), _unfused()):
        model = _model('resnet20_32')
        tr = Trainer(model, crit, _NoStep(model), device='cuda', print_freq=10 ** 9, **flags)
        tr.use_graphs = False
        draws, real = [], tr._draw_mix

        def draw(batch_size, average_output=False):
            m = real(batch_size, average_output)
            draws.append((batch_size, m.mix_index.clone(), float(m.mix_values), getattr(m, 'box', None)))
            return m
        tr._draw_mix = draw
        random.seed(3)
        np.random.seed(3)
        torch.manual_seed(3)
        out, loss, _ = tr._step(x, y, training=True, chunk_batch=2)
        torch.cuda.synchronize()
        runs.append((out, loss, model._b200.arena.g32.clone(), draws))
    (o0, s0, g0, d0), (o1, l1, g1, d1) = runs
    assert torch.is_tensor(s0) and not torch.is_tensor(l1)
    assert [d[0] for d in d0] == [16, 16]
    assert len(d0) == len(d1)
    for a, b in zip(d0, d1):
        assert a[0] == b[0] and torch.equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]
    assert not torch.equal(d0[0][1], d0[1][1]), 'both chunks drew the same permutation'
    assert torch.allclose(o0, o1, rtol=1e-4, atol=1e-4)
    assert abs(float(s0[0]) - l1) < 1e-4
    assert float((g0 - g1).norm()) <= 1e-4 * float(g1.norm())


@pytest.mark.parametrize('name', ['resnet20_32', 'wrn16_4_dropout_32'])
def test_graph_replays_equal_eager(name):
    """6 chunked steps (B = 32, N = 3: two chunk shapes, each captured once): graph replays bit for bit eager"""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    cfg, px, classes = CONFIGS[name]
    g = torch.Generator().manual_seed(0)
    data = [(torch.randn(BATCH, 3, px, px, generator=g), torch.randint(0, classes, (BATCH,), generator=g))
            for _ in range(6)]
    fn = lambda: convert_b200(resnet(**cfg), 'cuda')     # noqa: E731
    l0, p0, tr = _run(fn, data, 3, use_graphs=True)
    assert tr.graph_replays == 6 * 3 - 2 * 2
    l1, p1, tr1 = _run(fn, data, 3, use_graphs=False)
    assert tr1.graph_replays == 0
    assert torch.equal(l0, l1), (l0, l1)
    assert torch.equal(p0, p1)


def test_launch_census():
    """one eager chunked step = N chunk train_steps + the launches of one optimizer step"""
    from convnet.pytorch_b200 import lib
    from convnet.pytorch_b200.utils.optim import OptimRegime
    x, y = _data('resnet20_32')
    model = _model('resnet20_32')
    tr = _trainer(model, opt=OptimRegime(model, copy.deepcopy(model.regime)))
    tr.use_graphs = False
    rt = model._b200
    up = torch.ones((), device='cuda')
    for _ in range(2):                       # warm-up of both shapes
        tr._step(x, y, training=True, chunk_batch=4)
        tr._step(x, y, training=True)
    torch.cuda.synchronize()

    def count(fn):
        n0 = lib.launch_count()
        fn()
        torch.cuda.synchronize()
        return lib.launch_count() - n0
    whole_step = count(lambda: tr._step(x, y, training=True))
    whole = count(lambda: rt.train_step(x, y, 0.0, up))
    chunk = count(lambda: rt.train_step(x[:8], y[:8], 0.0, up, reduce=False))
    chunked = count(lambda: tr._step(x, y, training=True, chunk_batch=4))
    optimizer = whole_step - whole
    assert optimizer > 0
    assert chunked == 4 * chunk + optimizer, (chunked, chunk, optimizer)
