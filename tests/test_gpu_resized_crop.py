"""RandomResizedCrop on the kernel path: the resized-crop relayout (b200_input_prep_u8_rrc) against b200_input_prep of
ResizedCropBatch.apply() -- torchvision's own PIL transform -- bit for bit, and whole Trainer runs fed a
ResizedCropBatch against the same runs fed the applied fp32 batch, with CUDA-graph replays that must follow each step's
regions and draws."""
import copy

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import ResizedCrop, ResizedCropBatch

pytestmark = pytest.mark.gpu

GUARD = 4096


def _batch(sizes, boxes, D, C, size, seed):
    """ResizedCropBatch of uniform regions of ``sizes`` [(h, w)] and hand-chosen ``boxes`` [B*D x (y, x, h, w, flip)]."""
    g = torch.Generator().manual_seed(seed)
    regions = [torch.randint(0, 256, (h, w, C), generator=g, dtype=torch.uint8) for h, w in sizes]
    offsets = np.cumsum([0] + [r.numel() for r in regions[:-1]]).tolist()
    index = torch.tensor([[o, h, w] for o, (h, w) in zip(offsets, sizes)], dtype=torch.int64)
    draws = torch.tensor(boxes, dtype=torch.int32)
    stats = {'mean': [0.485, 0.456, 0.406][:C], 'std': [0.229, 0.224, 0.225][:C]}
    spec = ResizedCrop(size, duplicates=D, normalize=stats)
    return ResizedCropBatch(torch.cat([r.reshape(-1) for r in regions]), index, draws, spec, C)


def _rrc(batch):
    from convnet.pytorch_b200 import ops
    return ops.Rrc(batch.index.cuda(), batch.draws.cuda(), batch.spec.lut(batch.channels).cuda(),
                   batch.spec.duplicates, batch.spec.size, (batch.index, batch.draws, batch.nbytes))


def _cases():
    S = 224
    return [  # name, sizes, boxes (B*D rows), D, C, size, cpad, s2d
        ('identity-and-whole', [(S, S), (300, 260), (S, 400)],
         [(0, 0, S, S, 0), (0, 0, 300, 260, 1), (0, 3, S, 397, 0)], 1, 3, S, 16, True),      # exact OH and/or OW
        ('upscale', [(40, 90), (150, 30), (17, 13)],
         [(3, 5, 30, 80, 1), (10, 2, 130, 20, 0), (0, 0, 17, 13, 1)], 1, 3, S, 8, False),
        ('downscale-many-taps', [(1600, 1700), (2000, 300)],
         [(0, 0, 1600, 1700, 0), (7, 0, 1990, 290, 1)], 1, 3, S, 16, True),                  # 15 and 19+ taps
        ('thin', [(50, 60), (1, 70), (80, 1)],
         [(4, 20, 40, 1, 0), (0, 0, 1, 70, 1), (0, 0, 80, 1, 1)], 1, 1, 128, 8, False),   # 1-px crops
        ('d2-odd-b', [(120, 100), (90, 200), (64, 64)],
         [(0, 0, 120, 100, 0), (30, 10, 50, 60, 1), (5, 40, 80, 150, 1), (0, 0, 90, 200, 0),
          (0, 0, 64, 64, 1), (10, 20, 30, 40, 0)], 2, 3, 288, 16, False),
        ('d5', [(300, 400), (250, 180)],
         [(0, 0, 300, 400, 0), (10, 20, 200, 100, 1), (100, 300, 150, 100, 0), (0, 0, 1, 1, 1), (299, 0, 1, 400, 0),
          (0, 0, 250, 180, 1), (40, 30, 100, 100, 0), (3, 7, 64, 64, 1), (200, 100, 50, 80, 0), (0, 179, 250, 1, 1)],
         5, 3, 64, 16, True),
        ('c1-mode2', [(100, 140)], [(20, 30, 60, 90, 1)], 1, 1, 64, 16, True),
        ('huge-downscale', [(2100, 2300)], [(0, 0, 2100, 2300, 1)], 1, 3, 64, 8, False),     # 65+ taps: slab chunks
    ]


@pytest.mark.parametrize('name,sizes,boxes,D,C,size,cpad,s2d', _cases(), ids=[c[0] for c in _cases()])
def test_input_prep_u8_rrc_is_exact(name, sizes, boxes, D, C, size, cpad, s2d):
    from convnet.pytorch_b200 import ops
    batch = _batch(sizes, boxes, D, C, size, seed=len(boxes) * 7 + C)
    want = ops.input_prep(batch.apply().cuda(), cpad, s2d=s2d, border=s2d)
    rrc = _rrc(batch)
    regions = batch.regions.cuda()
    n = want.numel()
    outs = []
    for _ in range(2):
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=torch.bfloat16, device='cuda')
        out = buf[GUARD:GUARD + n].view(want.shape)
        ops.input_prep_u8_rrc(regions, cpad, rrc, s2d=s2d, border=s2d, out=out)
        torch.cuda.synchronize()
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + n:].float()).all(), 'wrote outside'
        assert not torch.isnan(out.float()).any(), 'left elements unwritten'
        bad = (out.view(torch.int16) != want.view(torch.int16))
        assert not bad.any(), 'differs from input_prep(apply()) at %d elements, first %s' % (
            int(bad.sum()), bad.nonzero()[0].tolist())
        outs.append(out.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))


def test_input_prep_u8_rrc_rejects_bad_tables():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    batch = _batch([(40, 50), (30, 30)], [(0, 0, 40, 50, 0), (1, 2, 20, 20, 1)], 1, 3, 32, seed=0)
    regions = batch.regions.cuda()
    ops.input_prep_u8_rrc(regions, 16, _rrc(batch))
    bad_draws = [(0, 0, 41, 50, 0), (0, 45, 10, 6, 0), (-1, 0, 10, 10, 0), (0, 0, 0, 10, 0), (0, 0, 10, 10, 2)]
    for row in bad_draws:
        d = batch.draws.clone()
        d[0] = torch.tensor(row, dtype=torch.int32)
        b = ResizedCropBatch(batch.regions, batch.index, d, batch.spec, 3)
        with pytest.raises(B200Error, match='crop box'):
            ops.input_prep_u8_rrc(regions, 16, _rrc(b))
    for row in ((6001, 30, 30), (-1, 30, 30), (0, 0, 30), (0, 100, 50)):
        ix = batch.index.clone()
        ix[1] = torch.tensor(row)
        b = ResizedCropBatch(batch.regions, ix, batch.draws, batch.spec, 3)
        with pytest.raises(B200Error, match='region'):
            ops.input_prep_u8_rrc(regions, 16, _rrc(b))
    with pytest.raises(B200Error, match='Cpad'):
        ops.input_prep_u8_rrc(regions, 12, _rrc(batch))
    with pytest.raises(B200Error, match='border'):
        ops.input_prep_u8_rrc(regions, 16, _rrc(batch), s2d=True, border=False)


def _random_batches(steps, B, D, size, seed):
    """ResizedCropBatches of seeded PIL-sized images through the loader's own per-image draw (ResizedCrop.__call__)."""
    from PIL import Image
    from convnet.pytorch_b200.utils.augment import ResizedCropCollate
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


def _run_pair(model_fn, batches, expect_replays):
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.cuda.set_device(0)
    runs = []
    for form in ('rrc', 'fp32'):
        torch.manual_seed(123)
        model = convert_b200(model_fn(), 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9)
        losses, step = [], tr._step

        def recording_step(inputs, target, **kw):
            out, loss, grad = step(inputs, target, **kw)
            losses.append(loss.detach().clone())
            return out, loss, grad
        tr._step = recording_step
        data = batches if form == 'rrc' else [(b.apply(), t) for b, t in batches]
        tr.train(data)
        torch.cuda.synchronize()
        assert tr.graph_replays == expect_replays
        runs.append((torch.stack([x.reshape(-1)[0] for x in losses]).cpu(),
                     model._b200.arena.p32.detach().clone().cpu()))
    (l0, p0), (l1, p1) = runs
    assert torch.equal(l0, l1), (l0, l1)
    assert torch.equal(p0, p1)


def test_trainer_resnet18_resized_crop_matches_applied_batch_bitwise():
    """ResNet-18 (mode-2 space-to-depth stem), 64 px, B=8, D=2: 6 steps with fresh regions and draws, the last 4
    replayed from a captured graph; losses and final arena parameters bit-identical to the fp32 batch of apply()."""
    from convnet.pytorch_b200.models import resnet
    batches = _random_batches(6, 8, 2, 64, seed=1)
    assert len({b.draws.numpy().tobytes() for b, _ in batches}) == 6
    _run_pair(lambda: resnet(dataset='imagenet', depth=18), batches, 4)


def test_trainer_mobilenet_v2_resized_crop_matches_applied_batch_bitwise():
    """MobileNet-v2 (mode-0 3x3/s2 stem), 3 steps (one replay)."""
    from convnet.pytorch_b200.models import mobilenet_v2

    def factory():
        m = mobilenet_v2(dataset='imagenet')
        m.classifier[0].p = 0.0
        return m
    _run_pair(factory, _random_batches(3, 4, 1, 64, seed=2), 1)


def test_trainer_alternating_sizes_keep_their_graphs():
    """Mix&Match: two input sizes alternate; each size captures its own graph and every step stays bit-identical."""
    from convnet.pytorch_b200.models import resnet
    a, b = _random_batches(4, 4, 1, 64, seed=3), _random_batches(4, 4, 1, 96, seed=4)
    batches = [x for pair in zip(a, b) for x in pair]
    _run_pair(lambda: resnet(dataset='imagenet', depth=18), batches, 4)
