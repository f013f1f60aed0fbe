"""Batch augmentation on the kernel path: the augmenting relayout (b200_input_prep_u8_aug) against
b200_input_prep of BatchAugment.apply, bit for bit, and whole Trainer runs fed an AugmentedBatch against the same runs
fed the applied fp32 batch, with CUDA-graph replays that must follow each step's draws."""
import copy

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment

pytestmark = pytest.mark.gpu

GUARD = 4096


def _hand_draws(n_rows, H, W, pad, holes, wild=False):
    """int16 [n_rows, 3 + 4*holes]: cycles through crop offsets (0,0), (2p,2p) and mixed, both flips, and Cutout boxes
    clipped at a corner, at each edge, interior and empty.  ``wild``: offsets, flips and boxes far outside their
    ranges (the kernel must treat any values safely: out-of-image pixels read the pad value)."""
    offs = [(0, 0), (2 * pad, 2 * pad), (0, 2 * pad), (2 * pad, 0), (pad, 1), (1, pad)]
    boxes = [(0, H // 4, 0, W // 4), (0, H // 2, W // 3, W // 2), (H // 2, H, 1, W // 3), (1, H // 3, 0, W // 2),
             (H // 3, H // 2, W // 2, W), (H - 1, H, W - 2, W), (H // 3, H // 3, 2, 5), (2, H - 2, 3, W - 1)]
    rows = []
    for n in range(n_rows):
        oy, ox = offs[n % len(offs)]
        row = [oy, ox, (n // len(offs)) % 2]
        for h in range(holes):
            row += list(boxes[(n + 3 * h) % len(boxes)])
        if wild and n % 3 == 0:
            row[:3] = [-700 + n, 3000 - 5 * n, 7]
            if holes:
                row[3:7] = [-9, 30000, -20000, W // 2]
        rows.append(row)
    return torch.tensor(rows, dtype=torch.int16)


CASES = [  # B, D, C, H, W, Cpad, pad, holes, wild
    (5, 3, 3, 32, 32, 16, 4, 1, False),
    (3, 40, 3, 32, 32, 16, 4, 1, False),
    (7, 1, 1, 12, 20, 8, 2, 2, False),
    (4, 3, 3, 24, 16, 8, 3, 0, False),
    (3, 4, 3, 32, 32, 16, 4, 2, False),
    (2, 5, 3, 18, 30, 16, 5, 1, True),
]


@pytest.mark.parametrize('B,D,C,H,W,cpad,pad,holes,wild', CASES)
def test_input_prep_u8_aug_is_exact(B, D, C, H, W, cpad, pad, holes, wild):
    from convnet.pytorch_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + D)
    images = torch.randint(0, 256, (B, H, W, C), generator=g, dtype=torch.uint8)
    stats = {'mean': [0.485, 0.456, 0.406][:C], 'std': [0.229, 0.224, 0.225][:C]}
    spec = BatchAugment(padding=pad, cutout={'holes': holes, 'length': 8} if holes else None, duplicates=D,
                        normalize=stats)
    params = _hand_draws(B * D, H, W, pad, holes, wild)
    want = ops.input_prep(spec.apply(images, params).cuda(), cpad)
    aug = ops.Aug(params.cuda(), spec.lut(C).cuda(), D, pad)
    n = B * D * H * W * cpad
    outs = []
    for _ in range(2):
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=torch.bfloat16, device='cuda')
        out = buf[GUARD:GUARD + n].view(B * D, H, W, cpad)
        ops.input_prep_u8_aug(images.cuda(), cpad, aug, out=out)
        torch.cuda.synchronize()
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + n:].float()).all(), 'wrote outside'
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)), 'differs from input_prep(apply())'
        outs.append(out.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    if holes and not wild:
        assert (out.view(torch.int16) == -32768).any(), 'expected cut negative values (-0.0)'


def test_input_prep_u8_aug_rejects_bad_arguments():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    spec = BatchAugment(duplicates=2)
    x = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device='cuda')
    good = ops.Aug(torch.zeros((4, 3), dtype=torch.int16, device='cuda'), spec.lut(3).cuda(), 2, 4)
    ops.input_prep_u8_aug(x, 8, good)
    for bad in (ops.Aug(good.params[:3], good.lut, 2, 4),                             # rows != N*D
                ops.Aug(torch.zeros((4, 5), dtype=torch.int16, device='cuda'), good.lut, 2, 4),   # 3 + 4*holes
                ops.Aug(good.params, good.lut[:1], 2, 4),                              # LUT channels
                ops.Aug(good.params.int(), good.lut, 2, 4)):                           # dtype
        with pytest.raises(B200Error):
            ops.input_prep_u8_aug(x, 8, bad)
    with pytest.raises(B200Error, match='Cpad'):
        ops.input_prep_u8_aug(x, 12, good)
    with pytest.raises(B200Error, match='pad'):
        ops.input_prep_u8_aug(x, 8, ops.Aug(good.params, good.lut, 2, -1))


def test_trainer_device_augment_matches_applied_batch_bitwise():
    """ResNet-20, B=16, D=4, Cutout: one Trainer fed AugmentedBatch (prefetched, augmented in the relayout kernel), one
    fed the fp32 batch of apply() with the expanded targets; identical starting state.  6 steps with fresh draws, the
    last 4 replayed from captured graphs: every step's loss and the final arena parameters are bit-identical."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.cuda.set_device(0)
    spec = BatchAugment(padding=4, cutout={'holes': 1, 'length': 16}, duplicates=4)
    g = torch.Generator().manual_seed(0)
    torch.manual_seed(5)
    np.random.seed(5)
    batches = []
    for _ in range(6):
        images = torch.randint(0, 256, (16, 32, 32, 3), generator=g, dtype=torch.uint8)
        batches.append((AugmentedBatch(images, spec.sample(16, 32, 32), spec),
                        torch.randint(0, 10, (16,), generator=g).repeat_interleave(4)))
    assert len({b.params.numpy().tobytes() for b, _ in batches}) == 6
    runs = []
    for form in ('aug', 'fp32'):
        torch.manual_seed(123)
        model = convert_b200(resnet(dataset='cifar10', depth=20), 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9)
        losses, step = [], tr._step

        def recording_step(inputs, target, **kw):
            out, loss, grad = step(inputs, target, **kw)
            losses.append(loss.detach().clone())
            return out, loss, grad
        tr._step = recording_step
        data = batches if form == 'aug' else [(b.apply(), t) for b, t in batches]
        res = tr.train(data)
        torch.cuda.synchronize()
        assert tr.graph_replays == 4
        runs.append((torch.stack(losses).cpu(), model._b200.arena.p32.detach().clone().cpu(), res))
    (l0, p0, r0), (l1, p1, r1) = runs
    assert torch.equal(l0, l1), (l0, l1)
    assert torch.equal(p0, p1)
    assert r0['loss'] == r1['loss'] and r0['prec1'] == r1['prec1']
