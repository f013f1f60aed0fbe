"""The Mix&Match CIFAR size regimes on the kernel path: the resizing relayout (b200_input_prep_u8_aug_resize) against
b200_input_prep of BatchAugment(resize=...).apply -- torchvision's own PIL transform -- bit for bit, the copies of the
unmodified reference transform (tests/golden/mixsize_augment.npz), the argument checks, and whole Trainer runs over the
four ``sampled_D+`` configurations fed AugmentedBatches against the same runs fed the applied fp32 batches, captured
graphs against eager launches."""
import collections
import copy
import os

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment

pytestmark = pytest.mark.gpu

GUARD = 4096
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mixsize_augment.npz')


def _hand_draws(n_rows, OH, OW, pad, holes, wild=False):
    """int16 [n_rows, 3 + 4*holes]: cycles through crop offsets (0,0), (2p,2p) and mixed, both flips, and Cutout boxes
    (output coordinates) clipped at a corner, at each edge, interior and empty.  ``wild``: offsets, flips and boxes far
    outside their ranges (any values are safe: pixels outside the image read the fill, boxes are intersected)."""
    offs = [(0, 0), (2 * pad, 2 * pad), (0, 2 * pad), (2 * pad, 0), (pad, 1), (1, pad)]
    H, W = OH, OW
    boxes = [(0, H // 4, 0, W // 4), (0, H // 2, W // 3, W // 2), (H // 2, H, 1, W // 3), (1, H // 3, 0, W // 2),
             (H // 3, H // 2, W // 2, W), (H - 1, H, W - 2, W), (H // 3, H // 3, 2, 5), (2, H - 2, 3, W - 1)]
    rows = []
    for n in range(n_rows):
        oy, ox = offs[n % len(offs)]
        row = [oy, ox, (n // len(offs)) % 2]
        for h in range(holes):
            row += list(boxes[(n + 3 * h) % len(boxes)])
        if wild and n % 3 == 0:
            row[:3] = [-700 + n, 3000 - 5 * n, 7] if n % 2 else [-3 - n, 2 * pad + 5, 1]
            if holes:
                row[3:7] = [-9, 30000, -20000, W // 2]
        rows.append(row)
    return torch.tensor(rows, dtype=torch.int16)


CASES = [  # B, D, C, H, W, OH, OW, Cpad, pad, holes, wild
    (16, 4, 3, 32, 32, 16, 16, 16, 4, 1, False),      # the three resizing configurations of sampled_D+
    (16, 2, 3, 32, 32, 24, 24, 16, 4, 0, False),
    (7, 1, 3, 32, 32, 48, 48, 16, 4, 1, False),
    (7, 3, 3, 32, 32, 32, 32, 16, 4, 2, False),       # scale 1: the identity
    (5, 2, 1, 32, 32, 40, 40, 8, 0, 1, False),
    (3, 4, 4, 32, 32, 64, 64, 8, 4, 2, False),
    (7, 3, 3, 28, 36, 20, 50, 16, 4, 1, False),       # non-square source, down in one axis and up in the other
    (3, 1, 3, 64, 64, 128, 128, 8, 4, 0, False),      # the limits
    (2, 2, 4, 64, 64, 7, 5, 8, 3, 1, False),          # many taps per output
    (4, 3, 3, 32, 32, 24, 24, 24, 4, 2, True),
]


@pytest.mark.parametrize('B,D,C,H,W,OH,OW,cpad,pad,holes,wild', CASES)
def test_input_prep_u8_aug_resize_is_exact(B, D, C, H, W, OH, OW, cpad, pad, holes, wild):
    from convnet.pytorch_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + D * 10 + C)
    images = torch.randint(0, 256, (B, H, W, C), generator=g, dtype=torch.uint8)
    stats = {'mean': [0.485, 0.456, 0.406, 0.5][:C], 'std': [0.229, 0.224, 0.225, 0.25][:C]}
    spec = BatchAugment(padding=pad, cutout={'holes': holes, 'length': 8} if holes else None, duplicates=D,
                        normalize=stats, resize=(OH, OW))
    params = _hand_draws(B * D, OH, OW, pad, holes, wild)
    want = ops.input_prep(spec.apply(images, params).cuda(), cpad)
    aug = ops.Aug(params.cuda(), spec.lut(C).cuda(), D, pad, (OH, OW))
    n = B * D * OH * OW * cpad
    outs = []
    for _ in range(2):
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=torch.bfloat16, device='cuda')
        out = buf[GUARD:GUARD + n].view(B * D, OH, OW, cpad)
        ops.input_prep_u8_aug(images.cuda(), cpad, aug, out=out)
        torch.cuda.synchronize()
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + n:].float()).all(), 'wrote outside'
        assert torch.equal(out.view(torch.int16), want.view(torch.int16)), 'differs from input_prep(apply())'
        outs.append(out.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
    assert (out[..., C:].view(torch.int16) == 0).all(), 'padded channels must be +0'
    if holes and not wild:
        assert (out.view(torch.int16) == -32768).any(), 'expected cut negative values (-0.0)'
    if (OH, OW) == (H, W):
        plain = ops.input_prep_u8_aug(images.cuda(), cpad, ops.Aug(aug.params, aug.lut, D, pad))
        assert torch.equal(out.view(torch.int16), plain.view(torch.int16)), 'scale 1 differs from the plain relayout'


@pytest.mark.parametrize('size', [16, 24, 48])
def test_reference_copies_from_the_device(size):
    """The draws the unmodified reference transform made: the kernel's copies are its fp32 copies rounded to bf16."""
    from convnet.pytorch_b200 import ops
    z = np.load(GOLD)
    images, draws = torch.from_numpy(z['images']), torch.from_numpy(z['draws_%d' % size])
    holes, length = (int(v) for v in z['cutout_%d' % size])
    spec = BatchAugment(padding=int(z['padding']), cutout={'holes': holes, 'length': length} if holes else None,
                        duplicates=draws.shape[1], resize=size)
    want = spec.apply(images, draws)              # pinned to the fixture's digests by test_mixsize_augment_cpu.py
    aug = ops.Aug(draws.reshape(-1, draws.shape[-1]).cuda(), spec.lut(3).cuda(), spec.duplicates, spec.padding,
                  spec.resize)
    out = ops.input_prep_u8_aug(images.cuda(), 16, aug)
    assert out.shape == (want.shape[0], size, size, 16)
    got = out[..., :3].permute(0, 3, 1, 2).float().cpu()
    assert torch.equal(got, want.to(torch.bfloat16).float())
    assert (out[..., 3:] == 0).all()


def test_input_prep_u8_aug_resize_rejects_bad_arguments():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    spec = BatchAugment(duplicates=2)
    x = torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device='cuda')
    params, lut = torch.zeros((4, 3), dtype=torch.int16, device='cuda'), spec.lut(3).cuda()
    good = ops.Aug(params, lut, 2, 4, (12, 12))
    assert ops.input_prep_u8_aug(x, 8, good).shape == (4, 12, 12, 8)
    for bad in (ops.Aug(params[:3], lut, 2, 4, (12, 12)),                                            # rows != N*D
                ops.Aug(torch.zeros((4, 5), dtype=torch.int16, device='cuda'), lut, 2, 4, (12, 12)),   # 3 + 4*holes
                ops.Aug(params, lut[:1], 2, 4, (12, 12)),                                              # LUT channels
                ops.Aug(params.int(), lut, 2, 4, (12, 12))):                                           # dtype
        with pytest.raises(B200Error):
            ops.input_prep_u8_aug(x, 8, bad)
    with pytest.raises(B200Error, match='Cpad'):
        ops.input_prep_u8_aug(x, 12, good)
    with pytest.raises(B200Error, match='pad'):
        ops.input_prep_u8_aug(x, 8, ops.Aug(params, lut, 2, -1, (12, 12)))
    with pytest.raises(B200Error, match='bad argument'):
        ops.input_prep_u8_aug(x, 8, ops.Aug(params, lut, 2, 4, (0, 12)))
    with pytest.raises(B200Error, match='above'):                                      # outputs above 128 px
        ops.input_prep_u8_aug(x, 8, ops.Aug(params, lut, 2, 4, (12, 129)))
    with pytest.raises(B200Error, match='above'):                                      # sources above 64 px
        ops.input_prep_u8_aug(torch.zeros((2, 65, 8, 3), dtype=torch.uint8, device='cuda'), 8, good)
    with pytest.raises(B200Error, match='out has shape'):
        ops.input_prep_u8_aug(x, 8, good, out=torch.empty((4, 8, 8, 8), dtype=torch.bfloat16, device='cuda'))
    # the output size is part of what a captured step is keyed by
    assert good.key != ops.Aug(params, lut, 2, 4, (16, 16)).key and good.key != ops.Aug(params, lut, 2, 4).key
    assert good.with_tables((params.clone(),)).key == good.key


class FakeCIFAR10(object):
    """Stands in for torchvision.datasets.CIFAR10 (no dataset files here): seeded uniform uint8 ``data`` [1280, 32, 32,
    3] and ``targets``, which is all device augmentation reads of it."""

    def __init__(self, root=None, train=True, download=False):
        g = torch.Generator().manual_seed(0 if train else 1)
        self.data = torch.randint(0, 256, (1280, 32, 32, 3), generator=g, dtype=torch.uint8).numpy()
        self.targets = torch.randint(0, 10, (1280,), generator=g).tolist()


def _sampled_batches(seed):
    """The batches one epoch of the ``sampled_D+`` CIFAR-10 regime yields with device augmentation."""
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import DataRegime, SampledDataRegime
    torch.manual_seed(seed)
    np.random.seed(seed)
    probs, configs = zip(*models.resnet(dataset='cifar10', depth=8, regime='sampled_D+').sampled_data_regime)
    defaults = {'name': 'cifar10', 'split': 'train', 'augment': True, 'shuffle': True, 'num_workers': 0,
                'drop_last': True, 'device_augment': True, 'cutout': {'holes': 1, 'length': 8}}
    data = SampledDataRegime([DataRegime(None, defaults={**defaults, **c}) for c in configs], probs)
    data.set_epoch(0)
    return list(data.get_loader())


def test_trainer_sampled_regime_matches_applied_batches_bitwise(monkeypatch):
    """ResNet-20 with the ``sampled_D+`` regime (GradSmooth, 32 / 48 / 24 / 16 px, duplicates 1 / 1 / 2 / 4): one
    Trainer fed the AugmentedBatches (augmented and resized in the relayout kernel) with captured graphs, one with eager
    launches, one fed the fp32 batches of apply(); identical starting state.  Every step's loss and the final arena
    parameters are bit-identical, and every size replays its own graph."""
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.cuda.set_device(0)
    import torchvision.datasets as tvd
    monkeypatch.setattr(tvd, 'CIFAR10', FakeCIFAR10)
    batches = _sampled_batches(seed=7)
    steps = collections.Counter((b.spec.resize or (32, 32))[0] for b, _ in batches)
    assert set(steps) == {16, 24, 32, 48} and min(steps.values()) >= 3, steps
    assert {(b.spec.resize or (32, 32))[0]: b.rows for b, _ in batches} == {32: 64, 48: 28, 24: 128, 16: 256}
    calls = collections.Counter()
    prep = ops.input_prep_u8_aug

    def counting_prep(x, cpad, aug, **kw):
        calls[aug.out_hw] += 1
        return prep(x, cpad, aug, **kw)
    monkeypatch.setattr(ops, 'input_prep_u8_aug', counting_prep)
    runs = []
    for form in ('aug', 'aug-eager', 'fp32'):
        torch.manual_seed(123)
        model = convert_b200(resnet(dataset='cifar10', depth=20, regime='sampled_D+'), 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9)
        tr.use_graphs = form != 'aug-eager'
        losses, step = [], tr._step

        def recording_step(inputs, target, **kw):
            out, loss, grad = step(inputs, target, **kw)
            losses.append(loss.detach().clone())
            return out, loss, grad
        tr._step = recording_step
        calls.clear()
        tr.train(batches if form != 'fp32' else [(b.apply(), t) for b, t in batches])
        torch.cuda.synchronize()
        if form == 'fp32':
            assert not calls
        else:       # the relayout kernel made the copies: every eager step of every size passed through it
            assert set(calls) == {None, (48, 48), (24, 24), (16, 16)}
            assert sum(calls.values()) == (len(batches) if form == 'aug-eager' else 4 * 3)   # 2 warm-ups + the capture
        assert tr.graph_replays == (0 if form == 'aug-eager' else len(batches) - 8)
        runs.append((torch.stack([x.reshape(-1)[0] for x in losses]).cpu(),
                     model._b200.arena.p32.detach().clone().cpu()))
    for losses, params in runs[1:]:
        assert torch.equal(runs[0][0], losses), (runs[0][0], losses)
        assert torch.equal(runs[0][1], params)


def test_resizing_step_adds_library_kernels_only():
    """Profiler traces of fused train_steps on 16 uint8 images resized to 24 px, 2 copies each, and of the same steps
    on the applied fp32 batch: the first runs the resizing relayout in place of the fp32 one and no kernel outside the
    library that the second does not run.  Two steps per trace, and the relayout -- the first kernel of a step -- is
    only required to appear: a trace may miss the kernels launched right after it starts."""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    torch.cuda.set_device(0)
    torch.manual_seed(3)
    np.random.seed(3)
    spec = BatchAugment(cutout={'holes': 1, 'length': 8}, duplicates=2, resize=24)
    g = torch.Generator().manual_seed(3)
    batch = AugmentedBatch(torch.randint(0, 256, (16, 32, 32, 3), generator=g, dtype=torch.uint8),
                           spec.sample(16, 32, 32), spec)
    y = torch.randint(0, 10, (16,), generator=g).repeat_interleave(2).cuda()
    aug = ops.Aug(batch.params.reshape(-1, 7).cuda(), spec.lut(3).cuda(), 2, 4, spec.resize)
    model = convert_b200(resnet(dataset='cifar10', depth=20), 'cuda')
    model.train()
    rt = model._b200
    traces = []
    for x, kw in ((batch.images.cuda(), dict(aug=aug)), (batch.apply().cuda(), {})):
        rt.train_step(x, y, **kw)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(2):
                rt.train_step(x, y, **kw)
            torch.cuda.synchronize()
        traces.append({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    fused, plain = traces

    def other(names):
        return {n for n in names if 'b200::' not in n and 'memset' not in n.lower()}
    assert len(fused) > 10 and other(fused) <= other(plain), other(fused) - other(plain)
    assert any('input_prep_aug_resize_kernel' in n for n in fused), sorted(fused)
    assert not any('input_prep_aug_resize_kernel' in n for n in plain)
    assert not any('input_prep_kernel' in n for n in fused) and any('input_prep_kernel' in n for n in plain)
