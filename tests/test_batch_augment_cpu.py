"""Batch augmentation with Cutout (reference preprocess.py:44-54,105-112,159-161,185-227; trainer.py:17-29) on the CPU:
BatchAugment.apply and the torchvision transform against the SHA-256 of every copy the unmodified reference produced
(tests/golden/batch_augment.npz, written by tools/make_batch_augment_golden.py), the draw distributions, the
device-augmenting loader, the Trainer's non-fused paths, the unsupported combinations and the command line.  CPU only."""
import hashlib
import os

import numpy as np
import pytest
import torch
from scipy.stats import chisquare

from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'batch_augment.npz')


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


@pytest.fixture(scope='module')
def gold():
    z = np.load(GOLD)
    return {k: z[k] for k in z.files}


def _spec(gold, duplicates=None):
    return BatchAugment(padding=int(gold['padding']), cutout={'holes': int(gold['holes']), 'length': int(gold['length'])},
                        duplicates=duplicates or gold['draws'].shape[1])


def test_apply_reproduces_reference_copies(gold):
    images, draws = torch.from_numpy(gold['images']), torch.from_numpy(gold['draws'])
    out = _spec(gold).apply(images, draws)
    assert out.shape == (draws.shape[0] * draws.shape[1], 3, 32, 32) and out.dtype == torch.float32
    assert [_digest(c) for c in out] == list(gold['sha256'])
    # the fixture reaches the corners of the draw space (tools/make_batch_augment_golden.py selects its seed so)
    d = gold['draws']
    assert {0, 8} <= set(d[..., 0].ravel()) and {0, 8} <= set(d[..., 1].ravel()) and {0, 1} <= set(d[..., 2].ravel())
    assert (d[..., 3] == 0).any() and (d[..., 4] == 32).any() and (d[..., 5] == 0).any() and (d[..., 6] == 32).any()
    # cut elements are v * 0: signed zeros, both signs present (negative normalised values are cut too)
    zeros = out[out == 0]
    assert (torch.signbit(zeros)).any() and (~torch.signbit(zeros)).any()


def test_torchvision_path_with_cutout_reproduces_reference(gold):
    from PIL import Image
    from convnet.pytorch_b200.data import real_dataset_transform
    D = gold['draws'].shape[1]
    tf = real_dataset_transform('cifar10', augment=True, cutout={'holes': int(gold['holes']), 'length': int(gold['length'])},
                                duplicates=D)
    torch.manual_seed(int(gold['seed']))
    np.random.seed(int(gold['seed']))
    hashes = []
    for img in gold['images']:
        out = tf(Image.fromarray(img))
        assert out.shape == (D, 3, 32, 32)
        hashes.extend(_digest(c) for c in out)
    assert hashes == list(gold['sha256'])


def test_draw_distributions_are_uniform():
    torch.manual_seed(0)
    np.random.seed(0)
    spec = BatchAugment(padding=4, cutout={'holes': 1, 'length': 16}, duplicates=8)
    p = spec.sample(12500, 32, 32).reshape(-1, 7).numpy().astype(np.int64)       # 10^5 copies
    assert p.shape == (100000, 7)
    for col, k in ((0, 9), (1, 9), (2, 2)):
        counts = np.bincount(p[:, col], minlength=k)
        assert len(counts) == k and chisquare(counts).pvalue > 1e-3, (col, counts)
    # Cutout centres, recovered from the clipped boxes: y = y1 + L/2 unless the box was clipped at 0
    for lo, hi in ((3, 4), (5, 6)):
        centre = np.where(p[:, lo] > 0, p[:, lo] + 8, p[:, hi] - 8)
        counts = np.bincount(centre, minlength=32)
        assert len(counts) == 32 and chisquare(counts).pvalue > 1e-3
        assert ((p[:, hi] - p[:, lo]) <= 16).all() and (p[:, lo] >= 0).all() and (p[:, hi] <= 32).all()
    # without flip / cutout the table still has the flip column, always 0
    q = BatchAugment(padding=2, flip=False, duplicates=3).sample(5, 8, 8)
    assert q.shape == (5, 3, 3) and (q[..., 2] == 0).all() and int(q[..., :2].max()) <= 4


def test_apply_row_order_and_geometry():
    """Row b*D + d is copy d of image b; a non-square, non-32 image with C = 1 follows the reference formula."""
    g = torch.Generator().manual_seed(3)
    images = torch.randint(0, 256, (3, 6, 10, 1), generator=g, dtype=torch.uint8)
    spec = BatchAugment(padding=2, cutout={'holes': 2, 'length': 4}, duplicates=2, normalize={'mean': [0.5], 'std': [0.25]})
    params = torch.tensor([[2, 0, 1, 0, 2, 0, 2, 5, 6, 8, 10]] * 6, dtype=torch.int16).view(3, 2, 11)
    params[1, 1, :3] = torch.tensor([4, 4, 0])
    out = spec.apply(images, params)
    assert out.shape == (6, 1, 6, 10)
    for b in range(3):
        for d in range(2):
            oy, ox, flip = (int(v) for v in params[b, d, :3])
            lut = spec.lut(1)[0]
            for r in range(6):
                for c in range(10):
                    sy, sx = r + oy - 2, (9 - c if flip else c) + ox - 2
                    u = int(images[b, sy, sx, 0]) if 0 <= sy < 6 and 0 <= sx < 10 else 0
                    v = float(lut[u])
                    cut = (0 <= r < 2 and 0 <= c < 2) or (5 <= r < 6 and 8 <= c < 10)
                    assert float(out[b * 2 + d, 0, r, c]) == (v * 0.0 if cut else v)


def test_device_augment_loader_shapes():
    from convnet.pytorch_b200.data import DataRegime
    torch.manual_seed(0)
    reg = DataRegime(None, defaults={'name': 'synthetic_cifar10', 'split': 'train', 'augment': True, 'batch_size': 8,
                                     'shuffle': True, 'num_workers': 0, 'drop_last': True, 'duplicates': 4,
                                     'cutout': {'holes': 1, 'length': 16}, 'device_augment': True,
                                     'synthetic_length': 64})
    loader = reg.get_loader()
    batch, target = next(iter(loader))
    assert isinstance(batch, AugmentedBatch)
    assert batch.images.shape == (8, 32, 32, 3) and batch.images.dtype == torch.uint8
    assert batch.params.shape == (8, 4, 7) and batch.params.dtype == torch.int16
    assert batch.rows == 32 and target.shape == (32,) and target.dtype == torch.long
    assert torch.equal(target.view(8, 4), target.view(8, 4)[:, :1].expand(8, 4))        # row b*D + d has label b
    x = batch.apply()
    assert x.shape == (32, 3, 32, 32)
    assert torch.equal(x[4 * 5 + 2], batch.spec.apply(batch.images[5:6], batch.params[5:6])[2])
    # labels follow the images: every sample of the dataset appears with its own label
    ds = reg._data
    labels = {tuple(ds.images[i % len(ds.images)].flatten()[:16].tolist()): ds.labels[i] for i in range(len(ds))}
    for b in range(8):
        assert int(labels[tuple(batch.images[b].flatten()[:16].tolist())]) == int(target[4 * b])
    # evaluation loaders are unchanged: plain fp32 batches
    val = DataRegime(None, defaults={'name': 'synthetic_cifar10', 'split': 'val', 'augment': False, 'batch_size': 4,
                                     'num_workers': 0, 'synthetic_length': 8, 'device_augment': False})
    xv, yv = next(iter(val.get_loader()))
    assert xv.shape == (4, 3, 32, 32) and xv.dtype == torch.float32


def test_unsupported_combinations_raise():
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import DataRegime, real_dataset_transform
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    spec = BatchAugment(duplicates=2)
    g = torch.Generator().manual_seed(0)
    batch = AugmentedBatch(torch.randint(0, 256, (4, 32, 32, 3), generator=g, dtype=torch.uint8), spec.sample(4, 32, 32),
                           spec)
    y = torch.randint(0, 10, (8,), generator=g)
    torch.manual_seed(0)
    model = models.resnet(dataset='cifar10', depth=8)
    for kw, match in ((dict(mixup=0.2), 'mixup'), (dict(cutmix=1.0), 'mixup'), (dict(adapt_grad_norm=1), 'adapt_grad_norm')):
        tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device_ids=None, device='cpu', **kw)
        with pytest.raises(NotImplementedError, match=match):
            tr.train([(batch, y)])
    tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device_ids=None, device='cpu')
    with pytest.raises(NotImplementedError, match='average_output'):
        tr.train([(batch, y)], average_output=True)
    base = {'name': 'synthetic_cifar10', 'split': 'train', 'augment': True, 'batch_size': 4, 'num_workers': 0,
            'synthetic_length': 8, 'duplicates': 2, 'device_augment': True}
    with pytest.raises(NotImplementedError, match='resize'):          # the Mix&Match sampled_* CIFAR regimes
        DataRegime(None, defaults=dict(base, input_size=24, scale_size=32))
    with pytest.raises(NotImplementedError, match='CIFAR'):
        DataRegime(None, defaults=dict(base, name='synthetic_imagenet'))
    with pytest.raises(NotImplementedError, match='autoaugment'):
        DataRegime(None, defaults=dict(base, autoaugment=True))
    with pytest.raises(NotImplementedError, match='autoaugment'):
        real_dataset_transform('cifar10', autoaugment=True)
    with pytest.raises(NotImplementedError, match='multi-crop'):
        real_dataset_transform('cifar10', augment=False, num_crops=5)


@pytest.mark.parametrize('chunk_batch', [1, 2])
def test_trainer_cpu_trains_on_the_applied_batch(chunk_batch):
    """The non-fused paths train on AugmentedBatch.apply(): the same losses and parameters as the fp32 batch."""
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    spec = BatchAugment(cutout={'holes': 1, 'length': 16}, duplicates=3)
    g = torch.Generator().manual_seed(1)
    torch.manual_seed(1)
    batches = [(AugmentedBatch(torch.randint(0, 256, (4, 32, 32, 3), generator=g, dtype=torch.uint8),
                               spec.sample(4, 32, 32), spec), torch.randint(0, 10, (4,), generator=g).repeat_interleave(3))
               for _ in range(2)]
    results = []
    for form in ('aug', 'fp32'):
        torch.manual_seed(0)
        model = models.resnet(dataset='cifar10', depth=8)
        tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device_ids=None, device='cpu')
        data = batches if form == 'aug' else [(b.apply(), t) for b, t in batches]
        res = tr.train(data, chunk_batch=chunk_batch)
        results.append((res['loss'], torch.cat([p.detach().flatten() for p in model.parameters()])))
    assert results[0][0] == results[1][0] and torch.equal(results[0][1], results[1][1])


def test_cli_cpu_run_with_device_augment(tmp_path):
    """ResNet-20, synthetic CIFAR-10, CPU: --device-augment --duplicates 4 --cutout for one short epoch."""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 20}", '--dataset', 'synthetic_cifar10',
              '--device', 'cpu', '-b', '8', '--epochs', '1', '--max-steps', '2', '--workers', '0',
              '--duplicates', '4', '--cutout', '--device-augment',
              '--results-dir', str(tmp_path), '--save', 'aug'])
    import csv
    rows = list(csv.DictReader(open(tmp_path / 'aug' / 'results.csv')))
    assert len(rows) == 1 and float(rows[0]['training loss']) > 0
