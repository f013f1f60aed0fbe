"""RandomResizedCrop on the device, CPU side: the loader's per-image draws and ResizedCropBatch.apply() against the
unmodified reference transform (tests/golden/resized_crop.npz, written by tools/make_resized_crop_golden.py), the
ragged batch plumbing, the combinations that raise, and a short CPU run from the command line."""
import hashlib
import os

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import ResizedCrop, ResizedCropBatch, ResizedCropCollate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resized_crop.npz')


def test_draws_and_apply_match_the_reference_transform():
    from convnet.pytorch_b200.data import resized_crop_spec, synthetic_imagenet_pool
    g = np.load(GOLDEN)
    D, size = int(g['duplicates']), int(g['size'])
    images = synthetic_imagenet_pool()[:len(g['image_hw'])]
    assert [[im.size[1], im.size[0]] for im in images] == g['image_hw'].tolist()
    spec = resized_crop_spec('imagenet', input_size=size, duplicates=D)
    torch.manual_seed(int(g['seed']))
    samples = [(spec(img), k) for k, img in enumerate(images)]          # the worker's work, in the loader's order
    batch, target = ResizedCropCollate(spec)(samples)
    # draws back in image coordinates: region origin + box inside the region
    draws = []
    for b, ((reg, d), _) in enumerate(samples):
        img_draws = g['draws'][b * D:(b + 1) * D]
        y0, x0 = int(img_draws[:, 0].min()), int(img_draws[:, 1].min())
        got = d.numpy().copy()
        got[:, 0] += y0
        got[:, 1] += x0
        draws.append(got)
        assert reg.shape[:2] == (int((img_draws[:, 0] + img_draws[:, 2]).max()) - y0,
                                 int((img_draws[:, 1] + img_draws[:, 3]).max()) - x0)
    assert np.array_equal(np.concatenate(draws), g['draws'])
    out = batch.apply()
    assert out.shape == (len(images) * D, 3, size, size) and out.dtype == torch.float32
    hashes = [hashlib.sha256(c.contiguous().numpy().tobytes()).hexdigest() for c in out]
    assert hashes == g['sha256'].tolist()
    assert target.tolist() == [k for k in range(len(images)) for _ in range(D)]


def test_batch_packing_and_pin_memory_round_trip():
    from PIL import Image
    spec = ResizedCrop(32, duplicates=3)
    g = torch.Generator().manual_seed(0)
    imgs = [Image.fromarray(torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy(), 'RGB')
            for h, w in ((40, 50), (100, 30), (37, 64), (200, 210))]
    torch.manual_seed(1)
    samples = [(spec(im), 10 + k) for k, im in enumerate(imgs)]
    batch, target = ResizedCropCollate(spec)(samples)
    assert batch.rows == 12 and target.tolist() == [10, 10, 10, 11, 11, 11, 12, 12, 12, 13, 13, 13]
    assert batch.index.dtype == torch.int64 and batch.draws.dtype == torch.int32 and batch.regions.dim() == 1
    off = 0
    for b, ((reg, d), _) in enumerate(samples):
        o, h, w = batch.index[b].tolist()
        assert o == off and (h, w) == tuple(reg.shape[:2])
        assert torch.equal(batch.regions[o:o + h * w * 3].view(h, w, 3), reg)
        assert torch.equal(batch.draws[3 * b:3 * b + 3], d)
        # the region is the bounding box of the copies' crops: every box inside, every edge touched
        assert (d[:, 0] >= 0).all() and (d[:, 1] >= 0).all()
        assert (d[:, 0] + d[:, 2] <= h).all() and (d[:, 1] + d[:, 3] <= w).all()
        assert int(d[:, 0].min()) == 0 and int(d[:, 1].min()) == 0
        assert int((d[:, 0] + d[:, 2]).max()) == h and int((d[:, 1] + d[:, 3]).max()) == w
        off += h * w * 3
    assert off == batch.nbytes == batch.regions.numel()
    # pin_memory() and replace() keep every tensor and the host tables
    moved = batch.replace(tuple(t.clone() for t in batch.tensors))
    assert isinstance(moved, ResizedCropBatch) and moved.nbytes == batch.nbytes and moved.host[0] is batch.index
    assert torch.equal(moved.apply(), batch.apply())
    if torch.cuda.is_available():
        pinned = batch.pin_memory()
        assert all(t.is_pinned() for t in pinned.tensors) and torch.equal(pinned.apply(), batch.apply())


def test_loader_yields_ragged_batches():
    from convnet.pytorch_b200.data import DataRegime
    reg = DataRegime(None, defaults={'name': 'synthetic_imagenet', 'split': 'train', 'augment': True,
                                     'input_size': 64, 'batch_size': 4, 'num_workers': 0, 'synthetic_length': 16,
                                     'duplicates': 2, 'device_resized_crop': True, 'shuffle': False})
    batch, target = next(iter(reg.get_loader()))
    assert isinstance(batch, ResizedCropBatch) and batch.rows == 8 and target.shape == (8,)
    assert batch.spec.size == (64, 64) and batch.apply().shape == (8, 3, 64, 64)
    assert torch.equal(target[0::2], target[1::2])


def test_unsupported_combinations_raise():
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import DataRegime, resized_crop_spec
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    base = {'name': 'synthetic_imagenet', 'split': 'train', 'augment': True, 'input_size': 64, 'batch_size': 4,
            'num_workers': 0, 'synthetic_length': 8, 'device_resized_crop': True}
    for extra, match in ((dict(cutout={'holes': 1, 'length': 16}), 'Cutout'), (dict(autoaugment=True), 'autoaugment'),
                         (dict(augment=False), 'training transform'), (dict(device_augment=True), 'device_augment'),
                         (dict(name='synthetic_cifar10'), 'ImageNet')):
        with pytest.raises(NotImplementedError, match=match):
            DataRegime(None, defaults=dict(base, **extra))
    with pytest.raises(NotImplementedError, match='bilinear'):
        resized_crop_spec('imagenet', interpolation='bicubic')
    with pytest.raises(NotImplementedError, match='colour jitter'):
        resized_crop_spec('imagenet', color_jitter=0.4)
    with pytest.raises(NotImplementedError, match='cifar10'):
        DataRegime(None, defaults=dict(base, name='cifar10', transform_name='imagenet'))
    spec = ResizedCrop(32, duplicates=2)
    from PIL import Image
    torch.manual_seed(0)
    img = Image.fromarray(np.zeros((40, 40, 3), np.uint8), 'RGB')
    batch, y = ResizedCropCollate(spec)([(spec(img), 1), (spec(img), 2)])
    torch.manual_seed(0)
    model = models.resnet(dataset='imagenet', depth=18)
    for kw, match in ((dict(mixup=0.2), 'mixup'), (dict(cutmix=1.0), 'mixup'), (dict(adapt_grad_norm=1), 'adapt_grad_norm')):
        tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device_ids=None, device='cpu', **kw)
        with pytest.raises(NotImplementedError, match=match):
            tr.train([(batch, y)])
    tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device_ids=None, device='cpu')
    with pytest.raises(NotImplementedError, match='average_output'):
        tr.train([(batch, y)], average_output=True)


def test_cli_cpu_run_with_device_resized_crop(tmp_path):
    """ResNet-18, synthetic ImageNet at 64 px, CPU: --device-resized-crop for two steps."""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 18}", '--dataset', 'synthetic_imagenet',
              '--device', 'cpu', '-b', '4', '--epochs', '1', '--max-steps', '2', '--workers', '0',
              '--input-size', '64', '--device-resized-crop', '--results-dir', str(tmp_path), '--save', 'rrc'])
    import csv
    rows = list(csv.DictReader(open(tmp_path / 'rrc' / 'results.csv')))
    assert len(rows) == 1 and float(rows[0]['training loss']) > 0
