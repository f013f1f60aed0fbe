"""Resize + CenterCrop on the device, CPU side: ScaleCropBatch.apply() against the unmodified reference evaluation
transform (tests/golden/scale_crop.npz, written by tools/make_scale_crop_golden.py), the loader's host geometry against
torchvision's own functions, the host-side table validation, batch packing, the settings that raise, and a short CPU
run from the command line."""
import hashlib
import os

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import ScaleCrop, ScaleCropBatch, ScaleCropCollate

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'scale_crop.npz')


def _image(h, w, mode, seed):
    """the fixture's images: uniform uint8 from torch.Generator(seed), 3 channels for RGB, 1 for L"""
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    c = 3 if mode == 'RGB' else 1
    a = torch.randint(0, 256, (h, w, c), generator=g, dtype=torch.uint8).numpy()
    return Image.fromarray(a if c == 3 else a[:, :, 0], mode)


def _stats(c):
    return {'mean': [0.485, 0.456, 0.406][:c], 'std': [0.229, 0.224, 0.225][:c]}


def golden_cases():
    """[(input_size, scale_size, PIL image, sha256)] of the fixture"""
    g = np.load(GOLDEN)
    return [(int(s), int(sc), _image(int(h), int(w), str(m), int(seed)), str(d))
            for (s, sc, h, w), m, seed, d in zip(g['cases'], g['modes'], g['seeds'], g['sha256'])]


def test_apply_matches_the_reference_transform():
    from convnet.pytorch_b200.data import scale_crop_spec
    cases = golden_cases()
    assert len(cases) == 14
    for size, scale, img, digest in cases:
        c = len(img.getbands())
        spec = scale_crop_spec('imagenet', input_size=size, scale_size=scale, normalize=_stats(c))
        batch, target = ScaleCropCollate(spec)([(spec(img), 7)])
        out = batch.apply()
        assert out.shape == (1, c, size, size) and out.dtype == torch.float32 and target.tolist() == [7]
        assert hashlib.sha256(out[0].contiguous().numpy().tobytes()).hexdigest() == digest, (size, scale, img.size)


def _sweep():
    g = torch.Generator().manual_seed(5)
    sizes = [(int(h), int(w)) for h, w in torch.randint(20, 700, (40, 2), generator=g)]
    sizes += [(73, 73), (64, 64), (63, 90), (90, 63), (2, 300), (300, 2), (1, 1), (1000, 37)]
    return [(size, scale, h, w) for h, w in sizes for size, scale in ((64, 73), (64, 64), (32, 36), (48, 40))]


def test_host_geometry_matches_torchvision():
    """resized size, crop origin (padding included) and support region, on a sweep of image and output sizes"""
    import torchvision.transforms.functional as F
    from PIL import Image
    from torchvision.transforms import InterpolationMode
    rng = np.random.default_rng(0)
    for size, scale, h, w in _sweep():
        spec = ScaleCrop(size, scale)
        geom, (rh_, rw_) = spec.geometry(h, w)
        y0, x0, H, W, RH, RW, top, left = geom.tolist()
        assert (H, W) == (h, w)
        if scale != size:
            assert [RH, RW] == F._compute_resized_output_size((h, w), [scale])
        else:
            assert (RH, RW) == (h, w)
        # the crop origin: torchvision's center_crop of an index image of the resized size (0 = its padding)
        idx = torch.arange(1, RH * RW + 1, dtype=torch.float64).view(1, RH, RW)
        got = F.center_crop(idx, [size, size])[0]
        yy, xx = torch.arange(size).view(-1, 1) + top, torch.arange(size).view(1, -1) + left
        inside = (yy >= 0) & (yy < RH) & (xx >= 0) & (xx < RW)
        assert torch.equal(got, torch.where(inside, yy * RW + xx + 1, torch.zeros(())).double()), (size, scale, h, w)
        # the support region lies in the image and holds every source pixel with a nonzero tap: zeroing the rest of a
        # random image leaves torchvision's output unchanged
        assert 0 <= y0 and y0 + rh_ <= h and 0 <= x0 and x0 + rw_ <= w and rh_ >= 1 and rw_ >= 1
        if h * w > 250000:
            continue
        a = rng.integers(1, 256, (h, w), dtype=np.uint8)
        cut = np.zeros_like(a)
        cut[y0:y0 + rh_, x0:x0 + rw_] = a[y0:y0 + rh_, x0:x0 + rw_]

        def ref(arr):
            im = Image.fromarray(arr, 'L')
            if scale != size:
                im = F.resize(im, scale, InterpolationMode.BILINEAR)
            return np.asarray(F.center_crop(im, [size, size]))
        assert np.array_equal(ref(a), ref(cut)), (size, scale, h, w)


def test_table_validation():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    spec = ScaleCrop(64, 73)
    samples = [(spec(_image(h, w, 'RGB', k)), k) for k, (h, w) in enumerate(((375, 500), (90, 60), (64, 64)))]
    batch, _ = ScaleCropCollate(spec)(samples)
    ops.check_scale_crop_tables(batch.index, batch.geom, batch.nbytes, 3, spec.size)
    assert batch.geom[0, 0] > 0 and batch.geom[0, 1] > 0
    for col, value, match in ((0, 0, 'misses'), (1, 0, 'misses'), (2, 70000, 'outside 1'), (4, 0, 'outside 1'),
                              (0, 10 ** 4, 'outside its'), (6, 0, 'misses'), (7, 40, 'misses')):
        geom = batch.geom.clone()
        geom[0, col] = value
        with pytest.raises(B200Error, match=match):
            ops.check_scale_crop_tables(batch.index, geom, batch.nbytes, 3, spec.size)
    for row in ((batch.nbytes, 10, 10), (-1, 10, 10), (0, 0, 10), (0, 70000, 1)):
        ix = batch.index.clone()
        ix[1] = torch.tensor(row)
        with pytest.raises(B200Error, match='buffer'):
            ops.check_scale_crop_tables(ix, batch.geom, batch.nbytes, 3, spec.size)
    with pytest.raises(B200Error, match=r'\[B, 8\]'):
        ops.check_scale_crop_tables(batch.index, batch.geom[:, :7], batch.nbytes, 3, spec.size)


def test_batch_packing_and_replace():
    spec = ScaleCrop(32, 36)
    imgs = [_image(h, w, 'RGB', k) for k, (h, w) in enumerate(((40, 50), (100, 30), (37, 64), (200, 210)))]
    samples = [(spec(im), 10 + k) for k, im in enumerate(imgs)]
    batch, target = ScaleCropCollate(spec)(samples)
    assert batch.rows == 4 and target.tolist() == [10, 11, 12, 13]
    assert batch.index.dtype == torch.int64 and batch.geom.dtype == torch.int32 and batch.regions.dim() == 1
    off = 0
    for b, ((reg, g), _) in enumerate(samples):
        o, h, w = batch.index[b].tolist()
        assert o == off and (h, w) == tuple(reg.shape[:2]) and torch.equal(batch.geom[b], g)
        y0, x0 = g[0].item(), g[1].item()
        assert torch.equal(batch.regions[o:o + h * w * 3].view(h, w, 3),
                           torch.from_numpy(np.asarray(imgs[b])[y0:y0 + h, x0:x0 + w].copy()))
        off += h * w * 3
    assert off == batch.nbytes == batch.regions.numel()
    moved = batch.replace(tuple(t.clone() for t in batch.tensors))
    assert isinstance(moved, ScaleCropBatch) and moved.nbytes == batch.nbytes and moved.host[0] is batch.index
    assert torch.equal(moved.apply(), batch.apply())


def test_loader_yields_scale_crop_batches():
    from convnet.pytorch_b200.data import DataRegime
    reg = DataRegime(None, defaults={'name': 'synthetic_imagenet', 'split': 'val', 'augment': False,
                                     'input_size': 64, 'batch_size': 4, 'num_workers': 0, 'synthetic_length': 16,
                                     'device_scale_crop': True, 'shuffle': False, 'pin_memory': True})
    batch, target = next(iter(reg.get_loader()))
    assert isinstance(batch, ScaleCropBatch) and batch.rows == 4 and target.shape == (4,)
    assert batch.spec.size == (64, 64) and batch.spec.scale_size == 73 and batch.apply().shape == (4, 3, 64, 64)


def test_unsupported_settings_raise():
    from convnet.pytorch_b200.data import DataRegime, scale_crop_spec
    base = {'name': 'synthetic_imagenet', 'split': 'val', 'augment': False, 'input_size': 64, 'batch_size': 4,
            'num_workers': 0, 'synthetic_length': 8, 'device_scale_crop': True}
    for extra, match in ((dict(augment=True), 'evaluation transform'), (dict(num_crops=5), 'multi-crop'),
                         (dict(duplicates=2), 'duplicates'), (dict(autoaugment=True), 'autoaugment'),
                         (dict(device_augment=True), 'different'), (dict(device_resized_crop=True), 'different'),
                         (dict(name='synthetic_cifar10'), 'ImageNet'),
                         (dict(name='cifar10', transform_name='imagenet'), 'cifar10')):
        with pytest.raises(NotImplementedError, match=match):
            DataRegime(None, defaults=dict(base, **extra))
    with pytest.raises(NotImplementedError, match='bilinear'):
        scale_crop_spec('imagenet', interpolation='bicubic')
    assert scale_crop_spec('imagenet').scale_size == 256 and scale_crop_spec('imagenet').size == (224, 224)


def test_cli_cpu_run_with_device_scale_crop(tmp_path):
    """ResNet-18, synthetic ImageNet at 64 px, CPU: two training steps, then two validation steps with
    --device-scale-crop (on the CPU the batch's apply() is evaluated)."""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 18}", '--dataset', 'synthetic_imagenet',
              '--device', 'cpu', '-b', '4', '--epochs', '1', '--max-steps', '2', '--workers', '0',
              '--input-size', '64', '--device-scale-crop', '--results-dir', str(tmp_path), '--save', 'sc'])
    import csv
    rows = list(csv.DictReader(open(tmp_path / 'sc' / 'results.csv')))
    assert len(rows) == 1 and float(rows[0]['validation loss']) > 0
