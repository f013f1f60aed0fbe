"""The Mix&Match CIFAR size regimes with device augmentation (reference preprocess.py:44-54 with input_size !=
scale_size; models/resnet.py:274-285) on the CPU: BatchAugment(resize=S).apply against the SHA-256 of every copy the
unmodified reference transform produced (tests/golden/mixsize_augment.npz, written by tools/make_mixsize_golden.py),
the draw ranges, the data-regime plumbing of the four ``sampled_D+`` configurations over a stand-in for the CIFAR-10
files, the combinations that are still refused, the C ABI of the resizing relayout and the command line.  CPU only."""
import hashlib
import os
import re

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'mixsize_augment.npz')


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


@pytest.fixture(scope='module')
def gold():
    z = np.load(GOLD)
    return {k: z[k] for k in z.files}


def gold_spec(gold, size):
    holes, length = (int(v) for v in gold['cutout_%d' % size])
    return BatchAugment(padding=int(gold['padding']), cutout={'holes': holes, 'length': length} if holes else None,
                        duplicates=gold['draws_%d' % size].shape[1], resize=size)


@pytest.mark.parametrize('size', [16, 24, 48])
def test_apply_reproduces_reference_copies(gold, size):
    assert size in gold['sizes']
    images, draws = torch.from_numpy(gold['images']), torch.from_numpy(gold['draws_%d' % size])
    out = gold_spec(gold, size).apply(images, draws)
    assert out.shape == (draws.shape[0] * draws.shape[1], 3, size, size) and out.dtype == torch.float32
    assert [_digest(c) for c in out] == list(gold['sha256_%d' % size])
    d = gold['draws_%d' % size]
    assert {0, 8} <= set(d[..., 0].ravel()) | set(d[..., 1].ravel()) and {0, 1} <= set(d[..., 2].ravel())


def test_padding_is_resized_with_the_picture():
    """RandomCrop's zero fill lies inside the picture the filter sees: at offset (0, 0) the first output row and column
    blend it with image pixels, so they are neither the fill nor what crop-then-resize-then-pad would give."""
    images = torch.full((1, 32, 32, 3), 255, dtype=torch.uint8)
    spec = BatchAugment(padding=4, duplicates=1, resize=24, normalize={'mean': [0., 0., 0.], 'std': [1., 1., 1.]})
    out = spec.apply(images, torch.tensor([[[0, 0, 0]]], dtype=torch.int16))[0, 0]
    assert float(out[0, 0]) == 0.0 and float(out[-1, -1]) == 1.0
    row = out[-1]                                 # the bottom row lies inside the image; 4 padded columns on its left
    assert float(row[0]) == 0.0 and 0.0 < float(row[2]) < float(row[3]) < 1.0 and float(row[4]) == 1.0
    assert torch.equal(out[:, -1], row)           # and the same down the right column


def test_identity_resize_equals_the_plain_transform():
    g = torch.Generator().manual_seed(4)
    images = torch.randint(0, 256, (3, 32, 32, 3), generator=g, dtype=torch.uint8)
    torch.manual_seed(4)
    np.random.seed(4)
    plain = BatchAugment(cutout={'holes': 2, 'length': 8}, duplicates=3)
    params = plain.sample(3, 32, 32)
    same = BatchAugment(cutout={'holes': 2, 'length': 8}, duplicates=3, resize=32)
    assert torch.equal(plain.apply(images, params), same.apply(images, params))
    assert plain.resize is None and same.resize == (32, 32)


def test_sample_ranges():
    torch.manual_seed(1)
    np.random.seed(1)
    spec = BatchAugment(padding=4, cutout={'holes': 2, 'length': 8}, duplicates=4, resize=16)
    p = spec.sample(500, 32, 32).reshape(-1, 11).numpy().astype(np.int64)
    assert set(p[:, 0]) == set(range(9)) and set(p[:, 1]) == set(range(9)) and set(p[:, 2]) == {0, 1}
    boxes = p[:, 3:].reshape(-1, 4)
    assert boxes.min() == 0 and boxes.max() == 16                       # boxes live in the 16 x 16 output
    assert ((boxes[:, 1] - boxes[:, 0]) <= 8).all() and ((boxes[:, 3] - boxes[:, 2]) <= 8).all()
    # a non-square output: rows against OH, columns against OW
    q = BatchAugment(cutout={'holes': 1, 'length': 64}, duplicates=1, resize=(12, 40)).sample(400, 32, 32)
    q = q.reshape(-1, 7).numpy()
    assert q[:, 4].max() == 12 and q[:, 6].max() == 40
    with pytest.raises(ValueError):
        BatchAugment(resize=0)


class FakeCIFAR10(torch.utils.data.Dataset):
    """Stands in for torchvision.datasets.CIFAR10 (no dataset files here): seeded uniform uint8 ``data`` [N, 32, 32, 3]
    and ``targets``, samples as torchvision yields them."""
    length = 640

    def __init__(self, root=None, train=True, transform=None, target_transform=None, download=False):
        g = torch.Generator().manual_seed(0 if train else 1)
        n = self.length if train else 64
        self.data = torch.randint(0, 256, (n, 32, 32, 3), generator=g, dtype=torch.uint8).numpy()
        self.targets = torch.randint(0, 10, (n,), generator=g).tolist()
        self.transform = transform

    def __len__(self):
        return len(self.targets)

    def __getitem__(self, i):
        from PIL import Image
        img = Image.fromarray(self.data[i])
        return (self.transform(img) if self.transform is not None else img), self.targets[i]


@pytest.fixture
def fake_cifar10(monkeypatch):
    import torchvision.datasets as tvd
    monkeypatch.setattr(tvd, 'CIFAR10', FakeCIFAR10)


def test_spec_and_dataset_accept_the_resize(fake_cifar10):
    from convnet.pytorch_b200.data import device_augment_spec, u8_dataset
    spec = device_augment_spec('cifar10', input_size=24, duplicates=2, cutout={'holes': 1, 'length': 16})
    assert spec.resize == (24, 24) and spec.duplicates == 2 and spec.holes == 1 and spec.padding == 4
    assert device_augment_spec('cifar100', input_size=48, scale_size=32).resize == (48, 48)
    # no resize: what the spec was before
    for kw in (dict(), dict(input_size=32), dict(input_size=32, scale_size=32), dict(scale_size=32)):
        assert device_augment_spec('cifar10', **kw).resize is None
    # the dataset serves its 32-px images whatever the input size; it cannot crop at another size
    assert u8_dataset('cifar10', input_size=24).images.shape == (640, 32, 32, 3)
    assert u8_dataset('cifar10', input_size=24, scale_size=32, split='val').images.shape == (64, 32, 32, 3)
    with pytest.raises(NotImplementedError, match='image size'):
        u8_dataset('cifar10', input_size=24, scale_size=40)
    # a synthetic pool is generated at input_size and is not resized; asking for both sizes is refused as before
    assert device_augment_spec('synthetic_cifar10', input_size=24).resize is None
    assert u8_dataset('synthetic_cifar10', input_size=24, synthetic_length=8).images.shape == (8, 24, 24, 3)
    with pytest.raises(NotImplementedError, match='resize'):
        device_augment_spec('synthetic_cifar10', input_size=24, scale_size=32)


def test_resizing_regime_and_what_it_still_refuses(fake_cifar10):
    from convnet.pytorch_b200.data import DataRegime
    base = {'name': 'cifar10', 'split': 'train', 'augment': True, 'batch_size': 4, 'num_workers': 0, 'duplicates': 2,
            'device_augment': True, 'input_size': 24}
    torch.manual_seed(0)
    x, t = next(iter(DataRegime(None, defaults=base).get_loader()))
    assert isinstance(x, AugmentedBatch) and x.images.shape == (4, 32, 32, 3) and x.spec.resize == (24, 24)
    assert x.apply().shape == (8, 3, 24, 24) and t.shape == (8,)
    with pytest.raises(NotImplementedError, match='autoaugment'):
        DataRegime(None, defaults=dict(base, autoaugment=True))
    with pytest.raises(NotImplementedError, match='multi-crop'):
        DataRegime(None, defaults=dict(base, num_crops=5))
    with pytest.raises(ValueError, match='training transform'):
        DataRegime(None, defaults=dict(base, augment=False))
    with pytest.raises(NotImplementedError, match='image size'):
        DataRegime(None, defaults=dict(base, scale_size=40))


def test_sampled_regime_yields_augmented_batches_of_every_size(fake_cifar10):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import DataRegime, SampledDataRegime
    torch.manual_seed(0)
    model = models.resnet(dataset='cifar10', depth=8, regime='sampled_D+')
    probs, configs = zip(*model.sampled_data_regime)
    assert [(c['input_size'], c['batch_size'], c['duplicates']) for c in configs] == \
        [(32, 64, 1), (48, 28, 1), (24, 64, 2), (16, 64, 4)]
    defaults = {'name': 'cifar10', 'split': 'train', 'augment': True, 'shuffle': True, 'num_workers': 0,
                'drop_last': True, 'device_augment': True, 'cutout': {'holes': 1, 'length': 16}}
    data = SampledDataRegime([DataRegime(None, defaults={**defaults, **c}) for c in configs], probs)
    data.set_epoch(0)
    seen = {}
    for batch, target in data.get_loader():
        assert isinstance(batch, AugmentedBatch) and batch.images.shape[1:] == (32, 32, 3)
        size = (batch.spec.resize or (32, 32))[0]
        seen[size] = (batch.images.shape[0], batch.spec.duplicates, batch.rows, len(target))
        assert int(batch.params[..., 3:].max()) <= size
    assert seen == {32: (64, 1, 64, 64), 48: (28, 1, 28, 28), 24: (64, 2, 128, 128), 16: (64, 4, 256, 256)}
    x = batch.apply()
    assert x.shape == (batch.rows, 3, size, size)


def test_cli_cpu_run_of_the_sampled_regime_with_device_augment(fake_cifar10, tmp_path):
    """The README's Mix&Match command with --device-augment, on the CPU (the batches' apply()) for three steps."""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 8, 'regime': 'sampled_D+'}", '--dataset', 'cifar10',
              '-b', '64', '--device', 'cpu', '--epochs', '1', '--max-steps', '3', '--workers', '0', '--device-augment',
              '--results-dir', str(tmp_path), '--save', 'mix'])
    import csv
    rows = list(csv.DictReader(open(tmp_path / 'mix' / 'results.csv')))
    assert len(rows) == 1 and float(rows[0]['training loss']) > 0


def test_abi_declares_and_exports_the_resizing_relayout():
    from convnet.pytorch_b200 import lib
    src = open(os.path.join(ROOT, 'include', 'b200conv.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    m = re.search(r'int\s+b200_input_prep_u8_aug_resize\s*\(([^)]*)\)\s*;', src)
    assert m, 'b200_input_prep_u8_aug_resize is not declared in include/b200conv.h'
    args = [' '.join(a.split()) for a in m.group(1).split(',')]
    assert args == ['const uint8_t* x_nhwc', 'int N', 'int D', 'int C', 'int H', 'int W', 'int OH', 'int OW', 'int Cpad',
                    'int pad', 'const float* lut', 'const int16_t* params', 'int holes', 'void* out',
                    'b200_stream_t stream']
    import ctypes
    want = [ctypes.c_int if a.startswith('int ') else ctypes.c_void_p for a in args]
    assert lib.SIGNATURES['b200_input_prep_u8_aug_resize'] == want
    assert lib.available(), 'libb200conv.so missing: run __graft_entry__.build()'
    assert hasattr(lib.load(), 'b200_input_prep_u8_aug_resize')
