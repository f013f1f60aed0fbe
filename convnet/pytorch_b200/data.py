"""Data regimes: the (input size, batch size, duplicates) schedule side of the reference's data.py:74-203.

``DataRegime(regime, defaults)`` resolves, per epoch, the dataset / transform / loader settings from a regime
list (same grammar as the optimizer regimes) and hands out a ``DataLoader``; ``SampledDataRegime`` mixes
several regimes with given probabilities (Mix&Match, models/resnet.py:279-311 in the reference).

Datasets: the north-star configurations are synthetic, so ``synthetic_*`` names are first class here
(the reference has no synthetic option and needs downloads -- SURVEY.md section 8c shim 5):
  synthetic_cifar10 / synthetic_cifar100 : N(0,1) 3x32x32 tensors, 10 / 100 classes
  synthetic_imagenet                     : N(0,1) 3xSxS tensors (S = input_size, default 224), 1000 classes
Real datasets (cifar10, cifar100, imagenet folders) go through torchvision if it is importable; the basic PIL
augmentation stack of the reference (preprocess.py) is reproduced with Cutout, AutoAugment and colour jitter /
Lighting are out of scope (SURVEY.md section 2).

Batch augmentation on the device (transform key ``device_augment``, CIFAR-style training only): the loader yields
(utils.augment.AugmentedBatch of the B uint8 NHWC images and their per-copy draws, target repeated to B*D) and the
stem relayout kernel writes the B*D augmented copies.  Real cifar10 / cifar100 read the dataset's uint8 ``.data``;
synthetic_cifar* use a pool of uniform uint8 images.  When ``input_size`` differs from ``scale_size`` (the Mix&Match
``sampled*`` regimes on cifar10 / cifar100: crops of the 32-px images resized to 16 / 24 / 48 px) the same kernel path
resizes each crop; a synthetic pool is generated at ``input_size`` and is never resized.

RandomResizedCrop on the device (transform key ``device_resized_crop``, ImageNet-style training only): the workers
decode and draw the reference's crop boxes and flips per image; the loader yields (utils.augment.ResizedCropBatch of
the images' regions and draws, target repeated to B*D) and the stem relayout kernel resamples, flips and normalises.
Real imagenet decodes with the reference's pil_loader (convert('RGB')); synthetic_imagenet uses a seeded pool of 64
uniform uint8 images of 200-600 px.

Resize + CenterCrop on the device (transform key ``device_scale_crop``, ImageNet-style evaluation only): the workers
decode and compute each image's resized size, crop offsets and support region; the loader yields
(utils.augment.ScaleCropBatch of the regions and geometry, target) and the stem relayout kernel resamples the crop
window of each whole image's resize and normalises it.  Same datasets as ``device_resized_crop``.

JPEG decode on the device (transform key ``device_decode``, together with one of the two device crops): the workers
read the file bytes and parse the headers (utils/jpeg.py) but do not decode baseline JPEGs; the loader yields
(utils.augment.JpegBatch, target) and csrc/jpeg.cu decodes each image's region into the region buffer the crop's
relayout reads, byte for byte what Pillow decodes.  Other files (progressive, CMYK, PNG, ...) are decoded by PIL in the
worker and ride in the same batch.  Real imagenet reads the files' bytes; synthetic_imagenet encodes its seeded pool
in memory with PIL (quality 90, 4:2:0).
"""
import os
from copy import deepcopy
from itertools import accumulate, chain

import torch
from torch.utils.data import Dataset, Subset
from torch.utils.data.distributed import DistributedSampler

from .utils.augment import AugmentCollate, BatchAugment, Cutout, JpegCollate, JpegDecode, ResizedCrop, \
    ResizedCropCollate, ScaleCrop, ScaleCropCollate
from .utils.regime import Regime


class SyntheticImages(Dataset):
    """Deterministic N(0,1) images with uniform random labels; sample i is a pure function of (seed, i).

    A small pool of ``pool`` distinct images is generated once and indexed modulo, so that iterating costs
    nothing next to a training step (the metric excludes data loading: SURVEY.md section 8d)."""

    def __init__(self, length, shape, num_classes, seed=0, duplicates=1, pool=256):
        g = torch.Generator().manual_seed(seed)
        self.length = length
        self.duplicates = duplicates
        self.pool = min(pool, length)
        self.images = torch.randn(self.pool, *shape, generator=g)
        self.labels = torch.randint(0, num_classes, (length,), generator=g)

    def __len__(self):
        return self.length

    def __getitem__(self, idx):
        img = self.images[idx % self.pool]
        if self.duplicates > 1:  # batch augmentation: D "augmentations" of the sample (here: D pool neighbours)
            img = torch.stack([self.images[(idx + d) % self.pool] for d in range(self.duplicates)])
        return img, int(self.labels[idx])


class U8Images(Dataset):
    """(uint8 HWC image, label) samples for device augmentation: ``images`` uint8 [P, H, W, C] (indexed modulo P, so a
    small synthetic pool stands for a long dataset), ``labels`` one per sample."""

    def __init__(self, images, labels):
        self.images = torch.as_tensor(images)
        self.labels = torch.as_tensor(labels, dtype=torch.long)

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, idx):
        return self.images[idx % len(self.images)], int(self.labels[idx])


_IMAGE_STATS = {'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225]}   # preprocess.py:7-8 of the reference


def real_dataset_transform(transform_name='imagenet', input_size=None, scale_size=None, normalize=None, augment=True,
                           cutout=None, autoaugment=False, padding=None, duplicates=1, num_crops=1):
    """The basic transform stacks the reference's ``get_transform`` selects for real image datasets
    (preprocess.py:114-161): random-resized-crop + flip (imagenet, train), pad-4 random crop + flip (cifar, train),
    resize + centre crop (evaluation), then ToTensor + Normalize, then Cutout when ``cutout`` = {'holes', 'length'}
    (preprocess.py:159-160).  AutoAugment, Lighting/colour jitter and multi-crop evaluation are outside this repo's
    scope (SURVEY.md section 2, rows 14-15) and raise instead of being silently dropped."""
    import torchvision.transforms as T
    if autoaugment or num_crops != 1:
        raise NotImplementedError('autoaugment / multi-crop evaluation are outside the B200 hot path '
                                  '(reference preprocess.py, autoaugment.py); use the reference data pipeline')
    stats = normalize or _IMAGE_STATS
    tail = [T.ToTensor(), T.Normalize(**stats)]
    if 'imagenet' in transform_name:
        input_size = input_size or 224
        scale_size = scale_size or int(input_size * 8 / 7)
        if augment:
            # the reference's inception_preprocess adds ColorJitter + PCA Lighting (preprocess.py:77-97) which are not
            # reproduced: say so rather than train on a silently different distribution
            import logging
            logging.warning('imagenet training transform: RandomResizedCrop + flip only (no colour jitter / lighting)')
            head = [T.RandomResizedCrop(input_size), T.RandomHorizontalFlip()]
        else:
            head = ([T.Resize(scale_size)] if scale_size != input_size else []) + [T.CenterCrop(input_size)]
    elif 'cifar' in transform_name:
        input_size = input_size or 32
        scale_size = scale_size or 32
        if augment:
            head = [T.RandomCrop(scale_size, padding=padding or 4)]
            if input_size != scale_size:
                head.append(T.Resize(input_size))
            head.append(T.RandomHorizontalFlip())
        else:
            head = ([T.Resize(scale_size)] if scale_size != input_size else []) + [T.CenterCrop(input_size)]
    else:
        raise NotImplementedError('no transform for dataset family %r' % transform_name)
    if cutout is not None:
        tail.append(Cutout(**cutout))
    fn = T.Compose(head + tail)
    if duplicates > 1:   # batch augmentation: D independent draws of the transform per sample (preprocess.py:105-112)
        return T.Lambda(lambda img: torch.stack([fn(img) for _ in range(duplicates)], dim=0))
    return fn


_SYNTHETIC = {'synthetic_cifar10': (32, 10, 50000, 10000), 'synthetic_cifar100': (32, 100, 50000, 10000),
              'synthetic_imagenet': (224, 1000, 1281167, 50000)}


def get_dataset(name, split='train', transform=None, target_transform=None, download=True,
                datasets_path='~/Datasets', input_size=None, duplicates=1, synthetic_length=None):
    train = split == 'train'
    if name in _SYNTHETIC:
        size, classes, n_train, n_val = _SYNTHETIC[name]
        size = input_size or size
        length = synthetic_length or int(os.environ.get('B200_SYNTHETIC_LENGTH', n_train if train else n_val))
        return SyntheticImages(length, (3, size, size), classes, seed=0 if train else 1, duplicates=duplicates)
    try:
        import torchvision.datasets as tvd
        import torchvision.transforms as T
    except ImportError as e:  # pragma: no cover
        raise ValueError('dataset %r needs torchvision (%s); use a synthetic_* dataset' % (name, e))
    root = os.path.join(os.path.expanduser(datasets_path), name)
    if transform is None:
        transform = T.ToTensor()
    if name == 'cifar10':
        return tvd.CIFAR10(root=root, train=train, transform=transform, target_transform=target_transform,
                           download=download)
    if name == 'cifar100':
        return tvd.CIFAR100(root=root, train=train, transform=transform, target_transform=target_transform,
                            download=download)
    if name == 'imagenet':
        return tvd.ImageFolder(root=os.path.join(root, 'train' if train else 'val'), transform=transform,
                               target_transform=target_transform)
    raise ValueError('unknown dataset %r' % name)


def device_augment_spec(transform_name='cifar10', input_size=None, scale_size=None, normalize=None, augment=True,
                        cutout=None, autoaugment=False, padding=None, duplicates=1, num_crops=1, device_augment=True,
                        device_resized_crop=False, device_scale_crop=False, device_decode=False):
    """The BatchAugment of a ``device_augment`` transform setting: the CIFAR training transform of
    real_dataset_transform (pad-4 random crop + flip + ToTensor + Normalize [+ Cutout]) with its duplicates.  The
    settings it cannot reproduce raise."""
    if 'cifar' not in (transform_name or ''):
        raise NotImplementedError('device_augment reproduces the CIFAR training transform only (RandomResizedCrop of '
                                  'imagenet needs decoded variable-size images); got transform %r' % transform_name)
    if not augment:
        raise ValueError('device_augment is a training transform (augment=True); evaluation loaders do not take it')
    if autoaugment or num_crops != 1:
        raise NotImplementedError('device_augment does not reproduce autoaugment / multi-crop')
    # the reference crops at scale_size (32 unless set) and resizes to input_size when the two differ (preprocess.py:
    # 44-54,134-143): the Mix&Match size regimes.  A synthetic dataset has no scale_size: its "transform" is its
    # geometry, the pool is generated at input_size, and a setting that asks for both sizes is refused as before.
    if (transform_name or '').startswith('synthetic'):
        if scale_size is not None and input_size is not None and scale_size != input_size:
            raise NotImplementedError('device_augment does not resize a synthetic pool (it is generated at input_size): '
                                      'scale_size %s != input_size %s' % (scale_size, input_size))
    elif scale_size is None:
        scale_size = 32
    resize = input_size if scale_size is not None and input_size is not None and scale_size != input_size else None
    return BatchAugment(padding=padding or 4, flip=True, cutout=cutout, duplicates=duplicates or 1,
                        normalize=normalize or _IMAGE_STATS, resize=resize)


def u8_dataset(name, input_size=None, scale_size=None, split='train', download=True, datasets_path='~/Datasets',
               synthetic_length=None, **_):
    """uint8 NHWC samples for device augmentation: the dataset's own uint8 array (cifar10 / cifar100), or a pool of
    256 uniform uint8 images at ``input_size`` for synthetic_cifar*.  The real images have the size the transform crops
    at (``scale_size``, 32); a resize to ``input_size`` happens on the device."""
    train = split == 'train'
    if name in ('synthetic_cifar10', 'synthetic_cifar100'):
        size, classes, n_train, n_val = _SYNTHETIC[name]
        size = input_size or size
        length = synthetic_length or int(os.environ.get('B200_SYNTHETIC_LENGTH', n_train if train else n_val))
        g = torch.Generator().manual_seed(0 if train else 1)
        images = torch.randint(0, 256, (min(256, length), size, size, 3), generator=g, dtype=torch.uint8)
        return U8Images(images, torch.randint(0, classes, (length,), generator=g))
    if name in ('cifar10', 'cifar100'):
        import torchvision.datasets as tvd
        if scale_size not in (None, 32):
            raise NotImplementedError('device_augment crops at the image size: %s images are 32x32, scale_size %s'
                                      % (name, scale_size))
        cls = tvd.CIFAR10 if name == 'cifar10' else tvd.CIFAR100
        ds = cls(root=os.path.join(os.path.expanduser(datasets_path), name), train=train, download=download)
        return U8Images(ds.data, ds.targets)
    raise NotImplementedError('device_augment supports cifar10, cifar100 and synthetic_cifar*; got %r' % name)


def resized_crop_spec(transform_name='imagenet', input_size=None, scale_size=None, normalize=None, augment=True,
                      cutout=None, autoaugment=False, padding=None, duplicates=1, num_crops=1, device_augment=False,
                      device_resized_crop=True, interpolation='bilinear', color_jitter=None, lighting=None,
                      device_scale_crop=False, device_decode=False):
    """The ResizedCrop of a ``device_resized_crop`` transform setting: the imagenet training transform of
    real_dataset_transform (RandomResizedCrop(input_size) + flip + ToTensor + Normalize) with its duplicates.  The
    settings it cannot reproduce raise."""
    if 'imagenet' not in (transform_name or ''):
        raise NotImplementedError('device_resized_crop reproduces the ImageNet training transform only; got transform '
                                  '%r (CIFAR training: use device_augment)' % transform_name)
    if not augment:
        raise NotImplementedError('device_resized_crop is a training transform (augment=True); evaluation loaders do '
                                  'not take it')
    if device_augment:
        raise NotImplementedError('device_resized_crop and device_augment are two different transforms; set one')
    if cutout:
        raise NotImplementedError('device_resized_crop does not apply Cutout')
    if autoaugment or num_crops != 1:
        raise NotImplementedError('device_resized_crop does not reproduce autoaugment / multi-crop')
    if color_jitter or lighting:
        raise NotImplementedError('device_resized_crop does not reproduce colour jitter / Lighting')
    if str(interpolation).lower() != 'bilinear':
        raise NotImplementedError('device_resized_crop resamples bilinearly only; got %r' % (interpolation,))
    return ResizedCrop(input_size or 224, duplicates=duplicates or 1, normalize=normalize or _IMAGE_STATS)


def scale_crop_spec(transform_name='imagenet', input_size=None, scale_size=None, normalize=None, augment=False,
                    cutout=None, autoaugment=False, padding=None, duplicates=1, num_crops=1, device_augment=False,
                    device_resized_crop=False, device_scale_crop=True, interpolation='bilinear', device_decode=False):
    """The ScaleCrop of a ``device_scale_crop`` transform setting: the imagenet evaluation transform of
    real_dataset_transform (Resize(scale_size) + CenterCrop(input_size) + ToTensor + Normalize, scale_size =
    int(input_size * 8 / 7) unless set).  The settings it cannot reproduce raise."""
    if 'imagenet' not in (transform_name or ''):
        raise NotImplementedError('device_scale_crop reproduces the ImageNet evaluation transform only; got transform '
                                  '%r' % transform_name)
    if augment:
        raise NotImplementedError('device_scale_crop is an evaluation transform (augment=False); training loaders do '
                                  'not take it (ImageNet training: use device_resized_crop)')
    if device_augment or device_resized_crop:
        raise NotImplementedError('device_scale_crop and device_augment / device_resized_crop are different '
                                  'transforms; set one per loader')
    if num_crops != 1 or (duplicates or 1) != 1:
        raise NotImplementedError('device_scale_crop makes one centre crop per image (no multi-crop / duplicates)')
    if autoaugment or cutout:
        raise NotImplementedError('device_scale_crop does not reproduce autoaugment / Cutout')
    if str(interpolation).lower() != 'bilinear':
        raise NotImplementedError('device_scale_crop resamples bilinearly only; got %r' % (interpolation,))
    input_size = input_size or 224
    return ScaleCrop(input_size, scale_size or int(input_size * 8 / 7), normalize=normalize or _IMAGE_STATS)


class DecodedImages(Dataset):
    """(transform(PIL image), label) samples of ``images`` (PIL images, indexed modulo their count) and ``labels``."""

    def __init__(self, images, labels, transform=None):
        self.images, self.labels, self.transform = images, torch.as_tensor(labels, dtype=torch.long), transform

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, idx):
        img = self.images[idx % len(self.images)]
        return (self.transform(img) if self.transform is not None else img), int(self.labels[idx])


def synthetic_imagenet_pool(n=64, lo=200, hi=600, seed=0):
    """``n`` seeded uniform uint8 RGB PIL images with sides in [lo, hi]."""
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    sizes = torch.randint(lo, hi + 1, (n, 2), generator=g)
    return [Image.fromarray(torch.randint(0, 256, (int(h), int(w), 3), generator=g, dtype=torch.uint8).numpy(), 'RGB')
            for h, w in sizes]


def decoded_dataset(name, transform, split='train', datasets_path='~/Datasets', synthetic_length=None, **_):
    """Decode-only samples for device_resized_crop and device_scale_crop: ImageFolder with the reference's pil_loader
    (convert('RGB')) for imagenet, the seeded synthetic_imagenet_pool for synthetic_imagenet; ``transform`` (a
    ResizedCrop or a ScaleCrop) does the per-image host work."""
    train = split == 'train'
    if name == 'synthetic_imagenet':
        _, classes, n_train, n_val = _SYNTHETIC[name]
        length = synthetic_length or int(os.environ.get('B200_SYNTHETIC_LENGTH', n_train if train else n_val))
        pool = synthetic_imagenet_pool(seed=0 if train else 1)
        g = torch.Generator().manual_seed(2 if train else 3)
        return DecodedImages(pool, torch.randint(0, classes, (length,), generator=g), transform)
    if name == 'imagenet':
        import torchvision.datasets as tvd
        return tvd.ImageFolder(root=os.path.join(os.path.expanduser(datasets_path), name, 'train' if train else 'val'),
                               transform=transform)
    raise NotImplementedError('device_resized_crop / device_scale_crop support imagenet and synthetic_imagenet; got %r'
                              % name)


def read_bytes(path):
    """ImageFolder loader of ``device_decode``: the file's bytes (the workers parse headers, they do not decode)."""
    with open(path, 'rb') as f:
        return f.read()


def synthetic_imagenet_jpegs(seed=0):
    """synthetic_imagenet_pool(seed) encoded in memory by PIL (quality 90, 4:2:0): the files of ``device_decode``."""
    import io
    out = []
    for img in synthetic_imagenet_pool(seed=seed):
        buf = io.BytesIO()
        img.save(buf, 'JPEG', quality=90, subsampling=2)
        out.append(buf.getvalue())
    return out


def encoded_dataset(name, transform, split='train', datasets_path='~/Datasets', synthetic_length=None, **_):
    """File-bytes samples of ``device_decode``: ImageFolder with read_bytes for imagenet, synthetic_imagenet_jpegs for
    synthetic_imagenet; ``transform`` (a utils.augment.JpegDecode) does the per-image host work."""
    train = split == 'train'
    if name == 'synthetic_imagenet':
        _, classes, n_train, n_val = _SYNTHETIC[name]
        length = synthetic_length or int(os.environ.get('B200_SYNTHETIC_LENGTH', n_train if train else n_val))
        g = torch.Generator().manual_seed(2 if train else 3)
        return DecodedImages(synthetic_imagenet_jpegs(seed=0 if train else 1),
                             torch.randint(0, classes, (length,), generator=g), transform)
    if name == 'imagenet':
        import torchvision.datasets as tvd
        return tvd.ImageFolder(root=os.path.join(os.path.expanduser(datasets_path), name, 'train' if train else 'val'),
                               transform=transform, loader=read_bytes)
    raise NotImplementedError('device_decode supports imagenet and synthetic_imagenet; got %r' % name)


_DATA_ARGS = {'name', 'split', 'transform', 'target_transform', 'download', 'datasets_path', 'synthetic_length'}
_DATALOADER_ARGS = {'batch_size', 'shuffle', 'sampler', 'batch_sampler', 'num_workers', 'collate_fn', 'pin_memory',
                    'drop_last', 'timeout', 'worker_init_fn'}
_TRANSFORM_ARGS = {'transform_name', 'input_size', 'scale_size', 'normalize', 'augment', 'cutout', 'duplicates',
                   'num_crops', 'autoaugment', 'device_augment', 'device_resized_crop', 'device_scale_crop',
                   'device_decode'}
_OTHER_ARGS = {'distributed'}


class DataRegime(object):
    def __init__(self, regime, defaults={}):
        self.regime = Regime(regime, deepcopy(defaults))
        self.epoch = 0
        self.steps = None
        self._sampler = None
        self.get_loader(True)

    def get_setting(self):
        setting = self.regime.setting
        pick = lambda keys: {k: v for k, v in setting.items() if k in keys}  # noqa: E731
        out = {'data': pick(_DATA_ARGS), 'loader': pick(_DATALOADER_ARGS), 'transform': pick(_TRANSFORM_ARGS),
               'other': pick(_OTHER_ARGS)}
        out['transform'].setdefault('transform_name', out['data'].get('name'))
        return out

    def get(self, key, default=None):
        return self.regime.setting.get(key, default)

    def get_loader(self, force_update=False, override_settings=None, subset_indices=None):
        if force_update or self.regime.update(self.epoch, self.steps):
            setting = self.get_setting()
            if override_settings is not None:
                setting.update(override_settings)
            data_kwargs = dict(setting['data'])
            name = data_kwargs.get('name', '')
            collate = None
            tf_set = setting['transform']
            if tf_set.get('device_decode') and not (tf_set.get('device_scale_crop') or tf_set.get('device_resized_crop')):
                raise NotImplementedError('device_decode decodes into the region buffer of device_resized_crop or '
                                          'device_scale_crop; set one of them')
            if tf_set.get('device_decode'):
                spec = (scale_crop_spec if tf_set.get('device_scale_crop') else resized_crop_spec)(**tf_set)
                self._data = encoded_dataset(transform=JpegDecode(spec), **data_kwargs)
                collate = JpegCollate(spec)
            elif setting['transform'].get('device_scale_crop'):
                spec = scale_crop_spec(**setting['transform'])
                self._data = decoded_dataset(transform=spec, **data_kwargs)
                collate = ScaleCropCollate(spec)
            elif setting['transform'].get('device_resized_crop'):
                spec = resized_crop_spec(**setting['transform'])
                self._data = decoded_dataset(transform=spec, **data_kwargs)
                collate = ResizedCropCollate(spec)
            elif setting['transform'].get('device_augment'):
                spec = device_augment_spec(**setting['transform'])
                self._data = u8_dataset(input_size=setting['transform'].get('input_size'),
                                        scale_size=setting['transform'].get('scale_size'), **data_kwargs)
                collate = AugmentCollate(spec)
            elif name in _SYNTHETIC:  # the "transform" of a synthetic dataset is just its geometry
                data_kwargs['input_size'] = setting['transform'].get('input_size')
                data_kwargs['duplicates'] = setting['transform'].get('duplicates') or 1
            elif data_kwargs.get('transform') is None:
                # real images: build the transform the regime asks for (reference data.py:101-102) -- never fall back
                # to a bare ToTensor(), which would train on unnormalised, unaugmented, variable-size images
                tf = {k: v for k, v in setting['transform'].items()
                      if v is not None and k not in ('device_augment', 'device_resized_crop', 'device_scale_crop',
                                                     'device_decode')}
                data_kwargs['transform'] = real_dataset_transform(**tf)
            if collate is None:
                self._data = get_dataset(**data_kwargs)
            if subset_indices is not None:
                self._data = Subset(self._data, subset_indices)
            loader_kwargs = dict(setting['loader'])
            if name in _SYNTHETIC:
                loader_kwargs['num_workers'] = 0
            if setting['other'].get('distributed', False):
                loader_kwargs['sampler'] = DistributedSampler(self._data)
                loader_kwargs['shuffle'] = None
                loader_kwargs['pin_memory'] = False
            if collate is not None:
                loader_kwargs['collate_fn'] = collate
                # a pin-memory thread may not allocate pinned memory while the Trainer captures a step graph (global
                # capture mode); the batch is ~1/130 of the fp32 one, so its pageable copy costs little
                loader_kwargs['pin_memory'] = False
            self._sampler = loader_kwargs.get('sampler', None)
            self._loader = torch.utils.data.DataLoader(self._data, **loader_kwargs)
        return self._loader

    def set_epoch(self, epoch):
        self.epoch = epoch
        if self._sampler is not None and hasattr(self._sampler, 'set_epoch'):
            self._sampler.set_epoch(epoch)

    def __len__(self):
        return len(self._data)

    def __repr__(self):
        return str(self.regime)


class SampledDataLoader(object):
    """Interleaves several loaders; the order is a permutation seeded by the epoch only, so that all ranks
    draw the same (size, batch) sequence (data.py:133-139 in the reference)."""

    def __init__(self, dl_list):
        self.dl_list = dl_list
        self.epoch = 0

    def generate_order(self):
        order = list(chain(*[[idx] * len(dl) for idx, dl in enumerate(self.dl_list)]))
        g = torch.Generator().manual_seed(self.epoch)
        return torch.tensor(order)[torch.randperm(len(order), generator=g)].tolist()

    def __len__(self):
        return sum(len(dl) for dl in self.dl_list)

    def __iter__(self):
        iterators = [iter(dl) for dl in self.dl_list]
        for idx in self.generate_order():
            yield next(iterators[idx])


class SampledDataRegime(DataRegime):
    def __init__(self, data_regime_list, probs, split_data=True):
        self.probs = probs
        self.data_regime_list = data_regime_list
        self.split_data = split_data
        self.epoch = 0

    def get_setting(self):
        return [r.get_setting() for r in self.data_regime_list]

    def get(self, key, default=None):
        return [r.get(key, default) for r in self.data_regime_list]

    def get_loader(self, force_update=False):
        if self.split_data:
            sizes = {len(r._data.dataset) if isinstance(r._data, Subset) else len(r._data)
                     for r in self.data_regime_list}
            assert len(sizes) == 1, 'all datasets should be same size'
            total = sizes.pop()
            lengths = [int(p * total) for p in self.probs]
            lengths[-1] = total - sum(lengths[:-1])
            g = torch.Generator().manual_seed(1000003 + self.epoch)  # identical split on every rank
            perm = torch.randperm(total, generator=g).tolist()
            parts = [perm[end - n:end] for end, n in zip(accumulate(lengths), lengths)]
            loaders = [r.get_loader(force_update=True, subset_indices=parts[i])
                       for i, r in enumerate(self.data_regime_list)]
        else:
            loaders = [r.get_loader(force_update=force_update) for r in self.data_regime_list]
        self._loader = SampledDataLoader(loaders)
        self._loader.epoch = self.epoch
        return self._loader

    def set_epoch(self, epoch):
        self.epoch = epoch
        if hasattr(self, '_loader'):
            self._loader.epoch = epoch
        for r in self.data_regime_list:
            if r._sampler is not None and hasattr(r._sampler, 'set_epoch'):
                r._sampler.set_epoch(epoch)

    def __len__(self):
        return sum(len(r._data) for r in self.data_regime_list)

    def __repr__(self):
        return 'Sampled Data Regime:\n' + ''.join('w.p. %s:  %s\n' % (p, r)
                                                   for p, r in zip(self.probs, self.data_regime_list))
