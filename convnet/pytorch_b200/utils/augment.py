"""Batch augmentation ("Augment Your Batch", Hoffer et al., CVPR 2020) of the CIFAR training transform, drawn on the
host and applied on the device.

The reference runs the whole PIL transform D times per sample in the loader workers (preprocess.py:44-54,105-112):
RandomCrop(size, padding) -> RandomHorizontalFlip -> ToTensor -> Normalize [-> Cutout], and the trainer flattens the
[B, D, C, H, W] batch to B*D rows, row b*D + d (trainer.py:17-29).  Here the loader ships the B un-augmented uint8
images with a small table of per-copy draws (an ``AugmentedBatch``) and the stem relayout kernel writes the B*D
augmented, normalised copies (ops.input_prep_u8_aug).  ``BatchAugment.apply`` restates that kernel as a vectorised
gather: it is the CPU path, the path of every non-fused configuration and the tests' oracle.

Draw row of one copy (int16): (oy, ox, flip, y1, y2, x1, x2, ...) -- crop offsets in the padded image U{0..2p}, flip
in {0, 1}, then one [y1, y2) x [x1, x2) box per Cutout hole in output coordinates.  With ``resize`` the crop is resized before the flip, and "output" is the resized copy.  The distributions are the
reference's; the draws are made with one RNG call per quantity and batch, so they do not replay its per-image stream
(which depends on the DataLoader worker seeding anyway).
"""
import numpy as np
import torch

_IMAGE_STATS = {'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225]}   # preprocess.py:7-8 of the reference


class Cutout(object):
    """Zero ``holes`` square patches of side ``length`` of a normalised [C, H, W] tensor (the reference's Cutout,
    preprocess.py:185-227): centre y, x ~ np.random.randint(H | W), box [clip(y - L//2, 0, H), clip(y + L//2, 0, H))
    x the same in x; the image is multiplied by the 0/1 mask, so a cut element becomes v * 0 (a signed zero)."""

    def __init__(self, holes, length):
        self.holes = holes
        self.length = length

    def __call__(self, img):
        h, w = img.size(1), img.size(2)
        mask = np.ones((h, w), np.float32)
        for _ in range(self.holes):
            y, x = np.random.randint(h), np.random.randint(w)
            y1, y2 = np.clip(y - self.length // 2, 0, h), np.clip(y + self.length // 2, 0, h)
            x1, x2 = np.clip(x - self.length // 2, 0, w), np.clip(x + self.length // 2, 0, w)
            mask[y1:y2, x1:x2] = 0.
        return img * torch.from_numpy(mask).expand_as(img)


def normalize_lut(normalize, C):
    """fp32 [C, 256]: entry [c][u] = Normalize(ToTensor(u)) in torchvision's fp32 arithmetic -- u.float().div(255),
    then .sub(mean[c]).div(std[c])."""
    if len(normalize['mean']) < C or len(normalize['std']) < C:
        raise ValueError('normalisation statistics for fewer than %d channels' % C)
    u = torch.arange(256, dtype=torch.uint8).to(torch.float32).div(255).expand(C, 256)
    mean = torch.as_tensor(normalize['mean'][:C], dtype=torch.float32).view(C, 1)
    std = torch.as_tensor(normalize['std'][:C], dtype=torch.float32).view(C, 1)
    return u.sub(mean).div(std).contiguous()


class BatchAugment(object):
    """``duplicates`` copies per image of RandomCrop(padding) [+ Resize(``resize``), bilinear] + RandomHorizontalFlip
    (``flip``) + ToTensor + Normalize (``normalize``: {'mean', 'std'}) + Cutout (``cutout``: None or {'holes',
    'length'}).  ``resize``: None, S or (OH, OW) -- the Mix&Match CIFAR size regimes crop at the images' size and resize
    the crop (preprocess.py:44-54 of the reference with input_size != scale_size)."""

    def __init__(self, padding=4, flip=True, cutout=None, duplicates=1, normalize=None, resize=None):
        self.padding = int(padding)
        self.flip = bool(flip)
        self.holes = int(cutout['holes']) if cutout else 0
        self.length = int(cutout['length']) if cutout else 0
        self.duplicates = int(duplicates)
        self.normalize = normalize or _IMAGE_STATS
        if resize is not None:
            resize = (int(resize), int(resize)) if isinstance(resize, int) else (int(resize[0]), int(resize[1]))
        self.resize = resize
        if self.padding < 0 or self.duplicates < 1 or self.holes < 0 or self.length < 0:
            raise ValueError('BatchAugment: padding, holes and length must be >= 0 and duplicates >= 1')
        if resize is not None and min(resize) < 1:
            raise ValueError('BatchAugment: resize must be >= 1')
        self._luts = {}

    @property
    def row_len(self):
        """int16 entries per draw row."""
        return 3 + 4 * self.holes

    def sample(self, B, H, W):
        """-> int16 [B, D, 3 + 4*holes] draws for B images of H x W pixels: the crop offsets against the images, the
        Cutout boxes against the output (the resized copy when ``resize`` is set)."""
        D, p = self.duplicates, self.padding
        if max(H, W) + 2 * p > 32767:
            raise ValueError('BatchAugment: %dx%d images with padding %d do not fit the int16 draws' % (H, W, p))
        out = torch.zeros((B, D, self.row_len), dtype=torch.int16)
        out[..., 0] = torch.randint(0, 2 * p + 1, (B, D), dtype=torch.int16)       # RandomCrop.get_params: i, then j
        out[..., 1] = torch.randint(0, 2 * p + 1, (B, D), dtype=torch.int16)
        if self.flip:
            out[..., 2] = (torch.rand(B, D) < 0.5).to(torch.int16)                 # RandomHorizontalFlip: rand < p
        if self.holes:
            H, W = self.resize or (H, W)
            y = np.random.randint(H, size=(B, D, self.holes))
            x = np.random.randint(W, size=(B, D, self.holes))
            half = self.length // 2
            box = np.stack([np.clip(y - half, 0, H), np.clip(y + half, 0, H),
                            np.clip(x - half, 0, W), np.clip(x + half, 0, W)], axis=-1)
            out[..., 3:] = torch.from_numpy(box.reshape(B, D, 4 * self.holes).astype(np.int16))
        return out

    def lut(self, C):
        """fp32 [C, 256]: entry [c][u] = Normalize(ToTensor(u)) in torchvision's fp32 arithmetic -- u.float().div(255),
        then .sub(mean[c]).div(std[c])."""
        t = self._luts.get(C)
        if t is None:
            t = self._luts[C] = normalize_lut(self.normalize, C)
        return t

    def apply(self, images, params):
        """uint8 NHWC [B, H, W, C] images and [B, D, P] (or [B*D, P]) draws -> fp32 NCHW [B*D, C, H, W] on the images'
        device: row b*D + d is copy d of image b, as the reference's transform computes it."""
        B, H, W, C = images.shape
        dev = images.device
        p = params.reshape(-1, params.shape[-1]).to(dev, torch.long)
        N = p.shape[0]
        if N % B or (p.shape[1] - 3) % 4:
            raise ValueError('BatchAugment.apply: draws %s do not match %d images' % (tuple(params.shape), B))
        D, holes = N // B, (p.shape[1] - 3) // 4
        if self.resize is not None:
            return self._apply_resized(images.cpu(), p.cpu(), D, holes).to(dev)
        r, c = torch.arange(H, device=dev), torch.arange(W, device=dev)
        sy = r + p[:, 0:1] - self.padding                                           # [N, H]
        sx = torch.where(p[:, 2:3] != 0, W - 1 - c, c) + p[:, 1:2] - self.padding   # [N, W]
        ok = ((sy >= 0) & (sy < H))[:, :, None] & ((sx >= 0) & (sx < W))[:, None, :]
        src = torch.arange(N, device=dev).div(D, rounding_mode='floor')
        pix = (src[:, None, None] * H + sy.clamp(0, H - 1)[:, :, None]) * W + sx.clamp(0, W - 1)[:, None, :]
        u = images.reshape(-1, C)[pix].masked_fill(~ok[..., None], 0)              # [N, H, W, C], pad value 0
        v = self.lut(C).to(dev)[torch.arange(C, device=dev), u.long()]              # [N, H, W, C]
        v = v.permute(0, 3, 1, 2).contiguous()
        if holes:
            mask = torch.ones((N, H, W), dtype=torch.float32, device=dev)
            for h in range(holes):
                y1, y2, x1, x2 = (p[:, 3 + 4 * h + k].view(N, 1, 1) for k in range(4))
                inside = (r.view(1, H, 1) >= y1) & (r.view(1, H, 1) < y2) & (c.view(1, 1, W) >= x1) & \
                    (c.view(1, 1, W) < x2)
                mask.masked_fill_(inside, 0.)
            v = v * mask[:, None]
        return v

    def _apply_resized(self, images, p, D, holes):
        """The resizing form of apply(), -> fp32 NCHW [B*D, C, OH, OW]: torchvision's own pad / crop / resize / hflip /
        to_tensor / normalize on PIL images and the reference's Cutout mask (its arithmetic by construction).  Three
        channels make one RGB image; any other count is resampled channel by channel (the filter does not mix them)."""
        import torchvision.transforms.functional as F
        from PIL import Image
        from torchvision.transforms import InterpolationMode
        B, H, W, C = images.shape
        OH, OW = self.resize
        mean, std = list(self.normalize['mean'][:C]), list(self.normalize['std'][:C])
        if len(mean) < C or len(std) < C:
            raise ValueError('normalisation statistics for fewer than %d channels' % C)
        planes = [(slice(0, 3), 'RGB')] if C == 3 else [(c, 'L') for c in range(C)]
        out = []
        for b in range(B):
            px = images[b].numpy()
            padded = [F.pad(Image.fromarray(np.ascontiguousarray(px[:, :, sel]), mode), self.padding)
                      for sel, mode in planes]
            for d in range(D):
                row = [int(v) for v in p[b * D + d]]
                chans = []
                for img in padded:
                    t = F.resize(F.crop(img, row[0], row[1], H, W), [OH, OW], InterpolationMode.BILINEAR)
                    chans.append(F.to_tensor(F.hflip(t) if row[2] else t))
                t = F.normalize(torch.cat(chans), mean, std)
                if holes:
                    mask = np.ones((OH, OW), np.float32)
                    for h in range(holes):
                        y1, y2, x1, x2 = (min(max(v, 0), lim) for v, lim in zip(row[3 + 4 * h:7 + 4 * h],
                                                                                 (OH, OH, OW, OW)))
                        mask[y1:y2, x1:x2] = 0.
                    t = t * torch.from_numpy(mask).expand_as(t)
                out.append(t)
        return torch.stack(out)


class DeviceBatch(object):
    """What a device-augmenting loader yields in place of the fp32 batch.  ``rows``: the number of training rows it
    stands for; ``apply()``: that fp32 NCHW batch, computed on the host (every non-fused path and the tests' oracle);
    ``pin_memory()``; ``tensors``: the host tensors the device needs, which ``replace`` swaps for their device copies."""
    __slots__ = ()

    def pin_memory(self):
        return self.replace(tuple(t.pin_memory() for t in self.tensors))


class AugmentedBatch(DeviceBatch):
    """The B uint8 NHWC ``images`` and the int16 ``params`` [B, D, P] of ``spec`` (a BatchAugment).  The batch stands
    for spec.duplicates * B rows."""
    __slots__ = ('images', 'params', 'spec')

    def __init__(self, images, params, spec):
        self.images, self.params, self.spec = images, params, spec

    @property
    def rows(self):
        return self.images.shape[0] * self.spec.duplicates

    def apply(self):
        """-> fp32 NCHW [B*D, C, H, W] on the images' device."""
        return self.spec.apply(self.images, self.params)

    @property
    def tensors(self):
        return (self.images, self.params)

    def replace(self, tensors):
        return AugmentedBatch(tensors[0], tensors[1], self.spec)


class AugmentCollate(object):
    """DataLoader ``collate_fn`` of a device-augmenting loader: stacks the (uint8 HWC image, label) samples and draws
    the batch's augmentation in the worker, where the reference draws it.  -> (AugmentedBatch, target repeated to B*D,
    row b*D + d)."""

    def __init__(self, spec):
        self.spec = spec

    def __call__(self, batch):
        images = torch.stack([torch.as_tensor(img) for img, _ in batch])
        target = torch.as_tensor([int(t) for _, t in batch], dtype=torch.long)
        B, H, W, _ = images.shape
        return AugmentedBatch(images, self.spec.sample(B, H, W), self.spec), \
            target.repeat_interleave(self.spec.duplicates)


# ---------------------------------------------------------------------------------------------------------------------
# RandomResizedCrop on the device (the ImageNet training transform, preprocess.py:71-77 of the reference).  The loader
# workers decode and draw; each image ships only its region -- the bounding box of its D crop boxes -- in one flat
# uint8 buffer, and the stem relayout kernel resamples, flips and normalises (ops.input_prep_u8_rrc).

class ResizedCrop(object):
    """``duplicates`` copies per image of RandomResizedCrop(size, scale, ratio) (bilinear) + RandomHorizontalFlip +
    ToTensor + Normalize (``normalize``: {'mean', 'std'})."""

    def __init__(self, size, duplicates=1, normalize=None, scale=(0.08, 1.0), ratio=(3. / 4., 4. / 3.)):
        self.size = (int(size), int(size)) if isinstance(size, int) else (int(size[0]), int(size[1]))
        self.duplicates = int(duplicates)
        self.normalize = normalize or _IMAGE_STATS
        self.scale, self.ratio = scale, ratio
        if self.duplicates < 1 or min(self.size) < 1:
            raise ValueError('ResizedCrop: duplicates and size must be >= 1')
        self._luts = {}

    def lut(self, C):
        t = self._luts.get(C)
        if t is None:
            t = self._luts[C] = normalize_lut(self.normalize, C)
        return t

    def draw(self, img):
        """int32 [D, 5] crop boxes {top, left, height, width, flip} in the coordinates of ``img`` (a PIL image): for
        each copy RandomResizedCrop.get_params, then torch.rand(1) < 0.5 -- the reference transform's calls in its
        order, so equal seeds give its per-image stream."""
        import torchvision.transforms as T
        out = torch.empty((self.duplicates, 5), dtype=torch.int32)
        for d in range(self.duplicates):
            i, j, h, w = T.RandomResizedCrop.get_params(img, self.scale, self.ratio)
            out[d] = torch.tensor([i, j, h, w, int(torch.rand(1) < 0.5)], dtype=torch.int32)
        return out

    def __call__(self, img):
        """PIL image -> (uint8 HWC region, int32 [D, 5] draws relative to the region): the loader's per-image work."""
        draws = self.draw(img)
        y0, x0 = int(draws[:, 0].min()), int(draws[:, 1].min())
        y1, x1 = int((draws[:, 0] + draws[:, 2]).max()), int((draws[:, 1] + draws[:, 3]).max())
        a = np.asarray(img)
        region = torch.from_numpy(np.array(a[y0:y1, x0:x1].reshape(y1 - y0, x1 - x0, -1), copy=True))
        draws[:, 0] -= y0
        draws[:, 1] -= x0
        return region, draws

    def apply(self, regions, index, draws, C):
        """-> fp32 NCHW [B*D, C, OH, OW]: torchvision's own resized_crop / hflip / to_tensor / normalize on PIL images
        built from the C-channel regions (the reference's arithmetic by construction)."""
        import torchvision.transforms.functional as F
        from PIL import Image
        from torchvision.transforms import InterpolationMode
        D = draws.shape[0] // index.shape[0]
        regions = regions.cpu()
        out = []
        for b in range(index.shape[0]):
            off, h, w = (int(v) for v in index[b])
            px = regions[off:off + h * w * C].reshape(h, w, C).numpy()
            img = Image.fromarray(px[:, :, 0] if C == 1 else px, 'L' if C == 1 else 'RGB')
            for d in range(D):
                y, x, ch, cw, flip = (int(v) for v in draws[b * D + d])
                t = F.resized_crop(img, y, x, ch, cw, list(self.size), InterpolationMode.BILINEAR)
                if flip:
                    t = F.hflip(t)
                out.append(F.normalize(F.to_tensor(t), **self.normalize))
        return torch.stack(out)


class ResizedCropBatch(DeviceBatch):
    """B images' regions in one flat uint8 buffer ``regions`` (HWC, ``channels`` per pixel, the first ``nbytes`` bytes
    in use), ``index`` int64 [B, 3] {byte offset, h, w} and ``draws`` int32 [B*D, 5] {y, x, h, w, flip} of ``spec`` (a
    ResizedCrop) relative to each region.  Stands for B*D rows, row b*D + d = copy d of image b.  ``host`` keeps the CPU
    index and draws once the tensors have been staged on a device (their validation needs no device read-back)."""
    __slots__ = ('regions', 'index', 'draws', 'spec', 'channels', 'nbytes', 'host')

    def __init__(self, regions, index, draws, spec, channels, nbytes=None, host=None):
        self.regions, self.index, self.draws, self.spec = regions, index, draws, spec
        self.channels = int(channels)
        self.nbytes = int(regions.numel() if nbytes is None else nbytes)
        self.host = host if host is not None else (index, draws)

    @property
    def rows(self):
        return self.draws.shape[0]

    def apply(self):
        """-> fp32 NCHW [B*D, C, OH, OW] on the host."""
        return self.spec.apply(self.regions[:self.nbytes], self.host[0], self.host[1], self.channels)

    @property
    def tensors(self):
        return (self.regions, self.index, self.draws)

    def replace(self, tensors):
        return ResizedCropBatch(tensors[0], tensors[1], tensors[2], self.spec, self.channels, self.nbytes, self.host)


class ResizedCropCollate(object):
    """DataLoader ``collate_fn`` of a resized-crop loader: packs the (region, draws) samples made by ResizedCrop in the
    workers into one ResizedCropBatch.  -> (batch, target repeated to B*D, row b*D + d)."""

    def __init__(self, spec):
        self.spec = spec

    def __call__(self, batch):
        regions = [r for (r, _), _ in batch]
        sizes = [r.numel() for r in regions]
        offsets = [0]
        for s in sizes[:-1]:
            offsets.append(offsets[-1] + s)
        index = torch.tensor([[o, r.shape[0], r.shape[1]] for o, r in zip(offsets, regions)], dtype=torch.int64)
        draws = torch.cat([d for (_, d), _ in batch])
        target = torch.as_tensor([int(t) for _, t in batch], dtype=torch.long)
        flat = torch.cat([r.reshape(-1) for r in regions])
        return ResizedCropBatch(flat, index, draws, self.spec, regions[0].shape[2]), \
            target.repeat_interleave(self.spec.duplicates)


# ---------------------------------------------------------------------------------------------------------------------
# Resize + CenterCrop on the device (the ImageNet evaluation transform, the reference's scale_crop, preprocess.py:20-41,
# one crop).  The loader workers decode; each image ships only its support region -- the source pixels the crop
# window's filter taps touch -- in one flat uint8 buffer, and the stem relayout kernel resamples the window of the
# whole image's resize and normalises it (ops.input_prep_u8_scale_crop).

def resample_taps(n_in, n_out, i):
    """[first, end) source indices of output index ``i`` of Pillow's BILINEAR n_in -> n_out resample (ImagingResample's
    bounds, in the double arithmetic the relayout kernel uses)."""
    scale = n_in / n_out
    support = scale if scale >= 1.0 else 1.0
    center = (i + 0.5) * scale
    return max(int(center - support + 0.5), 0), min(int(center + support + 0.5), n_in)


def crop_support(n_in, n_resized, start, n_out):
    """[first, end) source indices that output indices start .. start + n_out - 1 of an n_in -> n_resized resample read
    (indices outside [0, n_resized) are padding and read nothing), or None when every index is padding."""
    a, b = max(start, 0), min(start + n_out, n_resized)
    if a >= b:
        return None
    return resample_taps(n_in, n_resized, a)[0], resample_taps(n_in, n_resized, b - 1)[1]


class ScaleCrop(object):
    """Resize(scale_size) (bilinear; skipped when scale_size == input_size) + CenterCrop(input_size) + ToTensor +
    Normalize (``normalize``: {'mean', 'std'}): the reference's scale_crop."""

    margin = 1      # source pixels shipped beyond the taps on each side (clamped to the image)

    def __init__(self, input_size, scale_size=None, normalize=None):
        self.input_size = int(input_size)
        self.size = (self.input_size, self.input_size)
        self.scale_size = int(scale_size) if scale_size is not None else int(self.input_size * 8 / 7)
        self.normalize = normalize or _IMAGE_STATS
        if min(self.size) < 1 or self.scale_size < 1:
            raise ValueError('ScaleCrop: input_size and scale_size must be >= 1')
        self._luts = {}

    def lut(self, C):
        t = self._luts.get(C)
        if t is None:
            t = self._luts[C] = normalize_lut(self.normalize, C)
        return t

    def resized_size(self, h, w):
        """(RH, RW) of Resize(scale_size) on an h x w image: torchvision's _compute_resized_output_size (short side to
        scale_size, long side int(scale_size * long / short)); (h, w) when scale_size == input_size (no Resize)."""
        if self.scale_size == self.input_size:
            return h, w
        short, long = (w, h) if w <= h else (h, w)
        new_short, new_long = self.scale_size, int(self.scale_size * long / short)
        return (new_long, new_short) if w <= h else (new_short, new_long)

    def geometry(self, h, w):
        """int32 [8] {y0, x0, H, W, RH, RW, top, left} and the support region's (h, w) of an h x w image: the crop
        origin in the resized image as CenterCrop computes it (int(round((RH - th) / 2.0)), or minus the top / left
        padding when the crop is larger), the region the window's taps touch plus ``margin``."""
        th, tw = self.size
        rh, rw = self.resized_size(h, w)
        top = -((th - rh) // 2) if th > rh else int(round((rh - th) / 2.0))
        left = -((tw - rw) // 2) if tw > rw else int(round((rw - tw) / 2.0))
        spans = []
        for n, nr, start, n_out in ((h, rh, top, th), (w, rw, left, tw)):
            s = crop_support(n, nr, start, n_out)
            lo, hi = (0, 1) if s is None else (max(s[0] - self.margin, 0), min(s[1] + self.margin, n))
            spans.append((lo, hi))
        (y0, y1), (x0, x1) = spans
        return torch.tensor([y0, x0, h, w, rh, rw, top, left], dtype=torch.int32), (y1 - y0, x1 - x0)

    def __call__(self, img):
        """PIL image -> (uint8 HWC support region, int32 [8] geometry): the loader's per-image work."""
        w, h = img.size
        geom, (rh, rw) = self.geometry(h, w)
        y0, x0 = int(geom[0]), int(geom[1])
        a = np.asarray(img)
        region = torch.from_numpy(np.array(a[y0:y0 + rh, x0:x0 + rw].reshape(rh, rw, -1), copy=True))
        return region, geom

    def apply(self, regions, index, geom, C):
        """-> fp32 NCHW [B, C, OH, OW]: each region pasted at (y0, x0) into a zero image of the original size, then
        torchvision's own resize / center_crop / to_tensor / normalize on PIL images.  Pixels outside the support region
        carry zero weight, so this is the reference's output (its arithmetic by construction).  Three channels make one
        RGB image; any other count is resampled channel by channel (the filter does not mix them)."""
        import torchvision.transforms.functional as F
        from PIL import Image
        from torchvision.transforms import InterpolationMode
        regions = regions.cpu()
        mean, std = list(self.normalize['mean'][:C]), list(self.normalize['std'][:C])
        if len(mean) < C or len(std) < C:
            raise ValueError('normalisation statistics for fewer than %d channels' % C)
        out = []
        for b in range(index.shape[0]):
            off, h, w = (int(v) for v in index[b])
            y0, x0, H, W = (int(v) for v in geom[b][:4])
            full = np.zeros((H, W, C), np.uint8)
            full[y0:y0 + h, x0:x0 + w] = regions[off:off + h * w * C].reshape(h, w, C).numpy()
            planes = [Image.fromarray(full, 'RGB')] if C == 3 else \
                [Image.fromarray(np.ascontiguousarray(full[:, :, c]), 'L') for c in range(C)]
            chans = []
            for img in planes:
                if self.scale_size != self.input_size:
                    img = F.resize(img, self.scale_size, InterpolationMode.BILINEAR)
                chans.append(F.to_tensor(F.center_crop(img, list(self.size))))
            out.append(F.normalize(torch.cat(chans), mean, std))
        return torch.stack(out)


class ScaleCropBatch(DeviceBatch):
    """B images' support regions in one flat uint8 buffer ``regions`` (HWC, ``channels`` per pixel, the first ``nbytes``
    bytes in use), ``index`` int64 [B, 3] {byte offset, h, w} and ``geom`` int32 [B, 8] {y0, x0, H, W, RH, RW, top,
    left} of ``spec`` (a ScaleCrop).  Stands for B rows.  ``host`` keeps the CPU index and geometry once the tensors
    have been staged on a device (their validation needs no device read-back)."""
    __slots__ = ('regions', 'index', 'geom', 'spec', 'channels', 'nbytes', 'host')

    def __init__(self, regions, index, geom, spec, channels, nbytes=None, host=None):
        self.regions, self.index, self.geom, self.spec = regions, index, geom, spec
        self.channels = int(channels)
        self.nbytes = int(regions.numel() if nbytes is None else nbytes)
        self.host = host if host is not None else (index, geom)

    @property
    def rows(self):
        return self.index.shape[0]

    def apply(self):
        """-> fp32 NCHW [B, C, OH, OW] on the host."""
        return self.spec.apply(self.regions[:self.nbytes], self.host[0], self.host[1], self.channels)

    @property
    def tensors(self):
        return (self.regions, self.index, self.geom)

    def replace(self, tensors):
        return ScaleCropBatch(tensors[0], tensors[1], tensors[2], self.spec, self.channels, self.nbytes, self.host)


class ScaleCropCollate(object):
    """DataLoader ``collate_fn`` of a scale-crop loader: packs the (region, geometry) samples made by ScaleCrop in the
    workers into one ScaleCropBatch.  -> (batch, target)."""

    def __init__(self, spec):
        self.spec = spec

    def __call__(self, batch):
        regions = [r for (r, _), _ in batch]
        offsets = [0]
        for r in regions[:-1]:
            offsets.append(offsets[-1] + r.numel())
        index = torch.tensor([[o, r.shape[0], r.shape[1]] for o, r in zip(offsets, regions)], dtype=torch.int64)
        geom = torch.stack([g for (_, g), _ in batch])
        target = torch.as_tensor([int(t) for _, t in batch], dtype=torch.long)
        flat = torch.cat([r.reshape(-1) for r in regions])
        return ScaleCropBatch(flat, index, geom, self.spec, regions[0].shape[2]), target
