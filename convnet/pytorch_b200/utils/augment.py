"""Batch augmentation ("Augment Your Batch", Hoffer et al., CVPR 2020) of the CIFAR training transform, drawn on the
host and applied on the device.

The reference runs the whole PIL transform D times per sample in the loader workers (preprocess.py:44-54,105-112):
RandomCrop(size, padding) -> RandomHorizontalFlip -> ToTensor -> Normalize [-> Cutout], and the trainer flattens the
[B, D, C, H, W] batch to B*D rows, row b*D + d (trainer.py:17-29).  Here the loader ships the B un-augmented uint8
images with a small table of per-copy draws (an ``AugmentedBatch``) and the stem relayout kernel writes the B*D
augmented, normalised copies (ops.input_prep_u8_aug).  ``BatchAugment.apply`` restates that kernel as a vectorised
gather: it is the CPU path, the path of every non-fused configuration and the tests' oracle.

Draw row of one copy (int16): (oy, ox, flip, y1, y2, x1, x2, ...) -- crop offsets in the padded image U{0..2p}, flip
in {0, 1}, then one [y1, y2) x [x1, x2) box per Cutout hole in output coordinates.  The distributions are the
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


class BatchAugment(object):
    """``duplicates`` copies per image of RandomCrop(padding) + RandomHorizontalFlip (``flip``) + ToTensor + Normalize
    (``normalize``: {'mean', 'std'}) + Cutout (``cutout``: None or {'holes', 'length'})."""

    def __init__(self, padding=4, flip=True, cutout=None, duplicates=1, normalize=None):
        self.padding = int(padding)
        self.flip = bool(flip)
        self.holes = int(cutout['holes']) if cutout else 0
        self.length = int(cutout['length']) if cutout else 0
        self.duplicates = int(duplicates)
        self.normalize = normalize or _IMAGE_STATS
        if self.padding < 0 or self.duplicates < 1 or self.holes < 0 or self.length < 0:
            raise ValueError('BatchAugment: padding, holes and length must be >= 0 and duplicates >= 1')
        self._luts = {}

    @property
    def row_len(self):
        """int16 entries per draw row."""
        return 3 + 4 * self.holes

    def sample(self, B, H, W):
        """-> int16 [B, D, 3 + 4*holes] draws for B images of H x W pixels."""
        D, p = self.duplicates, self.padding
        if max(H, W) + 2 * p > 32767:
            raise ValueError('BatchAugment: %dx%d images with padding %d do not fit the int16 draws' % (H, W, p))
        out = torch.zeros((B, D, self.row_len), dtype=torch.int16)
        out[..., 0] = torch.randint(0, 2 * p + 1, (B, D), dtype=torch.int16)       # RandomCrop.get_params: i, then j
        out[..., 1] = torch.randint(0, 2 * p + 1, (B, D), dtype=torch.int16)
        if self.flip:
            out[..., 2] = (torch.rand(B, D) < 0.5).to(torch.int16)                 # RandomHorizontalFlip: rand < p
        if self.holes:
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
            if len(self.normalize['mean']) < C or len(self.normalize['std']) < C:
                raise ValueError('BatchAugment: normalisation statistics for fewer than %d channels' % C)
            u = torch.arange(256, dtype=torch.uint8).to(torch.float32).div(255).expand(C, 256)
            mean = torch.as_tensor(self.normalize['mean'][:C], dtype=torch.float32).view(C, 1)
            std = torch.as_tensor(self.normalize['std'][:C], dtype=torch.float32).view(C, 1)
            t = self._luts[C] = u.sub(mean).div(std).contiguous()
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


class AugmentedBatch(object):
    """What a device-augmenting loader yields in place of the [B, D, C, H, W] batch: the B uint8 NHWC ``images``, the
    int16 ``params`` [B, D, P] of ``spec`` (a BatchAugment).  The batch stands for spec.duplicates * B rows."""
    __slots__ = ('images', 'params', 'spec')

    def __init__(self, images, params, spec):
        self.images, self.params, self.spec = images, params, spec

    @property
    def rows(self):
        return self.images.shape[0] * self.spec.duplicates

    def apply(self):
        """-> fp32 NCHW [B*D, C, H, W] on the images' device."""
        return self.spec.apply(self.images, self.params)

    def pin_memory(self):
        return AugmentedBatch(self.images.pin_memory(), self.params.pin_memory(), self.spec)


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
