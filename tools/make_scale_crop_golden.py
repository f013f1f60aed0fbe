"""Generates tests/golden/scale_crop.npz from the UNMODIFIED reference ImageNet evaluation transform (a checkout of
eladhoffer/convNet.pytorch, read-only).  Run once from the repo root:

    B200_REFERENCE=<reference checkout> python tools/make_scale_crop_golden.py

The transform is the reference's preprocess.scale_crop(input_size, scale_size): [Resize(scale_size) when it differs
from input_size] -> CenterCrop(input_size) -> ToTensor -> Normalize.  Each case is one seeded uniform uint8 image
(make_image below; RGB or L) of a chosen size.  The cases cover landscape, portrait and square images, an image whose
short side already is scale_size, images smaller than the crop with scale_size == input_size (CenterCrop pads), an
upscale, a downscale with more than 16 taps, odd (h - th) / (w - tw) (round half to even) and the (input, scale) pairs
of the ImageNet models' evaluation sizes.  The fixture stores the sizes, modes, seeds and the SHA-256 of every fp32
[C, input, input] output.
"""
import hashlib
import os
import sys

import numpy as np
import torch

REF = os.environ.get('B200_REFERENCE', '')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'scale_crop.npz')

# (input_size, scale_size, image h, image w, mode)
CASES = [
    (224, 256, 375, 500, 'RGB'),      # landscape; resized 256 x 341: left = round(58.5) = 58 (half to even)
    (224, 256, 500, 375, 'RGB'),      # portrait
    (224, 256, 300, 300, 'RGB'),      # square
    (224, 256, 256, 341, 'RGB'),      # already at scale_size: Resize is the identity
    (224, 224, 150, 200, 'RGB'),      # smaller than the crop, no Resize: padded on both axes
    (224, 224, 301, 180, 'L'),        # padded in width only; top = round(38.5) = 38
    (224, 256, 100, 120, 'RGB'),      # upscale
    (224, 256, 2000, 2300, 'RGB'),    # downscale with more than 16 taps per output pixel
    (128, 146, 333, 417, 'L'),
    (288, 329, 480, 640, 'RGB'),
    (64, 73, 375, 500, 'RGB'),
    (64, 73, 211, 97, 'L'),
    (224, 224, 224, 224, 'RGB'),      # the identity
    (224, 224, 225, 226, 'RGB'),      # odd and even one-pixel crops, no Resize
]


def make_image(h, w, mode, seed):
    """uniform uint8 PIL image of h x w pixels (3 channels for RGB, 1 for L) from torch.Generator(seed)"""
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    c = 3 if mode == 'RGB' else 1
    a = torch.randint(0, 256, (h, w, c), generator=g, dtype=torch.uint8).numpy()
    return Image.fromarray(a if c == 3 else a[:, :, 0], mode)


def digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


def main():
    if not REF or not os.path.isdir(REF):
        sys.exit('set B200_REFERENCE to a checkout of the reference')
    sys.path.insert(0, REF)
    from preprocess import scale_crop                                     # the reference's, unmodified
    hashes, seeds = [], []
    for k, (size, scale, h, w, mode) in enumerate(CASES):
        seed = 1000 + k
        c = 3 if mode == 'RGB' else 1
        stats = {'mean': [0.485, 0.456, 0.406][:c], 'std': [0.229, 0.224, 0.225][:c]}
        out = scale_crop(input_size=size, scale_size=scale, normalize=stats)(make_image(h, w, mode, seed))
        assert tuple(out.shape) == (c, size, size)
        hashes.append(digest(out))
        seeds.append(seed)
    np.savez_compressed(OUT, cases=np.array([c[:4] for c in CASES], dtype=np.int32),
                        modes=np.array([c[4] for c in CASES]), seeds=np.array(seeds, dtype=np.int64),
                        sha256=np.array(hashes))
    print('wrote %s (%d cases)' % (OUT, len(hashes)))


if __name__ == '__main__':
    main()
