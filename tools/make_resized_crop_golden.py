"""Generates tests/golden/resized_crop.npz from the UNMODIFIED reference ImageNet training transform with batch
augmentation (a checkout of eladhoffer/convNet.pytorch, read-only).  Run once from the repo root:

    B200_REFERENCE=<reference checkout> python tools/make_resized_crop_golden.py

The transform is the reference's get_transform('imagenet', input_size=SIZE, augment=True, duplicates=DUPLICATES): per
copy RandomResizedCrop(SIZE) -> RandomHorizontalFlip -> ToTensor -> Normalize, the copies stacked.  It runs on the
first IMAGES images of data.synthetic_imagenet_pool() (seeded uniform RGB images of 200-600 px), in order, in this
process (what a DataLoader with num_workers=0 does), after torch.manual_seed(SEED).

Every copy's draws are recovered by replaying the generator calls the transform made --
RandomResizedCrop.get_params(img, (0.08, 1.0), (3/4, 4/3)), then torch.rand(1) < 0.5 -- and the replay must end in
the same generator state as the transform did.  The fixture stores the image sizes, the draws {top, left, height,
width, flip} in image coordinates and the SHA-256 of every fp32 [3, SIZE, SIZE] copy.
"""
import hashlib
import os
import sys

import numpy as np
import torch

REF = os.environ.get('B200_REFERENCE', '')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, 'tests', 'golden', 'resized_crop.npz')
IMAGES, DUPLICATES, SIZE, SEED = 12, 3, 224, 2024


def digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


def main():
    if not REF or not os.path.isdir(REF):
        sys.exit('set B200_REFERENCE to a checkout of the reference')
    sys.path.insert(0, REF)
    sys.path.insert(0, ROOT)
    import torchvision.transforms as T
    from preprocess import get_transform                                  # the reference's, unmodified
    from convnet.pytorch_b200.data import synthetic_imagenet_pool
    images = synthetic_imagenet_pool()[:IMAGES]
    transform = get_transform('imagenet', input_size=SIZE, augment=True, duplicates=DUPLICATES)
    torch.manual_seed(SEED)
    draws, hashes = [], []
    for img in images:
        state = torch.get_rng_state()
        out = transform(img)
        after = torch.get_rng_state()
        torch.set_rng_state(state)
        for _ in range(DUPLICATES):
            i, j, h, w = T.RandomResizedCrop.get_params(img, (0.08, 1.0), (3. / 4., 4. / 3.))
            draws.append([i, j, h, w, int(torch.rand(1) < 0.5)])
        assert torch.equal(torch.get_rng_state(), after), 'the replay did not follow the transform'
        hashes += [digest(c) for c in out]
    d = np.array(draws, dtype=np.int32)
    print('scales: %s, flips: %d of %d' % (np.round(d[:, 2] * d[:, 3] / np.repeat([im.size[0] * im.size[1] for im in
                                                                                   images], DUPLICATES), 3).tolist(),
                                          int(d[:, 4].sum()), len(d)))
    np.savez_compressed(OUT, seed=SEED, size=SIZE, duplicates=DUPLICATES,
                        image_hw=np.array([[im.size[1], im.size[0]] for im in images], dtype=np.int32), draws=d,
                        sha256=np.array(hashes))
    print('wrote %s (%d copies)' % (OUT, len(hashes)))


if __name__ == '__main__':
    main()
