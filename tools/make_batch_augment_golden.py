"""Generates tests/golden/batch_augment.npz from the UNMODIFIED reference CIFAR training transform with batch
augmentation and Cutout (a checkout of eladhoffer/convNet.pytorch, read-only).  Run once from the repo root:

    B200_REFERENCE=<reference checkout> python tools/make_batch_augment_golden.py

The transform is the reference's get_transform('cifar10', augment=True, cutout={'holes': 1, 'length': 16},
duplicates=8): per copy RandomCrop(32, padding=4) -> RandomHorizontalFlip -> ToTensor -> Normalize -> Cutout, the 8
copies stacked.  It runs on IMAGES seeded uint8 32x32 RGB images, in order, in this process (what a DataLoader with
num_workers=0 does), after seeding torch and numpy with SEED.

Every copy's draws are recovered by replaying the generator calls the transform made: torch.randint (crop row),
torch.randint (crop column), torch.rand (flip), then numpy randint (centre row), randint (centre column); the replay must
end in the same generator states as the transform did.  The fixture stores the images, the draws as the int16 rows of
utils/augment.py (oy, ox, flip, y1, y2, x1, x2) and the SHA-256 of every augmented fp32 [3, 32, 32] copy.  The seed is
the first from SEED upwards whose draws cover crop offsets 0 and 8 in both axes, both flip values and boxes clipped
at each of the four edges.
"""
import hashlib
import os
import sys

import numpy as np
import torch

REF = os.environ.get('B200_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden',
                   'batch_augment.npz')
IMAGES, DUPLICATES, PAD, HOLES, LENGTH, SIZE = 8, 8, 4, 1, 16, 32
SEED = 2020


def digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


def replay_draws(n):
    """The draws of n transform copies, replayed from the current generator states (which it advances)."""
    rows = []
    for _ in range(n):
        oy = torch.randint(0, 2 * PAD + 1, size=(1,)).item()
        ox = torch.randint(0, 2 * PAD + 1, size=(1,)).item()
        flip = int(torch.rand(1) < 0.5)
        y, x = np.random.randint(SIZE), np.random.randint(SIZE)
        half = LENGTH // 2
        rows.append([oy, ox, flip, np.clip(y - half, 0, SIZE), np.clip(y + half, 0, SIZE),
                     np.clip(x - half, 0, SIZE), np.clip(x + half, 0, SIZE)])
    return rows


def run(seed, images, transform):
    from PIL import Image
    torch.manual_seed(seed)
    np.random.seed(seed)
    draws, hashes = [], []
    for img in images:
        t_state, n_state = torch.get_rng_state(), np.random.get_state()
        out = transform(Image.fromarray(img))
        t_after, n_after = torch.get_rng_state(), np.random.get_state()
        torch.set_rng_state(t_state)
        np.random.set_state(n_state)
        draws.append(replay_draws(DUPLICATES))
        assert torch.equal(torch.get_rng_state(), t_after), 'torch draws not replayed'
        assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), n_after)), 'numpy draws not replayed'
        assert out.shape == (DUPLICATES, 3, SIZE, SIZE) and out.dtype == torch.float32
        hashes.extend(digest(c) for c in out)
    return np.asarray(draws, dtype=np.int16), hashes


def covered(d):
    return {0, 2 * PAD} <= set(d[..., 0].ravel()) and {0, 2 * PAD} <= set(d[..., 1].ravel()) \
        and {0, 1} <= set(d[..., 2].ravel()) and (d[..., 3] == 0).any() and (d[..., 4] == SIZE).any() \
        and (d[..., 5] == 0).any() and (d[..., 6] == SIZE).any()


def main():
    if not REF or not os.path.isdir(REF):
        sys.exit('set B200_REFERENCE to a checkout of the reference repository')
    sys.path.insert(0, REF)
    import preprocess
    transform = preprocess.get_transform('cifar10', augment=True, cutout={'holes': HOLES, 'length': LENGTH},
                                         duplicates=DUPLICATES)
    g = torch.Generator().manual_seed(7)
    images = torch.randint(0, 256, (IMAGES, SIZE, SIZE, 3), generator=g, dtype=torch.uint8).numpy()
    seed = SEED
    while True:
        draws, hashes = run(seed, images, transform)
        if covered(draws):
            break
        seed += 1
    np.savez_compressed(OUT, images=images, draws=draws, sha256=np.asarray(hashes), seed=np.int64(seed),
                        padding=np.int64(PAD), holes=np.int64(HOLES), length=np.int64(LENGTH))
    print('wrote %s: seed %d, %d copies' % (OUT, seed, len(hashes)))


if __name__ == '__main__':
    main()
