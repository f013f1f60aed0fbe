"""Generates tests/golden/mixsize_augment.npz from the UNMODIFIED reference CIFAR training transform of the Mix&Match
size regimes (a checkout of eladhoffer/convNet.pytorch, read-only).  Run once from the repo root:

    B200_REFERENCE=<reference checkout> python tools/make_mixsize_golden.py

For every (input size S, duplicates D, Cutout) of CONFIGS the transform is the reference's get_transform('cifar10',
input_size=S, scale_size=32, augment=True, duplicates=D, cutout=...): per copy RandomCrop(32, padding=4) -> Resize(S)
-> RandomHorizontalFlip -> ToTensor -> Normalize [-> Cutout], the copies stacked.  It runs on IMAGES seeded uniform
uint8 32x32 RGB images, in order, in this process (what a DataLoader with num_workers=0 does), after seeding torch and
numpy with SEED.

Every copy's draws are recovered by replaying the generator calls the transform made: torch.randint (crop row),
torch.randint (crop column), torch.rand (flip), then per Cutout hole numpy randint (centre row), randint (centre
column) over the S x S output; the replay must end in the same generator states as the transform did.  The fixture
stores the images and, per configuration, the draws as the int16 rows of utils/augment.py (oy, ox, flip, y1, y2, x1,
x2; boxes in output coordinates) and the SHA-256 of every fp32 [3, S, S] copy.
"""
import hashlib
import os
import sys

import numpy as np
import torch

REF = os.environ.get('B200_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden',
                   'mixsize_augment.npz')
IMAGES, PAD, SCALE, SEED = 12, 4, 32, 2021
CONFIGS = [(16, 4, {'holes': 1, 'length': 8}), (24, 2, None), (48, 1, {'holes': 1, 'length': 16})]   # S, D, cutout


def digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


def replay_draws(n, size, cutout):
    """The draws of n transform copies, replayed from the current generator states (which it advances)."""
    rows = []
    for _ in range(n):
        row = [torch.randint(0, 2 * PAD + 1, size=(1,)).item(), torch.randint(0, 2 * PAD + 1, size=(1,)).item(),
               int(torch.rand(1) < 0.5)]
        for _ in range(cutout['holes'] if cutout else 0):
            y, x = np.random.randint(size), np.random.randint(size)
            half = cutout['length'] // 2
            row += [np.clip(y - half, 0, size), np.clip(y + half, 0, size),
                    np.clip(x - half, 0, size), np.clip(x + half, 0, size)]
        rows.append(row)
    return rows


def run(images, size, duplicates, cutout, transform):
    from PIL import Image
    torch.manual_seed(SEED + size)
    np.random.seed(SEED + size)
    draws, hashes = [], []
    for img in images:
        t_state, n_state = torch.get_rng_state(), np.random.get_state()
        out = transform(Image.fromarray(img))
        t_after, n_after = torch.get_rng_state(), np.random.get_state()
        torch.set_rng_state(t_state)
        np.random.set_state(n_state)
        draws.append(replay_draws(duplicates, size, cutout))
        assert torch.equal(torch.get_rng_state(), t_after), 'torch draws not replayed'
        assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), n_after)), 'numpy draws not replayed'
        out = out.view(duplicates, 3, size, size)
        assert out.dtype == torch.float32
        hashes.extend(digest(c) for c in out)
    return np.asarray(draws, dtype=np.int16), hashes


def main():
    if not REF or not os.path.isdir(REF):
        sys.exit('set B200_REFERENCE to a checkout of the reference repository')
    sys.path.insert(0, REF)
    import preprocess                                                       # the reference's, unmodified
    g = torch.Generator().manual_seed(11)
    images = torch.randint(0, 256, (IMAGES, SCALE, SCALE, 3), generator=g, dtype=torch.uint8).numpy()
    arrays = {'images': images, 'padding': np.int64(PAD), 'sizes': np.array([c[0] for c in CONFIGS], dtype=np.int64)}
    for size, duplicates, cutout in CONFIGS:
        transform = preprocess.get_transform('cifar10', input_size=size, scale_size=SCALE, augment=True,
                                             duplicates=duplicates, cutout=cutout)
        draws, hashes = run(images, size, duplicates, cutout, transform)
        arrays['draws_%d' % size] = draws
        arrays['sha256_%d' % size] = np.asarray(hashes)
        arrays['cutout_%d' % size] = np.array([cutout['holes'], cutout['length']] if cutout else [0, 0], dtype=np.int64)
        print('size %d: %d copies, offsets %d..%d, flips %d' % (size, len(hashes), draws[..., :2].min(),
                                                                draws[..., :2].max(), int(draws[..., 2].sum())))
    np.savez_compressed(OUT, **arrays)
    print('wrote %s (%d bytes)' % (OUT, os.path.getsize(OUT)))


if __name__ == '__main__':
    main()
