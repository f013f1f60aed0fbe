"""Step time of batch augmentation ("Augment Your Batch", the reference README's
``--duplicates 40 --cutout -b 64`` CIFAR-10 ResNet-44 command) through Trainer.train with captured graphs.

Three data paths, alternated round by round on the same model and Trainer, so drift of the card affects all alike:
  device  -- the loader yields AugmentedBatch (64 uint8 images + draws, collated in the loading process); the relayout
             kernel writes the 2560 augmented copies;
  host    -- the torchvision transform (pad-4 crop, flip, ToTensor, Normalize, Cutout, 40 copies per sample) in
             --workers DataLoader workers on in-memory PIL images, then the 31 MB fp32 batch is copied to the device;
  bound   -- pre-augmented fp32 batches already on the device: no data cost at all.
Each round of a path is one epoch of --warmup + --steps steps; only the last --steps are timed (from a device
synchronise after the warm-up steps to one after the last step), so loader start-up and graph capture are excluded.
Round 0 of every path is warm-up.  Also times the augmenting relayout kernel against plain input_prep_u8 at the same
output size (CUDA events over --kernel-iters launches each) with the bytes each must move.  Prints one JSON line
(also written to --out) with the card's name and power limit and the host's CPU count.

    python tools/batch_augment_bench.py [--rounds 3] [--steps 30] [--warmup 5] [--workers N] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, D, SIZE, CLASSES = 64, 40, 32, 10
CUTOUT = {'holes': 1, 'length': 16}


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(', ') + ['?', '?'])[:2]
    return name, power


class PILImages(torch.utils.data.Dataset):
    def __init__(self, images, labels, transform):
        from PIL import Image
        self.images = [Image.fromarray(im) for im in images.numpy()]
        self.labels, self.transform = labels, transform

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, i):
        return self.transform(self.images[i % len(self.images)]), int(self.labels[i])


def timed_epoch(tr, loader, warmup):
    """ms/step of the steps after the first ``warmup`` of one epoch, and the mean 'data' meter (host wait)."""
    marks, step = {}, tr._step

    def marking_step(inputs, target, **kw):
        out = step(inputs, target, **kw)
        n = marks.setdefault('n', 0) + 1
        marks['n'] = n
        if n == warmup:
            torch.cuda.synchronize()
            marks['t0'] = time.perf_counter()
        return out
    tr._step = marking_step
    try:
        res = tr.train(loader)
    finally:
        tr._step = step
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - marks['t0']) / (marks['n'] - warmup), res['data']


def kernel_times(iters):
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.utils.augment import BatchAugment
    spec = BatchAugment(padding=4, cutout=CUTOUT, duplicates=D)
    g = torch.Generator().manual_seed(1)
    x = torch.randint(0, 256, (B, SIZE, SIZE, 3), generator=g, dtype=torch.uint8).cuda()
    x_full = torch.randint(0, 256, (B * D, SIZE, SIZE, 3), generator=g, dtype=torch.uint8).cuda()
    aug = ops.Aug(spec.sample(B, SIZE, SIZE).reshape(B * D, -1).cuda(), spec.lut(3).cuda(), D, 4)
    out = torch.empty((B * D, SIZE, SIZE, 16), dtype=torch.bfloat16, device='cuda')
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    runs = {'input_prep_u8_aug': (lambda: ops.input_prep_u8_aug(x, 16, aug, out=out),
                                  x.numel() + 2 * aug.params.numel() + 4 * aug.lut.numel() + 2 * out.numel()),
            'input_prep_u8': (lambda: ops.input_prep_u8(x_full, 16, mean, std, out=out), x_full.numel() + 2 * out.numel())}
    res = {}
    for name, (fn, nbytes) in runs.items():
        for _ in range(10):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        res[name] = {'ms': round(ms, 4), 'bytes': nbytes, 'GB_per_s': round(nbytes / ms / 1e6, 1)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--workers', type=int, default=os.cpu_count())
    ap.add_argument('--kernel-iters', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('batch_augment_bench needs a CUDA device')
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import U8Images, real_dataset_transform
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.augment import AugmentCollate, BatchAugment
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    torch.cuda.set_device(0)
    torch.manual_seed(123)
    np.random.seed(0)
    model = convert_b200(models.resnet(dataset='cifar10', depth=44), 'cuda')
    tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device='cuda', print_freq=10 ** 9)

    steps = args.warmup + args.steps
    g = torch.Generator().manual_seed(0)
    pool = torch.randint(0, 256, (1024, SIZE, SIZE, 3), generator=g, dtype=torch.uint8)
    labels = torch.randint(0, CLASSES, (steps * B,), generator=g)
    spec = BatchAugment(padding=4, cutout=CUTOUT, duplicates=D)
    device_loader = torch.utils.data.DataLoader(U8Images(pool, labels), batch_size=B, shuffle=True, drop_last=True,
                                                num_workers=0, pin_memory=True, collate_fn=AugmentCollate(spec))
    tf = real_dataset_transform('cifar10', augment=True, cutout=CUTOUT, duplicates=D)
    host_loader = torch.utils.data.DataLoader(PILImages(pool, labels, tf), batch_size=B, shuffle=True, drop_last=True,
                                              num_workers=args.workers, pin_memory=True,
                                              persistent_workers=args.workers > 0)
    bound = []
    for k in range(2):
        xb, yb = next(iter(device_loader))
        bound.append((xb.apply().cuda(), yb.cuda()))
    bound_loader = [bound[i % 2] for i in range(steps)]
    # 'bound' captures the fp32 step graph that 'host' replays: a capture must not overlap the pin-memory thread of a
    # worker loader (pinning is not permitted while another thread captures in global mode), so 'host' runs last
    paths = (('bound', bound_loader), ('device', device_loader), ('host', host_loader))

    times = {k: [] for k, _ in paths}
    data_wait = {k: [] for k, _ in paths}
    for r in range(args.rounds + 1):
        for name, loader in paths:
            ms, data = timed_epoch(tr, loader, args.warmup)
            if r > 0:
                times[name].append(ms)
                data_wait[name].append(1e3 * data)
    kern = kernel_times(args.kernel_iters)
    gpu, power = card()
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {'model': 'resnet44', 'batch': B, 'duplicates': D, 'cutout': CUTOUT, 'size': SIZE,
           'steps_per_round': args.steps, 'rounds': args.rounds, 'workers': args.workers,
           'ms_per_step': {k: round(v, 3) for k, v in med.items()},
           'img_per_s': {k: round(B * D / (v / 1e3), 1) for k, v in med.items()},
           'ms_per_step_all': {k: [round(t, 3) for t in v] for k, v in times.items()},
           'data_wait_ms_mean': {k: round(statistics.mean(v), 3) for k, v in data_wait.items()},
           'kernels': kern, 'graph_replays': tr.graph_replays, 'gpu': gpu, 'power_limit': power,
           'host_cpus': os.cpu_count()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
