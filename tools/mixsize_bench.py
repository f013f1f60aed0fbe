"""Step time of the Mix&Match CIFAR size regimes (the reference README's ``--model-config "{'regime': 'sampled_D+'}"``
ResNet-44 command, and ``sampled_B+``) through Trainer.train with captured graphs, size by size.

The two regimes train at 32 / 48 / 24 / 16 px with (batch, duplicates) = (64, 1) / (28, 1) / (64, 2) / (64, 4) for D+
and (64, 1) / (28, 1) / (114, 1) / (256, 1) for B+: six distinct (size, batch, duplicates) configurations.  For each,
three data paths, alternated round by round on the same model and Trainer, so drift of the card affects all alike:
  device  -- the loader yields AugmentedBatch (the uint8 32-px images + draws, collated in the loading process); the
             relayout kernel crops, resizes, flips and normalises the copies;
  host    -- the torchvision transform (pad-4 crop, Resize, flip, ToTensor, Normalize, per copy) in --workers
             DataLoader workers on in-memory PIL images, then the fp32 batch is copied to the device;
  bound   -- pre-augmented fp32 batches already on the device: no data cost at all.
Each round of a path and configuration is one epoch of --warmup + --steps steps; only the last --steps are timed (from
a device synchronise after the warm-up steps to one after the last step), so loader start-up and graph capture are
excluded.  Round 0 is warm-up.  The relayout kernel's own time per configuration comes from a torch.profiler trace of
--kernel-iters launches, in a pass of its own after the timed rounds.  Prints one JSON line (also written to --out)
with the card's name and power limit and the host's CPU count.

    python tools/mixsize_bench.py [--rounds 3] [--steps 150] [--warmup 5] [--workers 16] [--out FILE]
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

SCALE, CLASSES = 32, 10


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
    """ms/step of the steps after the first ``warmup`` of one epoch."""
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
        tr.train(loader)
    finally:
        tr._step = step
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - marks['t0']) / (marks['n'] - warmup)


def kernel_us(spec, batch, iters):
    """Mean device time (us) of the relayout kernel that makes one step's copies, from a profiler trace."""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200 import ops
    g = torch.Generator().manual_seed(1)
    x = torch.randint(0, 256, (batch, SCALE, SCALE, 3), generator=g, dtype=torch.uint8).cuda()
    aug = ops.Aug(spec.sample(batch, SCALE, SCALE).reshape(batch * spec.duplicates, -1).cuda(), spec.lut(3).cuda(),
                  spec.duplicates, spec.padding, spec.resize)
    OH, OW = spec.resize or (SCALE, SCALE)
    out = torch.empty((batch * spec.duplicates, OH, OW, 16), dtype=torch.bfloat16, device='cuda')
    for _ in range(10):
        ops.input_prep_u8_aug(x, 16, aug, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            ops.input_prep_u8_aug(x, 16, aug, out=out)
        torch.cuda.synchronize()
    want = 'input_prep_aug_resize_kernel' if spec.resize else 'input_prep_u8_kernel'
    times = [e.device_time for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and want in e.name]
    assert len(times) == iters, (want, len(times))
    return want, statistics.mean(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=150)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--workers', type=int, default=min(16, os.cpu_count()))
    ap.add_argument('--kernel-iters', type=int, default=200)
    ap.add_argument('--depth', type=int, default=44)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('mixsize_bench needs a CUDA device')
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import U8Images, device_augment_spec, real_dataset_transform
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.augment import AugmentCollate
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    torch.cuda.set_device(0)
    torch.manual_seed(123)
    np.random.seed(0)
    # the (size, batch, duplicates) configurations of the two regimes, as the model states them
    configs = {}
    for regime in ('sampled_D+', 'sampled_B+'):
        for _, c in models.resnet(dataset='cifar10', depth=8, regime=regime).sampled_data_regime:
            configs.setdefault((c['input_size'], c['batch_size'], c['duplicates']), []).append(regime)
    model = convert_b200(models.resnet(dataset='cifar10', depth=args.depth, regime='sampled_D+'), 'cuda')
    tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device='cuda', print_freq=10 ** 9)

    steps = args.warmup + args.steps
    g = torch.Generator().manual_seed(0)
    pool = torch.randint(0, 256, (1024, SCALE, SCALE, 3), generator=g, dtype=torch.uint8)
    loaders, specs = {}, {}
    for size, batch, dup in configs:
        labels = torch.randint(0, CLASSES, (steps * batch,), generator=g)
        spec = specs[size, batch, dup] = device_augment_spec('cifar10', input_size=size, scale_size=SCALE,
                                                             duplicates=dup)
        device = torch.utils.data.DataLoader(U8Images(pool, labels), batch_size=batch, shuffle=True, drop_last=True,
                                             num_workers=0, collate_fn=AugmentCollate(spec))
        tf = real_dataset_transform('cifar10', input_size=size, scale_size=SCALE, augment=True, duplicates=dup)
        host = torch.utils.data.DataLoader(PILImages(pool, labels, tf), batch_size=batch, shuffle=True,
                                           drop_last=True, num_workers=args.workers, pin_memory=True)
        bound = []
        for _ in range(2):
            xb, yb = next(iter(device))
            bound.append((xb.apply().cuda(), yb.cuda()))
        loaders[size, batch, dup] = {'bound': [bound[i % 2] for i in range(steps)], 'device': device, 'host': host}

    # 'bound' captures the fp32 step graph that 'host' replays and 'device' its own: a capture must not overlap the
    # pin-memory thread of a worker loader (pinning is not permitted while another thread captures in global mode), so
    # within a round every configuration's 'bound' and 'device' epochs run before the first 'host' epoch
    paths = ('bound', 'device', 'host')
    times = {cfg: {p: [] for p in paths} for cfg in configs}
    for r in range(args.rounds + 1):
        for path in paths:
            for cfg in configs:
                ms = timed_epoch(tr, loaders[cfg][path], args.warmup)
                if r > 0:
                    times[cfg][path].append(ms)
    rows = []
    for cfg, regimes in configs.items():
        size, batch, dup = cfg
        name, us = kernel_us(specs[cfg], batch, args.kernel_iters)
        med = {p: statistics.median(v) for p, v in times[cfg].items()}
        rows.append({'size': size, 'batch': batch, 'duplicates': dup, 'rows': batch * dup, 'regimes': regimes,
                     'ms_per_step': {p: round(v, 3) for p, v in med.items()},
                     'ms_per_step_range': {p: [round(min(v), 3), round(max(v), 3)] for p, v in times[cfg].items()},
                     'rows_per_s': {p: round(batch * dup / (v / 1e3), 1) for p, v in med.items()},
                     'kernel': name, 'kernel_us': round(us, 2),
                     'kernel_share_of_device_step': round(us / (1e3 * med['device']), 4)})
    gpu, power = card()
    res = {'model': 'resnet%d' % args.depth, 'steps_per_round': args.steps, 'rounds': args.rounds,
           'workers': args.workers, 'configs': rows, 'graph_replays': tr.graph_replays, 'gpu': gpu,
           'power_limit': power, 'host_cpus': os.cpu_count()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
