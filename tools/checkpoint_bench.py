"""Cost and memory of activation checkpointing (``checkpoint_segments``) on the kernel path.

1. ResNet-50, batch 256, 224 px, synthetic fp32 NCHW batches: one process holds the models for s = 0 (no
   checkpointing), 1, 2 and 4 (same seed) and alternates them round by round, so drift of the card affects all alike.
   Per model: ms of one eager ``train_step`` (forward, loss, backward; CUDA events; median and range of the steps of
   rounds 1..), and the peak ``torch.cuda.max_memory_allocated`` of one eager step above what the model holds between
   steps.  ``s=2/nojoin`` is s = 2 with the weight-gradient stream joined only at the end of the backward pass instead
   of at every segment boundary (the recomputed tensors then stay alive until the end): the difference is what the
   joins cost in time and save in memory.
2. ResNet-152 and -200 at 224 px, s in {0, 1, 2, 4}: the eager-step peak at batch 128 and 256, and the largest batch
   the card's free memory holds by linear extrapolation of those two peaks (less 2 GiB for allocator rounding),
   confirmed by one step at that batch (10% less after an allocation failure, at most three tries; null if none
   fits).

Prints one JSON line with the card's name and power limit, read in the same process.

    python tools/checkpoint_bench.py [--rounds 4] [--steps 10] [--skip-fit]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(', ') + ['?', '?'])[:2]
    return name, power


def build(depth, s):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    torch.manual_seed(123)
    return convert_b200(models.resnet(dataset='imagenet', depth=depth, checkpoint_segments=s), 'cuda')._b200


def join_only_at_end(rt):
    """the runtime's backward pass without the joins at segment boundaries (measurement only)"""
    real_join, real_stem, real_bwd = rt._wgrad_join, rt._stem_bwd, rt.run_backward
    on = [False]

    def join():
        if on[0]:
            real_join()

    def stem(st, d):
        on[0] = True
        real_stem(st, d)

    def bwd(*a, **k):
        on[0] = False
        real_bwd(*a, **k)
    rt._wgrad_join, rt._stem_bwd, rt.run_backward = join, stem, bwd
    return rt


def batch(n, px):
    g = torch.Generator(device='cuda').manual_seed(n)
    return (torch.randn(n, 3, px, px, device='cuda', generator=g),
            torch.randint(0, 1000, (n,), device='cuda', generator=g))


def peak(rt, x, y):
    """extra device memory of one eager train_step above what is allocated before it"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    rt.train_step(x, y)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def step_times(rts, x, y, rounds, steps):
    times = {k: [] for k in rts}
    for r in range(rounds):
        for k, rt in rts.items():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
            ev[0].record()
            for i in range(steps):
                rt.train_step(x, y)
                ev[i + 1].record()
            torch.cuda.synchronize()
            if r:                                   # round 0: warm-up
                times[k] += [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]
    return {k: {'median_ms': round(statistics.median(v), 2), 'min_ms': round(min(v), 2), 'max_ms': round(max(v), 2)}
            for k, v in times.items()}


def largest_batch(depth, s, px=224, b0=128, b1=256, margin=2 << 30):
    rt = build(depth, s)
    p = {}
    for b in (b0, b1):
        x, y = batch(b, px)
        rt.train_step(x, y)
        p[b] = peak(rt, x, y)
        del x, y
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    per = (p[b1] - p[b0]) / (b1 - b0)
    fixed = p[b0] - b0 * per
    pred = int((free - margin - fixed) // per)
    fits = None
    for _ in range(3):          # the allocator refuses before anything is launched: step down 10% and try again
        try:
            x, y = batch(pred, px)
            rt.train_step(x, y)
            torch.cuda.synchronize()
            fits = pred
            break
        except torch.cuda.OutOfMemoryError:
            x = y = None
            torch.cuda.empty_cache()
            pred = int(pred * 0.9)
    del rt
    x = y = None
    torch.cuda.empty_cache()
    return {'peak_b%d_GiB' % b0: round(p[b0] / 2 ** 30, 2), 'peak_b%d_GiB' % b1: round(p[b1] / 2 ** 30, 2),
            'MiB_per_image': round(per / 2 ** 20, 1), 'largest_batch_confirmed': fits}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--skip-fit', action='store_true')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, power = card()
    out = {'card': name, 'power_limit': power, 'resnet50_b256_224': {}}
    rts = {'s=%d' % s: build(50, s) for s in (0, 1, 2, 4)}
    rts['s=2/nojoin'] = join_only_at_end(build(50, 2))
    x, y = batch(256, 224)
    times = step_times(rts, x, y, args.rounds, args.steps)
    for k, rt in rts.items():
        out['resnet50_b256_224'][k] = dict(times[k], peak_GiB=round(peak(rt, x, y) / 2 ** 30, 2))
    del rts, x, y
    torch.cuda.empty_cache()
    if not args.skip_fit:
        for depth in (152, 200):
            out['resnet%d_224' % depth] = {'s=%d' % s: largest_batch(depth, s) for s in (0, 1, 2, 4)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
