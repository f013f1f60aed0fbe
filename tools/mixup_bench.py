"""Step time of Trainer.train with no input mixing, MixUp and CutMix on the fused kernel path.

ResNet-50, batch 256, 224 px, synthetic fp32 NCHW batches, one process: the three settings alternate round by round on
the same model and Trainer (each setting has its own captured graph), so drift of the card affects all three alike.
The first round of each setting is warm-up (eager steps and capture).  Prints one JSON line with the median ms/step
of each setting, the overheads and the card's name and power limit.

    python tools/mixup_bench.py [--rounds 4] [--steps 20] [--batch 256] [--size 224]
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SETTINGS = (('none', dict(mixup=None, cutmix=None)), ('mixup', dict(mixup=0.2, cutmix=None)),
            ('cutmix', dict(mixup=None, cutmix=1.0)))


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(', ') + ['?', '?'])[:2]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--size', type=int, default=224)
    args = ap.parse_args()
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    if not torch.cuda.is_available():
        raise SystemExit('mixup_bench needs a CUDA device')
    torch.manual_seed(123)
    random.seed(0)
    np.random.seed(0)
    model = convert_b200(models.resnet(dataset='imagenet', depth=50), 'cuda')
    opt = OptimRegime(model, model.regime)
    tr = Trainer(model, CrossEntropyLoss(), opt, device='cuda', print_freq=10 ** 9)
    g = torch.Generator().manual_seed(0)
    pool = [(torch.randn(args.batch, 3, args.size, args.size, generator=g).pin_memory(),
             torch.randint(0, 1000, (args.batch,), generator=g)) for _ in range(2)]
    loader = [pool[i % 2] for i in range(args.steps)]
    times = {k: [] for k, _ in SETTINGS}
    for r in range(args.rounds + 1):
        for name, flags in SETTINGS:
            tr.mixup, tr.cutmix = flags['mixup'], flags['cutmix']
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tr.train(loader)
            torch.cuda.synchronize()
            ms = 1e3 * (time.perf_counter() - t0) / len(loader)
            if r > 0:                  # round 0: warm-up and graph capture of every setting
                times[name].append(ms)
    name, power = card()
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({'model': 'resnet50', 'batch': args.batch, 'size': args.size, 'steps_per_round': len(loader),
                      'rounds': args.rounds, 'ms_per_step': {k: round(v, 3) for k, v in med.items()},
                      'ms_per_step_all': {k: [round(t, 3) for t in v] for k, v in times.items()},
                      'overhead_pct': {k: round(100.0 * (med[k] / med['none'] - 1.0), 2) for k in ('mixup', 'cutmix')},
                      'graph_replays': tr.graph_replays, 'gpu': name, 'power_limit': power}))


if __name__ == '__main__':
    main()
