"""Step time and memory of gradient accumulation (``chunk_batch``) on the kernel path.

1. ResNet-50, 224 px, effective batch 256 of synthetic fp32 NCHW host batches through ``Trainer.train`` (prefetch,
   captured CUDA graphs, fused SGD): chunk_batch N = 1, 2 and 4 on the fused path, and N = 2 on the generic autograd
   path (the criterion under another type, which the fused path does not take: what chunked steps ran before the
   fused path supported them).  One process holds the four trainers and alternates them round by round, so drift of
   the card affects all alike; round 0 (eager warm-up and graph capture) is not timed.  Per configuration: ms/step of
   ``Trainer.train`` over each round's steps (host clock around work that ends in a device synchronise; median and
   range over the rounds), and the peak ``torch.cuda.max_memory_allocated`` of round 0 above what was allocated before
   it (activations, workspaces and the captured graphs' pool).
2. ResNet-152 with checkpoint_segments = 2 at 224 px, effective batch 1024 (above the 933 that fits one step) as
   N = 2 chunks of 512: ms/step and peak the same way.

Prints one JSON line with the card's name and power limit, read in the same process.

    python tools/chunk_batch_bench.py [--rounds 3] [--steps 8] [--skip-152]
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(', ') + ['?', '?'])[:2]
    return name, power


def trainer(depth, segments=0, generic=False):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime

    class Unfused(CrossEntropyLoss):
        """the plain criterion under another type: Trainer keeps the generic autograd path for it"""

    torch.manual_seed(123)
    model = convert_b200(models.resnet(dataset='imagenet', depth=depth, checkpoint_segments=segments), 'cuda')
    crit = Unfused() if generic else CrossEntropyLoss()
    return Trainer(model, crit, OptimRegime(model, copy.deepcopy(model.regime)), device='cuda', print_freq=10 ** 9)


def batches(n, B, px):
    g = torch.Generator().manual_seed(B)
    return [(torch.randn(B, 3, px, px, generator=g).pin_memory(), torch.randint(0, 1000, (B,), generator=g))
            for _ in range(n)]


def run_round(tr, data, N, steps):
    loader = [data[i % len(data)] for i in range(steps)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tr.train(loader, chunk_batch=N)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def measure(configs, data, rounds, steps):
    """configs: name -> (trainer, N).  -> name -> {median_ms, min_ms, max_ms, peak_GiB, graph_replays}"""
    times = {k: [] for k in configs}
    peaks = {}
    for r in range(rounds + 1):
        for k, (tr, N) in configs.items():
            if r == 0:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                run_round(tr, data, N, steps)
                peaks[k] = torch.cuda.max_memory_allocated() - base
            else:
                times[k].append(run_round(tr, data, N, steps))
    return {k: {'median_ms': round(statistics.median(v), 2), 'min_ms': round(min(v), 2), 'max_ms': round(max(v), 2),
                'peak_GiB': round(peaks[k] / 2 ** 30, 2), 'graph_replays': configs[k][0].graph_replays}
            for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--skip-152', action='store_true')
    args = ap.parse_args()
    torch.cuda.set_device(0)
    name, power = card()
    out = {'card': name, 'power_limit': power}
    data = batches(3, 256, 224)
    configs = {'N=1': (trainer(50), 1), 'N=2': (trainer(50), 2), 'N=4': (trainer(50), 4),
               'N=2/generic': (trainer(50, generic=True), 2)}
    out['resnet50_b256_224'] = measure(configs, data, args.rounds, args.steps)
    del configs, data
    torch.cuda.empty_cache()
    if not args.skip_152:
        data = batches(2, 1024, 224)
        out['resnet152_s2_b1024_224'] = measure({'N=2': (trainer(152, segments=2), 2)}, data, 1, 3)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
