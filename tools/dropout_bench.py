"""Step time of in-block dropout (resnet(dropout=p), csrc/dropout.cu) against the same network without dropout.

WRN-28-10 (depth 28, width [160, 320, 640]) at batch 128 and ResNet-44 at batch 64, 32 px CIFAR shapes, synthetic fp32
NCHW batches, captured Trainer steps.  Per network one process holds a p = 0.3 and a p = 0 model (same seed) with their
own Trainers; the two alternate round by round so drift of the card affects both alike.  Round 0 of each is warm-up
(eager steps and graph capture); the median ms/step of the remaining rounds is reported.

A second pass (no graphs, profiler on, after the timed rounds) runs one train_step of each model and reports per kernel
class the device time and the bandwidth computed from shapes (ops._T classes: bytes each call must move), and per BN
kernel the profiler's device time: the dropout apply and backward of the p = 0.3 model beside bn_apply / bn_bwd_* of
the same units in the p = 0 model.  Prints one JSON line with the card's name and power limit.

    python tools/dropout_bench.py [--rounds 3] [--steps 20] [--p 0.3] [--models wrn28_10,resnet44]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from l1_norm_bench import card, kernel_breakdown  # noqa: E402  (tools/ is on sys.path when run as a script)

NETS = {'wrn28_10': (dict(depth=28, width=[160, 320, 640], regime='wide-resnet'), 128),
        'resnet44': (dict(depth=44), 64)}


def build(cfg, p):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.manual_seed(123)
    model = convert_b200(models.resnet(dataset='cifar10', dropout=p, **cfg), 'cuda')
    return Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device='cuda', print_freq=10 ** 9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--p', type=float, default=0.3)
    ap.add_argument('--models', default='wrn28_10,resnet44')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('dropout_bench needs a CUDA device')
    out = {'p': args.p, 'rounds': args.rounds, 'steps_per_round': args.steps}
    for net in args.models.split(','):
        cfg, batch = NETS[net]
        g = torch.Generator().manual_seed(0)
        pool = [(torch.randn(batch, 3, 32, 32, generator=g).pin_memory(), torch.randint(0, 10, (batch,), generator=g))
                for _ in range(2)]
        loader = [pool[i % 2] for i in range(args.steps)]
        trainers = {'p0': build(cfg, 0.0), 'dropout': build(cfg, args.p)}
        times = {k: [] for k in trainers}
        for r in range(args.rounds + 1):
            for kind, tr in trainers.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.train(loader)
                torch.cuda.synchronize()
                if r > 0:
                    times[kind].append(1e3 * (time.perf_counter() - t0) / len(loader))
        med = {k: statistics.median(v) for k, v in times.items()}
        res = {'batch': batch, 'ms_per_step': {k: round(v, 3) for k, v in med.items()},
               'ms_per_step_all': {k: [round(t, 3) for t in v] for k, v in times.items()},
               'img_per_s': {k: round(batch * 1e3 / v, 1) for k, v in med.items()},
               'dropout_overhead_pct': round(100.0 * (med['dropout'] / med['p0'] - 1.0), 2),
               'graph_replays': {k: tr.graph_replays for k, tr in trainers.items()}}
        x, y = pool[0][0].cuda(), pool[0][1].cuda()
        for kind, tr in trainers.items():
            tr.use_graphs = False
            res['classes_' + kind], res['kernels_' + kind] = kernel_breakdown(tr, x, y)
        out[net] = res
        del trainers, pool, loader
        torch.cuda.empty_cache()
    out['gpu'], out['power_limit'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
