"""Step time of L1 batch normalization (bn_norm='L1') against the variance BatchNorm on the fused kernel path.

ResNet-18 at batch 128 and ResNet-50 at batch 256, 224 px, synthetic fp32 NCHW batches, captured Trainer steps.  Per
network one process holds a BN and an L1 model (same seed) with their own Trainers; the two alternate round by round so
drift of the card affects both alike.  Round 0 of each is warm-up (eager steps and graph capture); the median ms/step of
the remaining rounds is reported.  L1 BN reads every BN input twice more than the BN whose statistics come from the
convolution epilogue, and its statistics take four launches instead of one: the overhead is what that costs.

A second pass (no graphs, profiler on, after the timed rounds) runs one train_step of each model and reports per kernel
class the device time and the bandwidth computed from shapes (ops._T classes: bytes each call must move), and per BN
kernel the profiler's device time.  Prints one JSON line with the card's name and power limit.

    python tools/l1_norm_bench.py [--rounds 3] [--steps 20] [--size 224] [--models resnet18,resnet50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NETS = {'resnet18': (18, 128), 'resnet50': (50, 256)}


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(', ') + ['?', '?'])[:2]
    return name, power


def build(depth, bn_norm):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.manual_seed(123)
    cfg = dict(dataset='imagenet', depth=depth)
    if bn_norm:
        cfg['bn_norm'] = bn_norm
    model = convert_b200(models.resnet(**cfg), 'cuda')
    return Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device='cuda', print_freq=10 ** 9)


def kernel_breakdown(tr, x, y):
    """one eager train_step: {class: ms, GB/s} from the ops timing classes, {kernel: ms} of BN kernels"""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200 import ops
    rt = tr.b200
    rt.train_step(x, y)
    torch.cuda.synchronize()
    ops.start_timing()
    rt.train_step(x, y)
    classes = ops.stop_timing()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rt.train_step(x, y)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and 'bn_' in e.key:
            name = e.key.split('(')[0].replace('void ', '').replace('b200::', '')
            kern[name] = {'ms': round(e.device_time_total / 1e3, 3), 'calls': e.count}
    cls = {k: {'ms': round(v['ms'], 3), 'calls': v['calls'],
               'GB_per_s': round(v['bytes'] / (v['ms'] * 1e6), 1) if v['bytes'] and v['ms'] > 0 else None}
           for k, v in classes.items() if k.startswith('bn_')}
    return cls, kern


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--size', type=int, default=224)
    ap.add_argument('--models', default='resnet18,resnet50')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('l1_norm_bench needs a CUDA device')
    out = {'size': args.size, 'rounds': args.rounds, 'steps_per_round': args.steps}
    for net in args.models.split(','):
        depth, batch = NETS[net]
        g = torch.Generator().manual_seed(0)
        pool = [(torch.randn(batch, 3, args.size, args.size, generator=g).pin_memory(),
                 torch.randint(0, 1000, (batch,), generator=g)) for _ in range(2)]
        loader = [pool[i % 2] for i in range(args.steps)]
        trainers = {'bn': build(depth, None), 'l1': build(depth, 'L1')}
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
               'l1_overhead_pct': round(100.0 * (med['l1'] / med['bn'] - 1.0), 2),
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
