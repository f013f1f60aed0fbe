"""Evaluation throughput with Resize + CenterCrop on the device: ResNet-50 eval (BatchNorm folded), batch 256, 224 px
from scale 256, through Trainer.validate, on a temporary ImageFolder of seeded synthetic JPEGs of ImageNet-like sizes
(about 500x375, varied; written before any timing).

Four data paths, alternated round by round on the same model and Trainer, so drift of the card affects all alike:
  decode  -- --device-scale-crop --device-decode: the workers read the files and parse headers only; the loader yields
             JpegBatch and csrc/jpeg.cu decodes the support regions on the copy stream ahead of the relayout;
  device  -- --device-scale-crop: --workers DataLoader workers decode and cut each image's support region only; the
             loader yields ScaleCropBatch and the relayout kernel resizes, centre-crops and normalises;
  host    -- the host transform (real_dataset_transform('imagenet', augment=False): Resize, CenterCrop, ToTensor,
             Normalize in the same number of workers), then the fp32 batch is copied to the device;
  bound   -- pre-staged fp32 batches already on the device: no data cost at all.
Each round of a path runs --warmup + --steps steps from one persistent loader iterator; only the last --steps are
timed (device synchronise to device synchronise).  Round 0 of every path is warm-up.  Also reports the host-to-device
bytes per batch of each path and the relayout kernel's time from a torch.profiler trace of --kernel-iters launches on a
loader batch, with the bytes it moves, the decode kernels' times (torch.profiler, a run of its own) and the host CPU
time per image of the workers' work with and without the device decode.  Prints one JSON line (also written to --out) with the card's name and power
limit and the host's CPU count.

    python tools/scale_crop_bench.py [--rounds 3] [--steps 20] [--warmup 4] [--workers 16] [--out FILE]
"""
import argparse
import itertools
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, SIZE, SCALE, CLASSES, IMAGES = 256, 224, 256, 16, 1024


def card():
    q = subprocess.run(['nvidia-smi', '-i', str(torch.cuda.current_device()), '--query-gpu=name,power.limit',
                        '--format=csv,noheader'], capture_output=True, text=True)
    name, power = (q.stdout.strip().split(', ') + ['?', '?'])[:2]
    return name, power


def write_jpegs(root):
    """IMAGES seeded JPEGs (smooth random fields + noise, sides around 500x375) in CLASSES folders."""
    from PIL import Image
    rng = np.random.default_rng(0)
    for i in range(IMAGES):
        w, h = int(rng.integers(400, 640)), int(rng.integers(300, 480))
        if rng.random() < 0.3:
            w, h = h, w
        base = rng.integers(0, 256, (h // 16 + 1, w // 16 + 1, 3), dtype=np.uint8)
        img = Image.fromarray(base).resize((w, h), Image.BILINEAR)
        a = np.clip(np.asarray(img).astype(np.int16) + rng.integers(-20, 21, (h, w, 3)), 0, 255).astype(np.uint8)
        d = os.path.join(root, 'val', 'c%02d' % (i % CLASSES))
        os.makedirs(d, exist_ok=True)
        Image.fromarray(a).save(os.path.join(d, '%05d.jpg' % i), quality=90)


def timed(tr, it, warmup, steps):
    """ms/batch of ``steps`` batches after ``warmup`` batches from the iterator ``it``, and the mean 'data' meter."""
    tr.validate(itertools.islice(it, warmup))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = tr.validate(itertools.islice(it, steps))
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps, res['data']


def kernel_time(batch, iters):
    """mean device time of input_prep_scale_crop_kernel in a profiler trace of ``iters`` launches on ``batch``"""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200 import ops
    regions = batch.regions.cuda()
    sc = ops.ScaleCropTables(batch.index.cuda(), batch.geom.cuda(), batch.spec.lut(3).cuda(), batch.spec.size,
                             (batch.index, batch.geom, batch.nbytes))
    out = torch.empty((B, SIZE // 2 + 3, SIZE // 2 + 3, 16), dtype=torch.bfloat16, device='cuda')
    for _ in range(10):
        ops.input_prep_u8_scale_crop(regions, 16, sc, s2d=True, border=True, out=out)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            ops.input_prep_u8_scale_crop(regions, 16, sc, s2d=True, border=True, out=out)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and 'input_prep_scale_crop_kernel' in e.name]
    ms = 1e-3 * statistics.mean(times)
    nbytes = batch.nbytes + 2 * out.numel() + 8 * batch.index.numel() + 4 * batch.geom.numel()
    return {'ms': round(ms, 4), 'launches_traced': len(times), 'bytes': nbytes, 'region_bytes': batch.nbytes,
            'out_bytes': 2 * out.numel(), 'GB_per_s': round(nbytes / ms / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=4)
    ap.add_argument('--workers', type=int, default=16)
    ap.add_argument('--kernel-iters', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('scale_crop_bench needs a CUDA device')
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import DataRegime
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.cuda.set_device(0)
    torch.manual_seed(123)
    tmp = tempfile.mkdtemp(prefix='scale_crop_bench_')
    t0 = time.perf_counter()
    write_jpegs(os.path.join(tmp, 'imagenet'))
    setup_s = time.perf_counter() - t0
    model = convert_b200(models.resnet(dataset='imagenet', depth=50), 'cuda')
    tr = Trainer(model, CrossEntropyLoss().cuda(), device='cuda', print_freq=10 ** 9)

    sampler = torch.utils.data.RandomSampler(range(IMAGES), replacement=True, num_samples=10 ** 7)
    base = {'name': 'imagenet', 'datasets_path': tmp, 'split': 'val', 'augment': False, 'input_size': SIZE,
            'scale_size': SCALE, 'batch_size': B, 'sampler': sampler, 'num_workers': args.workers,
            'drop_last': True, 'pin_memory': False}
    device_it = iter(DataRegime(None, defaults=dict(base, device_scale_crop=True)).get_loader())
    host_it = iter(DataRegime(None, defaults=base).get_loader())
    decode_it = iter(DataRegime(None, defaults=dict(base, device_scale_crop=True, device_decode=True)).get_loader())
    jpeg_batch, _ = next(decode_it)
    sample, _ = next(device_it)
    bound = [(sample.apply().cuda(), torch.randint(0, CLASSES, (B,)).cuda()) for _ in range(2)]
    bound_it = itertools.cycle(bound)
    paths = (('bound', bound_it), ('decode', decode_it), ('device', device_it), ('host', host_it))
    times = {k: [] for k, _ in paths}
    data_wait = {k: [] for k, _ in paths}
    for r in range(args.rounds + 1):
        for name, it in paths:
            ms, data = timed(tr, it, args.warmup, args.steps)
            if r > 0:
                times[name].append(ms)
                data_wait[name].append(1e3 * data)
    kern = kernel_time(sample, args.kernel_iters)
    from resized_crop_bench import decode_kernels, worker_cpu_ms
    dec = decode_kernels(jpeg_batch)
    cpu = worker_cpu_ms(os.path.join(tmp, 'imagenet'), sample.spec)
    gpu, power = card()
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {'model': 'resnet50-eval-folded', 'batch': B, 'size': SIZE, 'scale': SCALE, 'images': IMAGES,
           'jpeg_setup_s': round(setup_s, 1), 'steps_per_round': args.steps, 'rounds': args.rounds,
           'workers': args.workers,
           'ms_per_batch': {k: round(v, 3) for k, v in med.items()},
           'ms_per_batch_range': {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
           'img_per_s': {k: round(B / (v / 1e3), 1) for k, v in med.items()},
           'img_per_s_range': {k: [round(B / (max(v) / 1e3), 1), round(B / (min(v) / 1e3), 1)]
                               for k, v in times.items()},
           'data_wait_ms_mean': {k: round(statistics.mean(v), 3) for k, v in data_wait.items()},
           'h2d_bytes_per_batch': {'device': sample.nbytes + 8 * sample.index.numel() + 4 * sample.geom.numel() + 8 * B,
                                   'host': 4 * B * 3 * SIZE * SIZE + 8 * B, 'bound': 0,
                                   'decode': jpeg_batch.payload.numel() + 8 * jpeg_batch.index.numel()
                                   + 4 * jpeg_batch.table.numel() + 8 * B},
           'decode_kernels_ms': dec, 'worker_cpu_ms_per_image': cpu,
           'relayout_kernel': kern, 'relayout_share_of_device_batch': round(kern['ms'] / med['device'], 5),
           'gpu': gpu, 'power_limit': power, 'host_cpus': os.cpu_count()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
