"""Step time of ImageNet training with RandomResizedCrop on the device: ResNet-50, batch 256, 224 px, through
Trainer.train with captured graphs, on a temporary ImageFolder of seeded synthetic JPEGs of ImageNet-like sizes
(about 500x375, varied; written before any timing).

Four data paths, alternated round by round on the same model and Trainer, so drift of the card affects all alike:
  decode  -- --device-resized-crop --device-decode: the workers read the files, parse headers and draw; the loader
             yields JpegBatch and csrc/jpeg.cu decodes the crops' regions on the copy stream ahead of the relayout;
  device  -- --device-resized-crop: --workers DataLoader workers decode and draw only; the loader yields
             ResizedCropBatch (the crops' regions + draws) and the relayout kernel resamples, flips and normalises;
  host    -- today's host transform (real_dataset_transform('imagenet'): RandomResizedCrop, flip, ToTensor,
             Normalize in the same number of workers), then the fp32 batch is copied to the device;
  bound   -- pre-staged fp32 batches already on the device: no data cost at all.
Each round of a path runs --warmup + --steps steps from one persistent loader iterator; only the last --steps are
timed (device synchronise to device synchronise).  Round 0 of every path is warm-up.  Also reports the relayout
kernel's time and bytes/s (CUDA events over --kernel-iters launches on a loader batch), the host-to-device bytes per
step of each path, and the cost of the region copy from pageable memory against staging it through a pinned buffer,
the decode kernels' times (torch.profiler over a loader batch, a run of its own after the timed rounds) and the host
CPU time per image of the workers' per-image work and collate, with and without the device decode.
Prints one JSON line (also written to --out) with the card's name and power limit and the host's CPU count.

    python tools/resized_crop_bench.py [--rounds 3] [--steps 20] [--warmup 4] [--workers N] [--out FILE]
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

B, SIZE, CLASSES, IMAGES = 256, 224, 16, 1024


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
        d = os.path.join(root, 'train', 'c%02d' % (i % CLASSES))
        os.makedirs(d, exist_ok=True)
        Image.fromarray(a).save(os.path.join(d, '%05d.jpg' % i), quality=90)


def timed(tr, it, warmup, steps):
    """ms/step of ``steps`` steps after ``warmup`` steps from the iterator ``it``, and the mean 'data' meter."""
    tr.train(itertools.islice(it, warmup))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = tr.train(itertools.islice(it, steps))
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps, res['data']


def kernel_time(batch, iters):
    from convnet.pytorch_b200 import ops
    regions = batch.regions.cuda()
    rrc = ops.Rrc(batch.index.cuda(), batch.draws.cuda(), batch.spec.lut(3).cuda(), 1, batch.spec.size,
                  (batch.index, batch.draws, batch.nbytes))
    out = torch.empty((B, SIZE // 2 + 3, SIZE // 2 + 3, 16), dtype=torch.bfloat16, device='cuda')
    for _ in range(10):
        ops.input_prep_u8_rrc(regions, 16, rrc, s2d=True, border=True, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.input_prep_u8_rrc(regions, 16, rrc, s2d=True, border=True, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    nbytes = batch.nbytes + 2 * out.numel() + 8 * batch.index.numel() + 4 * batch.draws.numel()
    return {'ms': round(ms, 4), 'bytes': nbytes, 'region_bytes': batch.nbytes, 'out_bytes': 2 * out.numel(),
            'GB_per_s': round(nbytes / ms / 1e6, 1)}


def copy_costs(batch, iters=10):
    """Host ms of the region H2D copy: from pageable memory, and memcpy into a persistent pinned buffer + async copy."""
    src = batch.regions
    dst = torch.empty(src.numel(), dtype=torch.uint8, device='cuda')
    pinned = torch.empty(src.numel(), dtype=torch.uint8).pin_memory()
    res = {}
    for name in ('pageable', 'pinned_staging'):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            if name == 'pageable':
                dst.copy_(src, non_blocking=True)
            else:
                pinned.copy_(src)
                dst.copy_(pinned, non_blocking=True)
            torch.cuda.synchronize()
        res[name] = round(1e3 * (time.perf_counter() - t0) / iters, 3)
    return res


def decode_kernels(batch, iters=5):
    """ms per batch of each decode kernel: torch.profiler with CUDA activities over ``iters`` decodes of a JpegBatch."""
    from torch.profiler import ProfilerActivity, profile
    dev = batch.replace(tuple(t.cuda() for t in batch.tensors))
    dev.decode()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            dev.decode()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ('jpeg_huffman_kernel', 'jpeg_idct_kernel', 'jpeg_color_kernel'):
            if k in e.key:
                t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
                out[k] = round(t / 1e3 / iters, 3)
    out['total'] = round(sum(out.values()), 3)
    return out


def worker_cpu_ms(root, spec, n=128):
    """Host CPU ms per image of the workers' work (per-image transform, then collate of the batch): the PIL decode
    path of the device crop against the header-only path of device_decode."""
    import glob
    from PIL import Image
    from convnet.pytorch_b200.utils.augment import JpegCollate, JpegDecode, ResizedCropCollate, ScaleCropCollate
    files = sorted(glob.glob(os.path.join(root, '**', '*.jpg'), recursive=True))[:n]
    datas = [open(f, 'rb').read() for f in files]
    host_collate = ResizedCropCollate(spec) if hasattr(spec, 'draw') else ScaleCropCollate(spec)
    res = {}
    for name, fn, collate in (('pil_decode', lambda d: spec(Image.open(__import__('io').BytesIO(d)).convert('RGB')),
                               host_collate), ('device_decode', JpegDecode(spec), JpegCollate(spec))):
        t0 = time.process_time()
        collate([(fn(d), 0) for d in datas])
        res[name] = round(1e3 * (time.process_time() - t0) / len(datas), 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=4)
    ap.add_argument('--workers', type=int, default=os.cpu_count())
    ap.add_argument('--kernel-iters', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('resized_crop_bench needs a CUDA device')
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.data import DataRegime
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    torch.cuda.set_device(0)
    torch.manual_seed(123)
    tmp = tempfile.mkdtemp(prefix='rrc_bench_')
    t0 = time.perf_counter()
    write_jpegs(os.path.join(tmp, 'imagenet'))
    setup_s = time.perf_counter() - t0
    model = convert_b200(models.resnet(dataset='imagenet', depth=50), 'cuda')
    tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device='cuda', print_freq=10 ** 9)

    sampler = torch.utils.data.RandomSampler(range(IMAGES), replacement=True, num_samples=10 ** 7)
    base = {'name': 'imagenet', 'datasets_path': tmp, 'split': 'train', 'augment': True, 'input_size': SIZE,
            'batch_size': B, 'sampler': sampler, 'num_workers': args.workers, 'drop_last': True}
    device_it = iter(DataRegime(None, defaults=dict(base, device_resized_crop=True, pin_memory=False)).get_loader())
    # the host path does not pin either: a pin-memory thread may not allocate while the Trainer captures a graph
    host_it = iter(DataRegime(None, defaults=dict(base, pin_memory=False)).get_loader())
    decode_it = iter(DataRegime(None, defaults=dict(base, device_resized_crop=True, device_decode=True,
                                                    pin_memory=False)).get_loader())
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
    copies = copy_costs(sample)
    dec = decode_kernels(jpeg_batch)
    cpu = worker_cpu_ms(os.path.join(tmp, 'imagenet'), sample.spec)
    gpu, power = card()
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {'model': 'resnet50', 'batch': B, 'size': SIZE, 'images': IMAGES, 'jpeg_setup_s': round(setup_s, 1),
           'steps_per_round': args.steps, 'rounds': args.rounds, 'workers': args.workers,
           'ms_per_step': {k: round(v, 3) for k, v in med.items()},
           'ms_per_step_range': {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
           'img_per_s': {k: round(B / (v / 1e3), 1) for k, v in med.items()},
           'data_wait_ms_mean': {k: round(statistics.mean(v), 3) for k, v in data_wait.items()},
           'h2d_bytes_per_step': {'device': sample.nbytes + 8 * sample.index.numel() + 4 * sample.draws.numel() + 8 * B,
                                  'host': 4 * B * 3 * SIZE * SIZE + 8 * B, 'bound': 0,
                                  'decode': jpeg_batch.payload.numel() + 8 * jpeg_batch.index.numel()
                                  + 4 * jpeg_batch.table.numel() + 8 * B},
           'decode_kernels_ms': dec, 'worker_cpu_ms_per_image': cpu,
           'relayout_kernel': kern, 'relayout_share_of_device_step': round(kern['ms'] / med['device'], 5),
           'region_copy_host_ms': copies, 'graph_replays': tr.graph_replays, 'gpu': gpu, 'power_limit': power,
           'host_cpus': os.cpu_count()}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
