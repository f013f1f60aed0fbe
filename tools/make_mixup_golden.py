"""Generates tests/golden/mixup.npz by running the UNMODIFIED reference Trainer with MixUp / CutMix (a checkout of
eladhoffer/convNet.pytorch, read-only).  Run once from the repo root:

    B200_REFERENCE=<reference checkout> python tools/make_mixup_golden.py

ResNet-20 on CIFAR-10 shapes (CPU, default init under seed 123).  One fresh batch of 8 per step; its pixels are
multiples of 1/16 in [-4, 4), so the batch is stored exactly as int8 codes (value = code / 16).  The batches come from
a private generator, so only the Trainer consumes the global generators.  After seeding random / numpy / torch, seven
Trainer._step calls run on one model and optimiser: three with mixup=0.2, three with cutmix=1.0, one with both flags
(the reference then runs CutMix with alpha 0.2).

Recorded per step:
  - the draws: permutation, final lambda, CutMix box (by wrapping the reference's _mixup and rand_bbox);
  - the SHA-256 of the mixed fp32 input the model received (bit-for-bit check without storing the tensors);
  - the loss.
For step GRAD_STEP also the gradients it produced: every parameter's gradient norm (fp64) and a fixed seeded sample of
up to 64 entries per parameter (fp32).

numpy >= 1.24 removed np.int, which the reference's rand_bbox calls: the alias is restored in this process only (the
reference itself is not modified).  Nothing here is needed at test time.
"""
import hashlib
import os
import random
import sys

import numpy as np
import torch

REF = os.environ.get('B200_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'mixup.npz')

STEPS = [('mixup', dict(mixup=0.2))] * 3 + [('cutmix', dict(cutmix=1.0))] * 3 + [('both', dict(mixup=0.2, cutmix=1.0))]
GRAD_STEP = 4              # the second CutMix step
SAMPLES_PER_PARAM = 64


def digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


def grad_sample_index(model):
    """{name: sorted int64 indices} -- a seeded sample of each parameter's flattened entries."""
    g = torch.Generator().manual_seed(17)
    return {n: torch.randperm(p.numel(), generator=g)[:SAMPLES_PER_PARAM].sort().values
            for n, p in model.named_parameters()}


def main():
    if not os.path.isdir(REF):
        raise SystemExit('set B200_REFERENCE to a checkout of eladhoffer/convNet.pytorch')
    sys.path.insert(0, REF)
    import models as ref_models            # noqa: E402
    import trainer as ref_trainer          # noqa: E402
    from utils import optim as ref_optim   # noqa: E402
    from utils import cross_entropy as ref_ce  # noqa: E402
    from utils import mixup as ref_mixup   # noqa: E402
    if not hasattr(np, 'int'):
        np.int = int
    torch.set_num_threads(8)
    torch.manual_seed(123)
    model = ref_models.resnet(dataset='cifar10', depth=20)
    opt = ref_optim.OptimRegime(model, model.regime)
    g = torch.Generator().manual_seed(11)
    codes = [torch.randint(-64, 64, (8, 3, 32, 32), generator=g, dtype=torch.int8) for _ in STEPS]
    targets = [torch.randint(0, 10, (8,), generator=g) for _ in STEPS]
    blob = {'x_codes': torch.stack(codes).numpy(), 'y': torch.stack(targets).numpy(),
            'steps': np.array([k for k, _ in STEPS]), 'grad_step': np.int64(GRAD_STEP)}
    draws, boxes, seen = [], [], []
    orig_mixup, orig_bbox = ref_trainer._mixup, ref_mixup.rand_bbox

    def rec_mixup(modules, alpha, batch_size):
        layer = orig_mixup(modules, alpha, batch_size)
        draws.append(layer)
        return layer

    def rec_bbox(size, lam):
        b = orig_bbox(size, lam)
        boxes.append(tuple(int(v) for v in b))
        return b

    ref_trainer._mixup, ref_mixup.rand_bbox = rec_mixup, rec_bbox
    model.register_forward_pre_hook(lambda m, inp: seen.append(digest(inp[0])))
    random.seed(5)
    np.random.seed(5)
    torch.manual_seed(5)
    grads = None
    for i, ((kind, flags), c, y) in enumerate(zip(STEPS, codes, targets)):
        x = c.float() / 16
        tr = ref_trainer.Trainer(model, ref_ce.CrossEntropyLoss(), opt, device_ids=None, device='cpu',
                                 dtype=torch.float, print_freq=1000, **flags)
        tr.training_steps = i
        if i == GRAD_STEP:
            step = opt.step

            def rec_step(*a, **kw):
                nonlocal grads
                grads = {n: p.grad.clone() for n, p in model.named_parameters()}
                return step(*a, **kw)
            opt.step = rec_step
        _, loss, _ = tr._step(x, y, training=True)
        if i == GRAD_STEP:
            del opt.step
        layer = draws[i]
        blob['perm/%d' % i] = layer.mix_index.numpy()
        blob['lam/%d' % i] = layer.mix_values.numpy()
        blob['cutmix/%d' % i] = np.int64(isinstance(layer, ref_mixup.CutMix))
        if isinstance(layer, ref_mixup.CutMix):
            # the reference's (x1, y1, x2, y2) are (first-dim start, second-dim start, ends): stored as (r0, r1, c0, c1)
            b = boxes[-1]
            blob['box/%d' % i] = np.array([b[0], b[2], b[1], b[3]], dtype=np.int64)
        blob['mixed_sha256/%d' % i] = np.array(seen[i])
        blob['loss/%d' % i] = np.float64(float(loss))
        print('mix step %d (%s): lambda %.6f loss %.5f' % (i, kind, float(layer.mix_values), float(loss)))
    ref_trainer._mixup, ref_mixup.rand_bbox = orig_mixup, orig_bbox
    idx = grad_sample_index(model)
    names = [n for n, _ in model.named_parameters()]
    blob['grad_names'] = np.array(names)
    blob['grad_norms'] = np.array([float(grads[n].double().norm()) for n in names])
    blob['grad_samples'] = np.concatenate([grads[n].flatten()[idx[n]].numpy() for n in names])
    np.savez_compressed(OUT, **blob)
    print('written', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
