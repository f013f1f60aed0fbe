"""Generates tests/golden/checkpoint_segments.npz by running the UNMODIFIED reference's
``resnet(checkpoint_segments=s)`` (a checkout of eladhoffer/convNet.pytorch, read-only) on the CPU.  Run once from the
repo root:

    B200_REFERENCE=<reference checkout> python tools/make_checkpoint_golden.py

Recorded, each model built under torch.manual_seed(123):
  - ResNet-50 (imagenet) with s in {1, 2, 4}: the state_dict keys, shapes and the SHA-256 of every tensor of the
    initial state, the parameter names in ``named_parameters()`` order and the names the reference's WeightDecay
    regularizer decays;
  - ResNet-18 (imagenet) with s in {1, 2}: one fp64 training-mode forward/backward at 32 px.  The BN weights, biases and
    running buffers are first set to the deterministic values of ``bn_state`` (below, restated by the test) so that no
    gamma is zero and the momentum update is visible; the batch of 4 is stored as int8 codes (value = code / 16).
    Stored: logits, loss, every parameter's gradient norm, the running buffers and every ``num_batches_tracked`` after
    the step (2 inside checkpointed segments: the reentrant recompute updates them again).
Nothing here is needed at test time.
"""
import hashlib
import os
import sys
import warnings

import numpy as np
import torch
import torch.nn as nn

REF = os.environ.get('B200_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden',
                   'checkpoint_segments.npz')


def digest(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


def bn_state(name, C):
    """deterministic BN parameters / buffers of the fp64 step (tests/test_checkpoint_cpu.py restates this)"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name)) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def main():
    if not os.path.isdir(REF):
        raise SystemExit('set B200_REFERENCE to a checkout of eladhoffer/convNet.pytorch')
    sys.path.insert(0, REF)
    import models as ref_models            # noqa: E402
    from utils import regularization as ref_reg   # noqa: E402
    warnings.filterwarnings('ignore', message='.*use_reentrant.*')   # the reference does not pass it
    torch.set_num_threads(8)
    blob = {}
    for s in (1, 2, 4):
        tag = 'resnet50_s%d' % s
        torch.manual_seed(123)
        model = ref_models.resnet(dataset='imagenet', depth=50, checkpoint_segments=s)
        sd = model.state_dict()
        blob[tag + '/keys'] = np.array(list(sd.keys()))
        blob[tag + '/shapes'] = np.array([','.join(map(str, v.shape)) for v in sd.values()])
        blob[tag + '/sha256'] = np.array([digest(v) for v in sd.values()])
        blob[tag + '/params'] = np.array([n for n, _ in model.named_parameters()])
        reg = dict(model.regime[0]['regularizer'])
        reg.pop('name')
        wd = ref_reg.WeightDecay(model, **reg)
        blob[tag + '/decayed'] = np.array([n for n, _ in wd.named_parameters()])
        print(tag, len(sd), 'tensors,', len(blob[tag + '/decayed']), 'decayed')
    g = torch.Generator().manual_seed(7)
    codes = torch.randint(-48, 48, (4, 3, 32, 32), generator=g, dtype=torch.int8)
    target = torch.randint(0, 1000, (4,), generator=g)
    blob['step/x_codes'] = codes.numpy()
    blob['step/target'] = target.numpy()
    for s in (1, 2):
        tag = 'step_s%d' % s
        torch.manual_seed(123)
        model = ref_models.resnet(dataset='imagenet', depth=18, checkpoint_segments=s).double()
        with torch.no_grad():
            for n, m in model.named_modules():
                if isinstance(m, nn.BatchNorm2d):
                    for k, v in bn_state(n, m.num_features).items():
                        getattr(m, k).copy_(v)
        model.train()
        logits = model(codes.double() / 16)
        loss = nn.functional.cross_entropy(logits, target)
        loss.backward()
        blob[tag + '/logits'] = logits.detach().numpy()
        blob[tag + '/loss'] = np.float64(loss.item())
        blob[tag + '/grad_names'] = np.array([n for n, _ in model.named_parameters()])
        blob[tag + '/grad_norms'] = np.array([p.grad.norm().item() for _, p in model.named_parameters()])
        sd = model.state_dict()
        bufs = [k for k in sd if 'running' in k]
        blob[tag + '/buffer_names'] = np.array(bufs)
        blob[tag + '/buffers'] = np.concatenate([sd[k].numpy().ravel() for k in bufs])
        tracked = [k for k in sd if k.endswith('num_batches_tracked')]
        blob[tag + '/tracked_names'] = np.array(tracked)
        blob[tag + '/tracked'] = np.array([int(sd[k]) for k in tracked])
        print(tag, 'loss %.12f' % loss.item(), 'num_batches_tracked', blob[tag + '/tracked'].tolist())
    np.savez_compressed(OUT, **blob)
    print('written', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
