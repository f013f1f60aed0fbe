"""Generates tests/golden/l1_norm.npz by running the UNMODIFIED reference's ``resnet(bn_norm='L1')`` (a checkout of
eladhoffer/convNet.pytorch, read-only) on the CPU.  Run once from the repo root:

    B200_REFERENCE=<reference checkout> python tools/make_l1_norm_golden.py

The reference selects L1BatchNorm2d by rebinding ``torch.nn.BatchNorm2d`` for the whole process, so every model built
here is an L1 model, and the binding is restored before the script ends.

Recorded for ResNet-20 (cifar10) and ResNet-18 (imagenet), each built under torch.manual_seed(123):
  - the state_dict keys, shapes and the SHA-256 of every tensor of the initial state (bit-for-bit init check);
  - the parameter names in ``named_parameters()`` order;
  - the names the reference's WeightDecay regularizer decays (model.regime[0]['regularizer']).
For ResNet-20 also one fp64 training-mode forward/backward: the BN weights, biases and running buffers are first set to
the deterministic values of ``bn_state`` (below, restated by the test) so that no gamma is zero and the momentum update
is visible; the batch of 8 is stored as int8 codes (value = code / 16).  Stored: logits, loss, every parameter's
gradient norm, and the updated running buffers.  Nothing here is needed at test time.
"""
import hashlib
import os
import sys

import numpy as np
import torch
import torch.nn as nn

REF = os.environ.get('B200_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'l1_norm.npz')
MODELS = {'resnet20': dict(dataset='cifar10', depth=20), 'resnet18': dict(dataset='imagenet', depth=18)}


def digest(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


def bn_state(name, C):
    """deterministic BN parameters / buffers of the fp64 step (tests/test_l1_norm_cpu.py restates this)"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name)) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def main():
    if not os.path.isdir(REF):
        raise SystemExit('set B200_REFERENCE to a checkout of eladhoffer/convNet.pytorch')
    sys.path.insert(0, REF)
    bn_class = nn.BatchNorm2d
    import models as ref_models            # noqa: E402
    from utils import regularization as ref_reg   # noqa: E402
    torch.set_num_threads(8)
    blob = {}
    try:
        for tag, cfg in MODELS.items():
            torch.manual_seed(123)
            model = ref_models.resnet(bn_norm='L1', **cfg)
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
            if tag != 'resnet20':
                continue
            model = model.double()
            with torch.no_grad():
                for n, m in model.named_modules():
                    if type(m).__name__ == 'L1BatchNorm2d':
                        for k, v in bn_state(n, m.running_mean.numel()).items():
                            getattr(m, k).copy_(v)
            g = torch.Generator().manual_seed(7)
            codes = torch.randint(-48, 48, (8, 3, 32, 32), generator=g, dtype=torch.int8)
            target = torch.randint(0, 10, (8,), generator=g)
            model.train()
            logits = model(codes.double() / 16)
            loss = nn.functional.cross_entropy(logits, target)
            loss.backward()
            blob['step/x_codes'] = codes.numpy()
            blob['step/target'] = target.numpy()
            blob['step/logits'] = logits.detach().numpy()
            blob['step/loss'] = np.float64(loss.item())
            blob['step/grad_names'] = np.array([n for n, _ in model.named_parameters()])
            blob['step/grad_norms'] = np.array([p.grad.norm().item() for _, p in model.named_parameters()])
            bufs = [(k, v) for k, v in model.state_dict().items() if 'running' in k]
            blob['step/buffer_names'] = np.array([k for k, _ in bufs])
            blob['step/buffers'] = np.concatenate([v.numpy().ravel() for _, v in bufs])
            print('step loss %.12f' % loss.item())
    finally:
        nn.BatchNorm2d = bn_class          # undo the reference's rebinding
    np.savez_compressed(OUT, **blob)
    print('written', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
