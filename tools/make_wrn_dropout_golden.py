"""Generates tests/golden/wrn_dropout.npz by running the UNMODIFIED reference's CIFAR ResNets with in-block dropout
(``resnet(dropout=0.3)``: nn.Dropout after relu(bn1(conv1(x))) in every BasicBlock) on the CPU.  Run once from the repo
root:

    B200_REFERENCE=<reference checkout> python tools/make_wrn_dropout_golden.py

For WRN-16-4 (depth 16, width [64, 128, 256]) and ResNet-20, each built under torch.manual_seed(123) and converted to
fp64, one training-mode forward/backward of a batch of 4 16x16 images (int8 codes, value = code / 16):
  - the BN weights, biases and running buffers are first set to the deterministic values of ``bn_state`` (restated by
    tests/test_dropout_cpu.py), so that no gamma is zero and every dropout mask reaches the loss;
  - nn.Dropout.forward is replaced, for the duration of the step, by ``input * (mask / (1 - p))`` -- torch's own
    formula -- with a stored Bernoulli(1 - p) keep mask per block, saved bit-packed (np.packbits of the [N, C, H, W]
    bool mask).
Stored: the masks, logits, loss, every parameter's gradient norm and the updated running buffers.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

REF = os.environ.get('B200_REFERENCE', '')
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'wrn_dropout.npz')
P = 0.3
MODELS = {'wrn16_4': dict(dataset='cifar10', depth=16, width=[64, 128, 256], dropout=P),
          'resnet20': dict(dataset='cifar10', depth=20, dropout=P)}
N, HW = 4, 16


def bn_state(name, C):
    """deterministic BN parameters / buffers of the fp64 step (tests/test_dropout_cpu.py restates this)"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name)) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def main():
    if not os.path.isdir(REF):
        raise SystemExit('set B200_REFERENCE to a checkout of eladhoffer/convNet.pytorch')
    sys.path.insert(0, REF)
    import models as ref_models            # noqa: E402
    torch.set_num_threads(8)
    blob = {}
    dropout_forward = nn.Dropout.forward
    try:
        for tag, cfg in MODELS.items():
            torch.manual_seed(123)
            model = ref_models.resnet(**cfg).double()
            with torch.no_grad():
                for n, m in model.named_modules():
                    if isinstance(m, nn.BatchNorm2d):
                        for k, v in bn_state(n, m.num_features).items():
                            getattr(m, k).copy_(v)
            g = torch.Generator().manual_seed(7)
            codes = torch.randint(-48, 48, (N, 3, HW, HW), generator=g, dtype=torch.int8)
            target = torch.randint(0, 10, (N,), generator=g)
            masks = {}

            def hook(mod, inp, out, prefix):       # records each block's activation shape on a dry run
                masks[prefix] = torch.rand(inp[0].shape, generator=g, dtype=torch.float64) < 1 - P
            handles = [m.dropout.register_forward_hook(lambda mod, i, o, p=n: hook(mod, i, o, p))
                       for n, m in model.named_modules() if type(m).__name__ == 'BasicBlock']
            with torch.no_grad():
                model.train()(codes.double() / 16)
            for h in handles:
                h.remove()
            by_module = {id(m.dropout): masks[n] for n, m in model.named_modules() if n in masks}
            nn.Dropout.forward = lambda self, x: x * (by_module[id(self)].to(x.dtype) / (1 - self.p))
            with torch.no_grad():                  # the dry run moved the running buffers: start again from bn_state
                for n, m in model.named_modules():
                    if isinstance(m, nn.BatchNorm2d):
                        for k, v in bn_state(n, m.num_features).items():
                            getattr(m, k).copy_(v)
                        m.num_batches_tracked.zero_()
            logits = model(codes.double() / 16)
            loss = nn.functional.cross_entropy(logits, target)
            loss.backward()
            nn.Dropout.forward = dropout_forward
            blob[tag + '/x_codes'] = codes.numpy()
            blob[tag + '/target'] = target.numpy()
            blob[tag + '/mask_names'] = np.array(sorted(masks))
            for n in sorted(masks):
                blob[tag + '/mask/' + n] = np.packbits(masks[n].numpy().ravel())
                blob[tag + '/mask_shape/' + n] = np.array(masks[n].shape)
            blob[tag + '/logits'] = logits.detach().numpy()
            blob[tag + '/loss'] = np.float64(loss.item())
            blob[tag + '/grad_names'] = np.array([n for n, _ in model.named_parameters()])
            blob[tag + '/grad_norms'] = np.array([p.grad.norm().item() for _, p in model.named_parameters()])
            bufs = [(k, v) for k, v in model.state_dict().items() if 'running' in k]
            blob[tag + '/buffer_names'] = np.array([k for k, _ in bufs])
            blob[tag + '/buffers'] = np.concatenate([v.numpy().ravel() for _, v in bufs])
            print(tag, 'loss %.12f' % loss.item(), len(masks), 'dropout layers')
    finally:
        nn.Dropout.forward = dropout_forward
    np.savez_compressed(OUT, **blob)
    print('written', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
