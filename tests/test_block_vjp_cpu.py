"""The block-local references of oracle.ref_model (resnet_stem_vjp, resnet_block_vjp, resnet_head_vjp), chained through
a whole network in fp64 without storage rounding, must reproduce ref_model.loss_and_grads -- the oracle pinned to the
unmodified reference by test_oracle_golden.py: logits, loss, every parameter gradient and every running buffer.  This
shows that the decomposition the GPU block replay (test_gpu_block_replay.py) compares against is the pinned oracle,
including the block strides, the downsample branches and the summation of a shared SE gate over its stage."""
import re

import pytest
import torch

from oracle import ref_model

D = torch.float64


def _state(factory, seed, **cfg):
    """fp64 state dict of a registry model with every BatchNorm affine parameter drawn away from its initial value (at
    init the last BN of each block has gamma = 0 and half of the gradients would be exactly zero)"""
    torch.manual_seed(seed)
    sd = {k: (v.to(D) if v.is_floating_point() else v) for k, v in factory(**cfg).state_dict().items()}
    g = torch.Generator().manual_seed(seed)
    for k in sd:
        if re.search(r'(^|\.)(bn\d*|downsample\.1)\.(weight|bias)$', k):
            sd[k] = 0.5 * torch.randn(sd[k].shape, generator=g, dtype=D) + (1.0 if k.endswith('weight') else 0.0)
        elif k.endswith('running_var'):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g, dtype=D)
    return sd


def _blocks(sd):
    out = []
    for li, layer in enumerate(('layer1', 'layer2', 'layer3', 'layer4')):
        for bi, p in enumerate(ref_model._block_names(sd, layer)):
            out.append((p, 2 if (bi == 0 and li > 0) else 1))
    return out


def _chain(sd, x, y):
    """logits, loss, {param: grad}, {buffer: value} of one step assembled from the block-local references"""
    blocks = _blocks(sd)
    stem_fwd = ref_model.resnet_stem_vjp(sd, x, None, quant=False)
    h, xs = stem_fwd['y'], []
    for p, s in blocks:
        xs.append(h)
        h = ref_model.resnet_block_vjp(sd, p, h, None, s, quant=False)['y']
    head = ref_model.resnet_head_vjp(sd, h, y, quant=False)
    grads, bufs = dict(head['grads']), dict(stem_fwd['bufs'])
    d = head['dh']
    for (p, s), xi in zip(reversed(blocks), reversed(xs)):
        r = ref_model.resnet_block_vjp(sd, p, xi, d, s, quant=False)
        for k, g in r['grads'].items():
            grads[k] = grads[k] + g if k in grads else g
        bufs.update(r['bufs'])
        d = r['dx']
    grads.update(ref_model.resnet_stem_vjp(sd, x, d, quant=False)['grads'])
    return head['logits'], head['loss'], grads, bufs


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize('family,cfg,shape,classes', [
    ('resnet', dict(dataset='cifar10', depth=20), (3, 32, 32), 10),
    ('resnet_se', dict(dataset='imagenet', depth=50), (3, 32, 32), 1000),
], ids=['resnet20', 'resnet_se50'])
def test_block_chain_reproduces_pinned_oracle(family, cfg, shape, classes):
    from convnet.pytorch_b200 import models
    sd = _state(getattr(models, family), 5, **cfg)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(4, *shape, generator=g, dtype=D)
    y = torch.randint(0, classes, (4,), generator=g)
    logits, loss, grads, bufs = _chain(sd, x, y)
    o_logits, o_loss, o_grads, o_bufs = ref_model.loss_and_grads(sd, x, y)
    assert _rel(logits, o_logits) < 1e-12
    assert abs(float(loss) - float(o_loss)) < 1e-12 * abs(float(o_loss))
    assert sorted(grads) == sorted(o_grads)
    if family == 'resnet_se':
        assert sum(1 for k in grads if 'residual_block' in k) == 4 * 4, 'one shared gate per stage'
    for k, v in o_grads.items():
        assert float(v.norm()) > 0, k
        assert _rel(grads[k], v) < 1e-10, '%s: %.3e' % (k, _rel(grads[k], v))
    assert sorted(bufs) == sorted(o_bufs)
    for k, v in o_bufs.items():
        if 'num_batches' in k:
            assert int(bufs[k]) == int(v) == int(sd[k]) + 1, k
        else:
            assert _rel(bufs[k], v) < 1e-12, k
