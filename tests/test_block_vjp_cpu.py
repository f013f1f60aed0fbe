"""The block-local references of oracle.ref_model (resnet_stem_vjp, resnet_block_vjp / mobilenet_block_vjp,
resnet_head_vjp), chained through a whole network in fp64 without storage rounding, must reproduce
ref_model.loss_and_grads -- the oracle pinned to the unmodified reference by test_oracle_golden.py: logits, loss, every
parameter gradient and every running buffer.  This shows that the decomposition the GPU block replay
(test_gpu_block_replay.py) compares against is the pinned oracle, including the block strides, the downsample
branches, the summation of a shared SE gate over its stage, the MobileNet identity skips and the head dropout."""
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
        if re.search(r'\.(weight|bias)$', k) and k.rsplit('.', 1)[0] + '.running_var' in sd:       # BatchNorm
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


def _chain(sd, x, y, drop=None):
    """logits, loss, {param: grad}, {buffer: value} of one step assembled from the block-local references"""
    if 'features.0.weight' in sd or 'features.conv0.0.weight' in sd:
        conv, norm, stride, pad, act = ref_model.mobilenet_stem(sd)
        stem = dict(conv=conv, norm=norm, stride=stride, padding=pad, act='relu' if act == 'relu' else 'relu6')
        blocks = [(p, None) for p, _, _ in ref_model.mobilenet_blocks(sd)]
        block_vjp = lambda p, s, h, d: ref_model.mobilenet_block_vjp(sd, p, h, d, quant=False)  # noqa: E731
        fc = 'fc' if 'fc.weight' in sd else 'classifier.1'
    else:
        stem, blocks, fc = {}, _blocks(sd), 'fc'
        block_vjp = lambda p, s, h, d: ref_model.resnet_block_vjp(sd, p, h, d, s, quant=False)  # noqa: E731
    stem_fwd = ref_model.resnet_stem_vjp(sd, x, None, quant=False, **stem)
    h, xs = stem_fwd['y'], []
    for p, s in blocks:
        xs.append(h)
        h = block_vjp(p, s, h, None)['y']
    head = ref_model.resnet_head_vjp(sd, h, y, quant=False, fc=fc, drop=drop)
    grads, bufs = dict(head['grads']), dict(stem_fwd['bufs'])
    d = head['dh']
    for (p, s), xi in zip(reversed(blocks), reversed(xs)):
        r = block_vjp(p, s, xi, d)
        for k, g in r['grads'].items():
            grads[k] = grads[k] + g if k in grads else g
        bufs.update(r['bufs'])
        d = r['dx']
    grads.update(ref_model.resnet_stem_vjp(sd, x, d, quant=False, **stem)['grads'])
    return head['logits'], head['loss'], grads, bufs


def _rel(a, b):
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize('family,cfg,shape,classes,p', [
    ('resnet', dict(dataset='cifar10', depth=20), (3, 32, 32), 10, 0.0),
    ('resnet_se', dict(dataset='imagenet', depth=50), (3, 32, 32), 1000, 0.0),
    ('mobilenet_v2', dict(dataset='imagenet'), (3, 64, 64), 1000, 0.2),
    ('mobilenet', dict(dataset='imagenet'), (3, 64, 64), 1000, 0.0),
    ('mobilenet', dict(dataset='imagenet', shallow=True, width=0.5), (3, 64, 64), 1000, 0.0),
], ids=['resnet20', 'resnet_se50', 'mobilenet_v2_drop02', 'mobilenet_v1', 'mobilenet_v1_shallow_w05'])
def test_block_chain_reproduces_pinned_oracle(family, cfg, shape, classes, p):
    from convnet.pytorch_b200 import models
    sd = _state(getattr(models, family), 5, **cfg)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(4, *shape, generator=g, dtype=D)
    y = torch.randint(0, classes, (4,), generator=g)
    drop = None
    if p > 0:
        # the mask F.dropout draws in the pinned oracle's forward: the same generator state, the same [N, C] draw
        torch.manual_seed(3)
        drop = (torch.nn.functional.dropout(torch.ones(4, sd['classifier.1.weight'].shape[1], dtype=D), p, True) != 0)
        drop = (drop.to(D), p)
        assert 0 < float(drop[0].mean()) < 1
    logits, loss, grads, bufs = _chain(sd, x, y, drop)
    torch.manual_seed(3)
    o_logits, o_loss, o_grads, o_bufs = ref_model.loss_and_grads(sd, x, y, dropout_p=p)
    assert _rel(logits, o_logits) < 1e-12
    assert abs(float(loss) - float(o_loss)) < 1e-12 * abs(float(o_loss))
    assert sorted(grads) == sorted(o_grads)
    if family == 'resnet_se':
        assert sum(1 for k in grads if 'residual_block' in k) == 4 * 4, 'one shared gate per stage'
    for k, v in o_grads.items():
        if k.endswith('.bias') and sd[k[:-len('bias')] + 'weight'].dim() == 4:
            # MobileNet-v1's depthwise bias in front of a training-mode BatchNorm: the gradient is zero up to rounding
            w = float(o_grads[k[:-len('bias')] + 'weight'].norm())
            assert float(v.norm()) < 1e-10 * w and float(grads[k].norm()) < 1e-10 * w, k
            continue
        assert float(v.norm()) > 0, k
        # BatchNorm d gamma and d beta on one scale: in front of a block that starts with conv + BN (MobileNet-v2's
        # blocks without a skip) the loss is invariant to a shift of the output, and d beta is rounding noise
        base = k.rsplit('.', 1)[0]
        scale = float(v.norm())
        if base + '.running_var' in sd:
            scale = max(float(o_grads[base + '.weight'].norm()), float(o_grads[base + '.bias'].norm()))
        assert float((grads[k] - v).norm()) < 1e-10 * scale, '%s: %.3e' % (k, float((grads[k] - v).norm()) / scale)
    assert sorted(bufs) == sorted(o_bufs)
    for k, v in o_bufs.items():
        if 'num_batches' in k:
            assert int(bufs[k]) == int(v) == int(sd[k]) + 1, k
        else:
            assert _rel(bufs[k], v) < 1e-12, k
