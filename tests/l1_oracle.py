"""TEST INFRASTRUCTURE ONLY -- functional CPU restatement of the reference's ResNet with L1 batch normalization
(``resnet(bn_norm='L1')``: models/modules/lp_norm.py:238-291, selected by models/resnet.py:393-399 of the reference).

The network code follows oracle/ref_model.py line by line (ResNet.features/forward, BasicBlock, Bottleneck, downsample,
the bf16 storage points of ``quant``) with every BatchNorm replaced by ``bn_l1``; the convolution, rounding, loss and
parameter-naming helpers are oracle.ref_model's own.  Squeeze-excitation gates are not restated here.
"""
import math

import torch
import torch.nn.functional as F

from oracle.ref_model import _block_names, _conv, _q, cross_entropy, param_names

L1_FIX = math.sqrt(math.pi / 2)


def bn_l1(x, sd, prefix, training, buffers_out):
    """L1BatchNorm2d: s = 1/(mean|x - mean| * sqrt(pi/2) + 1e-5); running = running*0.1 + batch*0.9 with running_var
    holding s; eval uses (running_mean, running_var) as (mean, s)"""
    w, b = sd[prefix + '.weight'], sd[prefix + '.bias']
    rm, rv = sd[prefix + '.running_mean'], sd[prefix + '.running_var']
    if training:
        mean = x.mean((0, 2, 3))
        scale = 1.0 / ((x - mean[None, :, None, None]).abs().mean((0, 2, 3)) * L1_FIX + 1e-5)
        if buffers_out is not None:
            buffers_out[prefix + '.running_mean'] = 0.1 * rm + 0.9 * mean.detach().to(rm.dtype)
            buffers_out[prefix + '.running_var'] = 0.1 * rv + 0.9 * scale.detach().to(rv.dtype)
    else:
        mean, scale = rm.to(x.dtype), rv.to(x.dtype)
    return (x - mean[None, :, None, None]) * (scale * w)[None, :, None, None] + b[None, :, None, None]


def _skip(x, sd, p, stride, training, bufs, quant):
    if p + '.downsample.0.weight' not in sd:
        return x
    return bn_l1(_conv(x, sd, p + '.downsample.0', stride, 0, quant), sd, p + '.downsample.1', training, bufs)


def _bottleneck(x, sd, p, stride, training, bufs, quant):
    out = _q(F.relu(bn_l1(_conv(x, sd, p + '.conv1', 1, 0, quant), sd, p + '.bn1', training, bufs)), quant)
    out = _q(F.relu(bn_l1(_conv(out, sd, p + '.conv2', stride, 1, quant), sd, p + '.bn2', training, bufs)), quant)
    out = bn_l1(_conv(out, sd, p + '.conv3', 1, 0, quant), sd, p + '.bn3', training, bufs)
    return _q(F.relu(out + _skip(x, sd, p, stride, training, bufs, quant)), quant)


def _basic(x, sd, p, stride, training, bufs, quant):
    out = _q(F.relu(bn_l1(_conv(x, sd, p + '.conv1', stride, 1, quant), sd, p + '.bn1', training, bufs)), quant)
    out = bn_l1(_conv(out, sd, p + '.conv2', 1, 1, quant), sd, p + '.bn2', training, bufs)
    return _q(F.relu(out + _skip(x, sd, p, stride, training, bufs, quant)), quant)


def forward(sd, x, training=True, buffers_out=None, quant=False):
    """logits of a reference-layout L1 ResNet ``state_dict`` (cifar or imagenet variant, basic or bottleneck)"""
    if any('.residual_block.' in k for k in sd):
        raise NotImplementedError('squeeze-excitation gates are not restated in the L1 oracle')
    x = _q(x, quant)
    if sd['conv1.weight'].shape[-1] == 7:
        x = _conv(x, sd, 'conv1', 2, 3, quant)
        x = _q(F.relu(bn_l1(x, sd, 'bn1', training, buffers_out)), quant)
        x = F.max_pool2d(x, 3, 2, 1)
    else:
        x = _conv(x, sd, 'conv1', 1, 1, quant)
        x = _q(F.relu(bn_l1(x, sd, 'bn1', training, buffers_out)), quant)
    for li, layer in enumerate(('layer1', 'layer2', 'layer3', 'layer4')):
        for bi, p in enumerate(_block_names(sd, layer)):
            stride = 2 if (bi == 0 and li > 0) else 1
            block = _bottleneck if (p + '.conv3.weight') in sd else _basic
            x = block(x, sd, p, stride, training, buffers_out, quant)
    x = _q(x.mean((2, 3)), quant)
    return F.linear(x, sd['fc.weight'], sd['fc.bias'])


def loss_and_grads(sd, x, y, quant=False, training=True):
    """one forward/backward: logits, loss, {param: grad}, updated running buffers (as oracle.ref_model's)"""
    names = param_names(sd)
    work = {k: (v.detach().clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
    bufs = {}
    logits = forward(work, x, training=training, buffers_out=bufs, quant=quant)
    loss = cross_entropy(logits, y)
    grads = torch.autograd.grad(loss, [work[k] for k in names])
    return logits.detach(), loss.detach(), dict(zip(names, grads)), bufs
