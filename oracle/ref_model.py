"""TEST INFRASTRUCTURE ONLY -- functional CPU restatement of the reference ResNet training step.

The arithmetic of the reference lives in torch (unpinned in its requirements.txt:1; here torch 2.11): the
restatement therefore spells the reference's model code as explicit calls of the same torch functionals on
a plain ``state_dict`` (no nn.Module, none of this repo's model classes), which makes it an independent
check of both the re-authored model classes and the CUDA pipeline.

Follows, line by line:
  ResNet.features/forward          models/resnet.py:196-213   -> ``forward``
  stem (imagenet / cifar)          models/resnet.py:226-230, 328-332
  Bottleneck.forward               models/resnet.py:141-165   -> ``_bottleneck``
  BasicBlock.forward               models/resnet.py:98-118    -> ``_basic``
  downsample                       models/resnet.py:173-181
  nn.BatchNorm2d train semantics   (eps 1e-5, momentum 0.1, biased var to normalise, unbiased into running_var)
  CrossEntropyLoss                 utils/cross_entropy.py:14-67
  Trainer._step + OptimRegime.step trainer.py:106-177, utils/optim.py:254-264, utils/regularization.py:127-131,
                                   torch.optim.SGD (momentum, first step m = g)   -> ``sgd_step``
  MobileNet_v2.forward             models/mobilenet_v2.py:151-156  -> ``forward_mobilenet_v2``
  ExpandedConv2d.forward           models/mobilenet_v2.py:39-73    (1x1 expand/BN/ReLU6, depthwise 3x3/BN/ReLU6,
                                   1x1 project/BN, identity skip when stride == 1 and C_in == C_out)
  MobileNet WeightDecay filter     models/mobilenet_v2.py:25-36    -> ``is_decayed`` (state-dict aware)
``quant`` emulates the storage precision of the CUDA path: a straight-through bf16 round placed where the
kernels store bf16 (conv outputs, BN/activation outputs, pooled features, their incoming gradients) --
the "T2" oracle of SURVEY.md section 8c.
"""
import re

import torch
import torch.nn.functional as F


class _STRound(torch.autograd.Function):
    """y = bf16(x) in forward; gradient rounded to bf16 in backward (storage emulation)."""

    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).to(g.dtype)


def _q(x, quant):
    return _STRound.apply(x) if quant else x


def _bn(x, sd, prefix, training, buffers_out, quant):
    w, b = sd[prefix + '.weight'], sd[prefix + '.bias']
    rm, rv = sd[prefix + '.running_mean'], sd[prefix + '.running_var']
    if training:
        n = x.numel() // x.size(1)
        mean = x.mean((0, 2, 3))
        var = x.var((0, 2, 3), unbiased=False)
        if buffers_out is not None:
            buffers_out[prefix + '.running_mean'] = 0.9 * rm + 0.1 * mean.detach().to(rm.dtype)
            buffers_out[prefix + '.running_var'] = 0.9 * rv + 0.1 * (var.detach() * n / max(n - 1, 1)).to(rv.dtype)
            buffers_out[prefix + '.num_batches_tracked'] = sd[prefix + '.num_batches_tracked'] + 1
    else:
        mean, var = rm.to(x.dtype), rv.to(x.dtype)
    inv = torch.rsqrt(var + 1e-5)
    return (x - mean[None, :, None, None]) * (inv * w)[None, :, None, None] + b[None, :, None, None]


def _conv(x, sd, name, stride, padding, quant):
    w = sd[name + '.weight']
    # a convolution bias exists only in MobileNet-v1's depthwise layers (models/mobilenet.py:44-46 of the reference)
    b, groups = sd.get(name + '.bias'), x.size(1) // w.size(1)
    if quant and b is not None:
        # storage model of the kernel path: the bf16 tensor holds the convolution WITHOUT its bias (the bias in front of
        # a BatchNorm only shifts the batch mean; the kernels add it to the statistics analytically)
        return _q(F.conv2d(x, w, None, stride=stride, padding=padding, groups=groups), quant) + b.view(1, -1, 1, 1)
    return _q(F.conv2d(x, w, b, stride=stride, padding=padding, groups=groups), quant)


def _block_names(sd, layer):
    idx = sorted({int(m.group(1)) for k in sd for m in [re.match(r'%s\.(\d+)\.' % layer, k)] if m})
    return ['%s.%d' % (layer, i) for i in idx]


def _se_canon(k):
    """resnet_se shares ONE SEBlock per stage between its blocks (models/resnet.py:182-191 of the reference): the
    state_dict lists it under every block; the parameter is the first block's."""
    m = re.match(r'^(layer\d+)\.\d+\.(residual_block\..*)$', k)
    return '%s.0.%s' % (m.group(1), m.group(2)) if m else k


def _skip(x, sd, p, stride, training, bufs, quant):
    r = x
    if p + '.downsample.0.weight' in sd:
        z = _conv(x, sd, p + '.downsample.0', stride, 0, quant)
        r = _bn(z, sd, p + '.downsample.1', training, bufs, quant)
    se = _se_canon(p + '.residual_block.transform.0.weight')
    if se in sd:
        # SEBlock.forward (models/modules/se.py:21-25) on the residual (models/resnet.py:112-113,159-160); storage
        # roundings where the kernels materialise bf16: the residual itself, the pooled mean, the hidden layer, the gate
        q = se[:-len('transform.0.weight')]
        r = _q(r, quant)
        mean = _q(r.mean((2, 3)), quant)
        h = _q(F.relu(F.linear(mean, sd[q + 'transform.0.weight'], sd[q + 'transform.0.bias'])), quant)
        gate = torch.sigmoid(F.linear(h, sd[q + 'transform.2.weight'], sd[q + 'transform.2.bias']))
        r = _q(r * gate[:, :, None, None], quant)
    return r


def _bottleneck(x, sd, p, stride, training, bufs, quant):
    out = _q(F.relu(_bn(_conv(x, sd, p + '.conv1', 1, 0, quant), sd, p + '.bn1', training, bufs, quant)), quant)
    out = _q(F.relu(_bn(_conv(out, sd, p + '.conv2', stride, 1, quant), sd, p + '.bn2', training, bufs, quant)), quant)
    out = _bn(_conv(out, sd, p + '.conv3', 1, 0, quant), sd, p + '.bn3', training, bufs, quant)
    return _q(F.relu(out + _skip(x, sd, p, stride, training, bufs, quant)), quant)


def _basic(x, sd, p, stride, training, bufs, quant):
    out = _q(F.relu(_bn(_conv(x, sd, p + '.conv1', stride, 1, quant), sd, p + '.bn1', training, bufs, quant)), quant)
    out = _bn(_conv(out, sd, p + '.conv2', 1, 1, quant), sd, p + '.bn2', training, bufs, quant)
    return _q(F.relu(out + _skip(x, sd, p, stride, training, bufs, quant)), quant)


# strides of the 17 ExpandedConv2d stages (models/mobilenet_v2.py:91-109: layers_config)
_MBV2_STRIDES = (1, 2, 1, 2, 1, 1, 2, 1, 1, 1, 1, 1, 1, 2, 1, 1, 1)


def _mb_conv_bn(x, sd, conv, bn, stride, pad, act, training, bufs, quant, skip=None, trace=None):
    """conv -> BN -> [ReLU6] (+ identity skip for the linear bottleneck output), with the storage roundings of the
    kernel pipeline: after the conv and after the BN/activation(/add) pass."""
    z = _conv(x, sd, conv, stride, pad, quant)          # groups inferred from the weight shape (depthwise: C/1)
    y = _bn(z, sd, bn, training, bufs, quant)
    if act == 'relu':
        y = F.relu(y)
    elif act:
        y = F.relu6(y)
    if skip is not None:
        y = y + skip
    y = _q(y, quant)
    if trace is not None:
        trace.append({'conv': conv, 'bn': bn, 'stride': stride, 'pad': pad, 'act': act, 'x': x, 'skip': skip, 'y': y})
    return y


# strides of MobileNet-v1's 13 depthwise-separable units (models/mobilenet.py:70-112; the shallow variant drops 5)
_MBV1_STRIDES = (1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)


def mobilenet_stem(sd):
    """(conv, bn, stride, pad, act) of the 3x3/s2 stem of a MobileNet-v2 / v1 ``state_dict``"""
    if 'features.conv0.0.weight' in sd:
        return 'features.conv0.0', 'features.conv0.1', 2, 1, True
    return 'features.0', 'features.1', 2, 1, 'relu'


def mobilenet_blocks(sd):
    """[(prefix, [(conv, bn, stride, pad, act)], add_res)] of the blocks after the stem of a MobileNet-v2 / v1
    ``state_dict``: v2 -- ``features.bottleneck{i}.block`` ([1x1 expand / BN / ReLU6], depthwise 3x3 / BN / ReLU6,
    1x1 project / BN, identity skip when stride == 1 and C_in == C_out), then ``features.conv1`` (1x1 / BN / ReLU6);
    v1 -- ``features.{i}.components`` (depthwise 3x3 with bias / BN / ReLU, 1x1 / BN / ReLU).  ``act``: 'relu',
    True (ReLU6) or False (none), as ``_mb_conv_bn`` takes it."""
    out = []
    if 'features.conv0.0.weight' in sd:
        i = 0
        while 'features.bottleneck%d.block.0.weight' % i in sd:
            p = 'features.bottleneck%d.block' % i
            stride, units, j = _MBV2_STRIDES[i], [], 0
            w0 = sd[p + '.0.weight']
            c_in = w0.shape[1] if w0.shape[1] != 1 else w0.shape[0]
            if w0.shape[1] != 1:                    # expansion != 1: the block starts with the 1x1 expand conv
                units.append((p + '.0', p + '.1', 1, 0, True))
                j = 3
            units.append(('%s.%d' % (p, j), '%s.%d' % (p, j + 1), stride, 1, True))
            units.append(('%s.%d' % (p, j + 3), '%s.%d' % (p, j + 4), 1, 0, False))
            out.append((p, units, stride == 1 and c_in == sd['%s.%d.weight' % (p, j + 3)].shape[0]))
            i += 1
        out.append(('features.conv1', [('features.conv1.0', 'features.conv1.1', 1, 0, True)], False))
        return out
    idx = sorted({int(m.group(1)) for k in sd for m in [re.match(r'features\.(\d+)\.components\.', k)] if m})
    strides = _MBV1_STRIDES if len(idx) == 13 else tuple(s for j, s in enumerate(_MBV1_STRIDES) if not 6 <= j <= 10)
    for j, i in enumerate(idx):
        p = 'features.%d.components' % i
        out.append((p, [(p + '.0', p + '.1', strides[j], 1, 'relu'), (p + '.3', p + '.4', 1, 0, 'relu')], False))
    return out


def _mb_block(x, sd, units, add_res, training, bufs, quant, trace=None):
    """one MobileNet block: its conv/BN(/activation) units in order, the block input added to the last unit's output
    when ``add_res``"""
    inp = x
    for j, (conv, bn, stride, pad, act) in enumerate(units):
        skip = inp if (add_res and j == len(units) - 1) else None
        x = _mb_conv_bn(x, sd, conv, bn, stride, pad, act, training, bufs, quant, skip=skip, trace=trace)
    return x


def _mb_features(sd, x, training, buffers_out, quant, trace):
    x = _q(x, quant)
    x = _mb_conv_bn(x, sd, *mobilenet_stem(sd), training, buffers_out, quant, trace=trace)
    for _, units, add_res in mobilenet_blocks(sd):
        x = _mb_block(x, sd, units, add_res, training, buffers_out, quant, trace=trace)
    return _q(x.mean((2, 3)), quant)


def forward_mobilenet_v1(sd, x, training=True, buffers_out=None, quant=False, trace=None):
    """logits of a reference-layout MobileNet (v1) ``state_dict`` (models/mobilenet.py:39-156): stem conv/BN/ReLU, then
    ``features.{i}.components`` = depthwise 3x3 (with bias) / BN / ReLU / 1x1 / BN / ReLU, average pool, ``fc``."""
    x = _mb_features(sd, x, training, buffers_out, quant, trace)
    return F.linear(x, sd['fc.weight'], sd['fc.bias'])


def mobilenet_v2_unit_trace(sd, x, y, quant=True):
    """Teacher-forcing data for unit-level parity: every conv+BN(+ReLU6)(+skip) unit of one training forward/backward
    with its input ``x``, skip input, output ``y`` and the gradient ``dy`` arriving at its output (all detached).
    Default-init MobileNet-v2 is chaotic end to end (see make_golden.mobilenet_v2_fixture); unit by unit, on the real
    activations and gradients, the comparison is well posed."""
    work = {k: (v.detach().clone().requires_grad_(True) if k in param_names(sd) else v) for k, v in sd.items()}
    trace = []
    if 'features.conv0.0.weight' in sd:
        logits = forward_mobilenet_v2(work, x, True, {}, quant, 0.0, trace=trace)
    else:
        logits = forward_mobilenet_v1(work, x, True, {}, quant, trace=trace)
    loss = cross_entropy(logits, y)
    dys = torch.autograd.grad(loss, [u['y'] for u in trace])
    units = []
    for u, dy in zip(trace, dys):
        units.append({k: (v.detach() if torch.is_tensor(v) else v) for k, v in u.items()})
        units[-1]['dy'] = dy.detach()
    return logits.detach(), loss.detach(), units


def mobilenet_v2_unit_vjp(sd, unit, quant=True, dtype=torch.float64):
    """Local reference of one traced unit in ``dtype``: output y and the vector-Jacobian products of ``dy`` with
    respect to the unit input, the conv weight and the BN affine parameters (same storage roundings as the net)."""
    x = unit['x'].to(dtype).requires_grad_(True)
    names = [unit['conv'] + '.weight', unit['bn'] + '.weight', unit['bn'] + '.bias']
    if unit['conv'] + '.bias' in sd:
        names.append(unit['conv'] + '.bias')
    local = {k: v for k, v in sd.items() if k.startswith(unit['conv'] + '.') or k.startswith(unit['bn'] + '.')}
    local = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in local.items()}
    for n in names:
        local[n] = local[n].detach().clone().requires_grad_(True)
    skip = unit['skip'].to(dtype) if unit['skip'] is not None else None
    yy = _mb_conv_bn(x, local, unit['conv'], unit['bn'], unit['stride'], unit['pad'], unit['act'], True, None, quant,
                     skip=skip)
    grads = torch.autograd.grad(yy, [x] + [local[n] for n in names], unit['dy'].to(dtype))
    return (yy.detach(),) + tuple(grads)          # y, dx, dW, dgamma, dbeta [, dbias of the convolution]


def forward_mobilenet_v2(sd, x, training=True, buffers_out=None, quant=False, dropout_p=0.0, trace=None):
    """logits of a reference-layout MobileNet-v2 ``state_dict`` (models/mobilenet_v2.py:85-156)."""
    x = _mb_features(sd, x, training, buffers_out, quant, trace)
    if training and dropout_p > 0:
        x = F.dropout(x, dropout_p, True)              # same torch generator stream as nn.Dropout in the reference
    return F.linear(x, sd['classifier.1.weight'], sd['classifier.1.bias'])


def forward(sd, x, training=True, buffers_out=None, quant=False, dropout_p=0.0):
    """logits of a reference-layout ``state_dict``: ResNet (cifar or imagenet variant, basic or bottleneck; also
    ResNeXt, whose grouped convolutions are inferred from the weight shapes) or MobileNet-v2."""
    if 'features.conv0.0.weight' in sd:
        return forward_mobilenet_v2(sd, x, training, buffers_out, quant, dropout_p)
    if 'features.0.weight' in sd:
        return forward_mobilenet_v1(sd, x, training, buffers_out, quant)
    x = _q(x, quant)
    imagenet = sd['conv1.weight'].shape[-1] == 7
    if imagenet:
        x = _conv(x, sd, 'conv1', 2, 3, quant)
        x = _q(F.relu(_bn(x, sd, 'bn1', training, buffers_out, quant)), quant)
        x = F.max_pool2d(x, 3, 2, 1)
    else:
        x = _conv(x, sd, 'conv1', 1, 1, quant)
        x = _q(F.relu(_bn(x, sd, 'bn1', training, buffers_out, quant)), quant)
    for li, layer in enumerate(('layer1', 'layer2', 'layer3', 'layer4')):
        for bi, p in enumerate(_block_names(sd, layer)):
            stride = 2 if (bi == 0 and li > 0) else 1
            block = _bottleneck if (p + '.conv3.weight') in sd else _basic
            x = block(x, sd, p, stride, training, buffers_out, quant)
    x = _q(x.mean((2, 3)), quant)
    return F.linear(x, sd['fc.weight'], sd['fc.bias'])


def _leaves(sd, keys, dtype, device):
    """fp64 (``dtype``) copies of the state-dict entries ``keys`` on ``device``; the parameters among them require grad"""
    local = {}
    for k in keys:
        v = sd[k].to(device)
        if v.is_floating_point():
            v = v.to(dtype)
            if not (k.endswith('running_mean') or k.endswith('running_var')):
                v = v.detach().clone().requires_grad_(True)
        local[k] = v
    return local


def _vjp(y, dy, x, local):
    params = [k for k, v in local.items() if torch.is_tensor(v) and v.requires_grad]
    inputs = ([x] if x is not None else []) + [local[k] for k in params]
    grads = torch.autograd.grad(y, inputs, dy.to(y.dtype))
    dx = grads[0] if x is not None else None
    return dx.detach() if dx is not None else None, dict(zip(params, (g.detach() for g in grads[len(inputs) - len(params):])))


def resnet_block_vjp(sd, prefix, x, dy, stride, quant=True, block=None, training=True, dtype=torch.float64):
    """Local reference of one residual block ``prefix`` (e.g. 'layer2.0') of a ResNet-family ``state_dict``: the block
    run in ``dtype`` on the device of ``x`` (NCHW) with the storage roundings of ``quant``, and the vector-Jacobian
    products of ``dy`` (the gradient arriving at its output; None: forward only).  ``block``: the block function (signature of ``_basic``;
    default ``_basic`` / ``_bottleneck`` by the state dict) -- the L1 and dropout restatements plug in here.  A shared
    squeeze-excitation gate appears under its canonical (first block's) names; the gradient of a stage's gate is the sum
    of its blocks' VJPs.  Returns {'y', 'dx', 'grads': {name: grad}, 'bufs': {name: updated running buffer}}."""
    if block is None:
        block = _bottleneck if (prefix + '.conv3.weight') in sd else _basic
    se = _se_canon(prefix + '.residual_block.transform.0.weight')[:-len('transform.0.weight')]
    keys = [k for k in sd if k.startswith(prefix + '.') and not k.startswith(prefix + '.residual_block.')]
    keys += [k for k in sd if k.startswith(se)] if se.endswith('residual_block.') else []
    local = _leaves(sd, keys, dtype, x.device)
    xx = x.to(dtype).requires_grad_(True)
    bufs = {}
    y = block(xx, local, prefix, stride, training, bufs, quant)
    dx, grads = _vjp(y, dy, xx, local) if dy is not None else (None, {})
    return {'y': y.detach(), 'dx': dx, 'grads': grads, 'bufs': {k: v.detach() for k, v in bufs.items()}}


def mobilenet_block_vjp(sd, prefix, x, dy, quant=True, training=True, dtype=torch.float64):
    """Local reference of one MobileNet-v2 / v1 block ``prefix`` (a prefix of ``mobilenet_blocks``, e.g.
    'features.bottleneck2.block', 'features.conv1' or 'features.3.components'), like ``resnet_block_vjp``: the block run
    in ``dtype`` on the device of ``x`` (NCHW) with the storage roundings of ``quant`` and the vector-Jacobian products
    of ``dy`` (None: forward only).  MobileNet-v1's depthwise biases get their (training mode: rounding-noise) gradient
    like any parameter.  Returns {'y', 'dx', 'grads': {name: grad}, 'bufs': {name: updated running buffer}}."""
    (units, add_res), = [(u, a) for p, u, a in mobilenet_blocks(sd) if p == prefix]
    local = _leaves(sd, [k for k in sd if k.startswith(prefix + '.')], dtype, x.device)
    xx = x.to(dtype).requires_grad_(True)
    bufs = {}
    y = _mb_block(xx, local, units, add_res, training, bufs, quant)
    dx, grads = _vjp(y, dy, xx, local) if dy is not None else (None, {})
    return {'y': y.detach(), 'dx': dx, 'grads': grads, 'bufs': {k: v.detach() for k, v in bufs.items()}}


def resnet_stem_vjp(sd, x, dy, quant=True, bn=None, dtype=torch.float64, conv='conv1', norm='bn1', stride=None,
                    padding=None, act='relu'):
    """Local reference of the stem on its relayouted input ``x`` (NCHW, the bf16 values the convolution reads): conv
    ``conv`` -> BN ``norm`` -> activation (-> 3x3/s2 max-pool for the 7x7 stem), with the VJPs of ``dy`` (None:
    forward only).  Defaults: the ResNet stem (7x7/s2/pad 3 + max-pool or 3x3/s1/pad 1, ReLU); the MobileNet stems
    pass their names, stride 2, padding 1 and ``act`` 'relu6' (v2) or 'relu' (v1), see ``mobilenet_stem``.  ``bn``:
    the BatchNorm function (signature of ``_bn`` without ``quant``; default ``_bn``).  Returns {'y', 'grads',
    'bufs'}."""
    if bn is None:
        bn = lambda t, sd_, p, training, bufs: _bn(t, sd_, p, training, bufs, quant)  # noqa: E731
    local = _leaves(sd, [k for k in sd if k.startswith(conv + '.') or k.startswith(norm + '.')], dtype, x.device)
    bufs = {}
    imagenet = local[conv + '.weight'].shape[-1] == 7
    if stride is None:
        stride, padding = (2, 3) if imagenet else (1, 1)
    z = _conv(x.to(dtype), local, conv, stride, padding, quant)
    y = bn(z, local, norm, True, bufs)
    y = _q(F.relu6(y) if act == 'relu6' else F.relu(y), quant)
    if imagenet:
        y = F.max_pool2d(y, 3, 2, 1)
    _, grads = _vjp(y, dy, None, local) if dy is not None else (None, {})
    return {'y': y.detach(), 'grads': grads, 'bufs': {k: v.detach() for k, v in bufs.items()}}


def resnet_head_vjp(sd, h, target, smooth_eps=0.0, soft=None, upstream=1.0, quant=True, dtype=torch.float64, fc='fc',
                    drop=None):
    """Local reference of the classifier head on the last block's output ``h`` (NCHW): global average pool ->
    (dropout) -> linear ``fc`` ('fc', or MobileNet-v2's 'classifier.1') -> mean cross-entropy (label smoothing
    ``smooth_eps``, or the soft MixUp / CutMix target of ``soft`` = (t2, lam): lam * onehot(target) + (1 - lam) *
    onehot(t2)), differentiated with the upstream gradient ``upstream``.  ``drop`` = (keep, p): the 0/1 keep mask
    [N, C] of a dropout with rate p, applied as F.dropout applies it, keep * x / (1 - p), with one storage rounding.
    The gradient of the logits is stored in bf16 before the classifier's backward reads it.  Returns {'logits', 'loss',
    'top1', 'top5' (percent of rows whose target is among the 1 / 5 largest logits), 'dlogits', 'grads', 'dh'}."""
    w, b = sd[fc + '.weight'].to(h.device, dtype), sd[fc + '.bias'].to(h.device, dtype)
    feat = _q(h.to(dtype).mean((2, 3)), quant)
    scale = None
    if drop is not None:
        scale = drop[0].to(h.device, dtype) / (1.0 - drop[1])
        feat = _q(feat * scale, quant)
    logits = (feat @ w.t() + b).detach().requires_grad_(True)
    n_cls = logits.shape[1]
    if soft is None:
        loss = cross_entropy(logits, target, smooth_eps)
    else:
        lam = float(soft[1])
        q = lam * F.one_hot(target, n_cls).to(dtype) + (1.0 - lam) * F.one_hot(soft[0], n_cls).to(dtype)
        loss = (-(q * F.log_softmax(logits, dim=-1)).sum(-1)).mean()
    (dl,) = torch.autograd.grad(loss, [logits])
    dl = _q(dl * upstream, quant)
    dfeat = _q(dl @ w, quant)
    if scale is not None:
        dfeat = _q(dfeat * scale, quant)
    HW = h.shape[2] * h.shape[3]
    dh = (dfeat / HW)[:, :, None, None].expand(h.shape)
    picked = logits.gather(1, target.view(-1, 1))
    above = (logits > picked).sum(1)        # a row counts when fewer than k logits lie strictly above its target's
    return {'logits': logits.detach(), 'loss': loss.detach(), 'top1': float((above < 1).double().mean()) * 100,
            'top5': float((above < 5).double().mean()) * 100, 'dlogits': dl, 'feat': feat,
            'grads': {fc + '.weight': dl.t() @ feat, fc + '.bias': dl.sum(0)}, 'dh': _q(dh, quant)}


def cross_entropy(logits, target, smooth_eps=0.0):
    """mean over the batch of -((1-eps-eps/C) lsm[t] + (eps/C) sum_c lsm[c])  (utils/cross_entropy.py:48-52);
    with eps = 0 this is F.cross_entropy (:20-24)."""
    lsm = F.log_softmax(logits, dim=-1)
    n_cls = logits.size(-1)
    u = smooth_eps / n_cls
    picked = lsm.gather(-1, target.view(-1, 1)).squeeze(-1)
    return (-((1.0 - u - smooth_eps) * picked + u * lsm.sum(-1))).mean()


def is_decayed(name, sd=None):
    """membership of the reference's WeightDecay filter: ResNet family (models/resnet.py:34-40) -- not a bias, not in
    a BN; MobileNet-v2 (models/mobilenet_v2.py:25-36, needs ``sd``) -- weights of nn.Linear and of the NON-depthwise
    convolutions only."""
    if name.endswith('bias'):
        return False
    if name.startswith('features.') or name.startswith('classifier.'):
        w = sd[name]
        return w.dim() == 2 or (w.dim() == 4 and w.shape[1] != 1)
    return not re.search(r'(^|\.)bn\d*\.|downsample\.1\.', name)


def param_names(sd):
    return [k for k in sd if not (k.endswith('running_mean') or k.endswith('running_var')
                                  or k.endswith('num_batches_tracked')) and _se_canon(k) == k]


def loss_and_grads(sd, x, y, smooth_eps=0.0, quant=False, training=True, dropout_p=0.0):
    """One forward/backward: returns logits, loss, {param: grad}, updated BN buffers."""
    names = param_names(sd)
    work = {k: (v.detach().clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
    bufs = {}
    logits = forward(work, x, training=training, buffers_out=bufs, quant=quant, dropout_p=dropout_p)
    loss = cross_entropy(logits, y, smooth_eps)
    grads = torch.autograd.grad(loss, [work[k] for k in names])
    return logits.detach(), loss.detach(), dict(zip(names, grads)), bufs


def sgd_step(sd, grads, momentum_buf, lr, momentum=0.9, weight_decay=1e-4, loss_scale=1.0):
    """unscale -> WeightDecay.pre_step (decayed set only) -> SGD with momentum (first step: m = g)."""
    new_sd, new_m = dict(sd), {}
    for k, g in grads.items():
        g = g / loss_scale
        if is_decayed(k, sd):
            g = g + weight_decay * sd[k]
        m = g.clone() if momentum_buf.get(k) is None else momentum * momentum_buf[k] + g
        new_m[k] = m
        new_sd[k] = sd[k] - lr * m
    for k in sd:                              # aliases of shared parameters (SE gates) follow their owner
        if _se_canon(k) != k and _se_canon(k) in new_sd:
            new_sd[k] = new_sd[_se_canon(k)]
    return new_sd, new_m


def train_steps(sd, x, y, steps, lr=0.1, momentum=0.9, weight_decay=1e-4, quant=False, smooth_eps=0.0):
    """``steps`` full training steps on one resident batch; returns final state, momentum and the loss trace."""
    mom, losses = {}, []
    for _ in range(steps):
        _, loss, grads, bufs = loss_and_grads(sd, x, y, smooth_eps=smooth_eps, quant=quant)
        sd, mom = sgd_step(sd, grads, mom, lr, momentum, weight_decay)
        sd.update(bufs)
        losses.append(float(loss))
    return sd, mom, losses
