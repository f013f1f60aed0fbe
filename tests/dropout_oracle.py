"""TEST INFRASTRUCTURE ONLY -- the dropout mask stream of csrc/dropout.cu restated in numpy, and a functional CPU
restatement of the reference's CIFAR ResNet with in-block dropout (BasicBlock: nn.Dropout after relu(bn1(conv1(x))),
models/resnet.py:81-118 of the reference) that applies given keep masks.

The network code follows oracle/ref_model.py (ResNet forward, BasicBlock, skip path, the bf16 storage points of
``quant``) with the dropout inserted; the BN, convolution, rounding, loss and parameter-naming helpers are
oracle.ref_model's own.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.ref_model import _block_names, _bn, _conv, _q, _skip, cross_entropy, param_names

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xffffffff)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11): ctr uint32 [n, 4], key (k0, k1) -> uint32 [n, 4]"""
    c = [np.asarray(ctr, dtype=np.uint64)[:, i].copy() for i in range(4)]
    k0, k1 = int(key[0]) & 0xffffffff, int(key[1]) & 0xffffffff
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & _LO, p1 >> np.uint64(32), p1 & _LO
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + _W0) & 0xffffffff, (k1 + _W1) & 0xffffffff
    return np.stack(c, axis=1).astype(np.uint32)


def key_words(key):
    """the 64-bit key (an int64 value as the runtime stores it) -> (k0, k1) = (low, high) word"""
    k = int(key) & 0xffffffffffffffff
    return k & 0xffffffff, k >> 32


def threshold(p):
    """(T, c) of ops.dropout_threshold, restated: T = round((1 - p) * 65536) in double, c = fp32(1 / (1 - p))"""
    return int(round((1.0 - p) * 65536.0)), float(np.float32(1.0 / (1.0 - p)))


def keep_mask(key, layer, M, C, T):
    """bool [M, C]: element (row, c) of dropout layer ``layer`` is kept.  Vector g = (row*C + c)/8 uses counter
    {g & 0xffffffff, g >> 32, layer, 0}; its element j the 16-bit uniform (w[j/2] >> 16*(j%2)) & 0xffff < T"""
    g = np.arange(M * C // 8, dtype=np.uint64)
    ctr = np.stack([g & _LO, g >> np.uint64(32), np.full_like(g, layer), np.zeros_like(g)], axis=1)
    w = philox4x32_10(ctr, key_words(key))
    u = np.stack([(w[:, j >> 1] >> np.uint32(16 * (j & 1))) & np.uint32(0xffff) for j in range(8)], axis=1)
    return (u < T).reshape(M, C)


def network_masks(key, spec, N):
    """keep masks of every dropout layer of a network for one step: spec = [(block prefix, layer, C, H, W, p)] ->
    {block prefix: bool tensor [N, C, H, W]} (the kernel numbers rows n*H*W + h*W + w of the NHWC activation)"""
    out = {}
    for prefix, layer, C, H, W, p in spec:
        T, _ = threshold(p)
        m = keep_mask(key, layer, N * H * W, C, T).reshape(N, H, W, C)
        out[prefix] = torch.from_numpy(np.ascontiguousarray(m.transpose(0, 3, 1, 2)))
    return out


def _basic(x, sd, p, stride, training, bufs, quant, mask, rate):
    out = F.relu(_bn(_conv(x, sd, p + '.conv1', stride, 1, quant), sd, p + '.bn1', training, bufs, quant))
    if training and mask is not None:      # nn.Dropout: input * (bernoulli / (1 - p)); the kernels scale by fp32(1/(1-p))
        out = out * (mask.to(out.dtype) * (threshold(rate)[1] if quant else 1.0 / (1.0 - rate)))
    out = _q(out, quant)
    out = _bn(_conv(out, sd, p + '.conv2', 1, 1, quant), sd, p + '.bn2', training, bufs, quant)
    return _q(F.relu(out + _skip(x, sd, p, stride, training, bufs, quant)), quant)


def forward(sd, x, masks, rate, training=True, buffers_out=None, quant=False):
    """logits of a reference-layout CIFAR BasicBlock ResNet ``state_dict`` whose blocks apply dropout with the keep
    masks ``masks`` ({block prefix: bool [N, C, H, W]}) at rate ``rate``; quant: the kernel path's scale fp32(1/(1-p))"""
    x = _q(x, quant)
    x = _conv(x, sd, 'conv1', 1, 1, quant)
    x = _q(F.relu(_bn(x, sd, 'bn1', training, buffers_out, quant)), quant)
    for li, layer in enumerate(('layer1', 'layer2', 'layer3')):
        for bi, p in enumerate(_block_names(sd, layer)):
            stride = 2 if (bi == 0 and li > 0) else 1
            x = _basic(x, sd, p, stride, training, buffers_out, quant, masks.get(p), rate)
    x = _q(x.mean((2, 3)), quant)
    return F.linear(x, sd['fc.weight'], sd['fc.bias'])


def loss_and_grads(sd, x, y, masks, rate, quant=False, training=True):
    """one forward/backward: logits, loss, {param: grad}, updated running buffers (as oracle.ref_model's)"""
    names = param_names(sd)
    work = {k: (v.detach().clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
    bufs = {}
    logits = forward(work, x, masks, rate, training=training, buffers_out=bufs, quant=quant)
    loss = cross_entropy(logits, y)
    grads = torch.autograd.grad(loss, [work[k] for k in names])
    return logits.detach(), loss.detach(), dict(zip(names, grads)), bufs


def block_spec(model, N, H, W):
    """[(block prefix, layer, C, H, W, p)] of a torch CIFAR ResNet's dropout layers in the order the runtime numbers
    them, for an N x 3 x H x W input"""
    spec, layer = [], 0
    for lname in ('layer1', 'layer2', 'layer3'):
        for bi, blk in enumerate(getattr(model, lname)):
            if blk.stride > 1:                # 3x3, padding 1
                H, W = (H + 1) // 2, (W + 1) // 2
            p = float(blk.dropout.p)
            if p:
                spec.append(('%s.%d' % (lname, bi), layer, blk.conv1.out_channels, H, W, p))
                layer += 1
    return spec
