"""Block-by-block replay of real ResNet-family and MobileNet training steps against fp64, teacher-forced from the
engine's own tensors.

The network-level checks (test_gpu_engine._check_against_bf16_oracle and its L1 / dropout copies) accept per-tensor
errors of several percent, because a whole bf16-storage network is that sensitive to which way single roundings fall.
A wiring error that moves one block's d gamma, one downsample gradient or one running variance by 1-3 % passes them.
Here the inputs of every block are the engine's own, so only that block's rounding separates the two sides:

  1. record one eager ``Runtime.train_step``: the stem / block / head methods of the runtime instance are wrapped
     so that each clones its input and output (x, y) and the gradient it receives and returns (dy, dx); the stem's
     input is the relayout output (decoded from the bordered space-to-depth layout of the 7x7 stem, or the padded
     NHWC input of a 3x3 stem), so MixUp / CutMix steps replay like any other; the head's dropout mask is taken from
     its tape.  The arena gradients and the running buffers are read before and after the step;
  2. run each block in fp64 on the GPU (``oracle.ref_model.resnet_block_vjp`` with the storage roundings of the kernel
     path; the L1 and dropout restatements of tests/l1_oracle.py and tests/dropout_oracle.py, the keep masks regenerated
     from ``rt.dropout_key``; ``oracle.ref_model.mobilenet_block_vjp`` for the MobileNet blocks), the stem (conv, BN,
     ReLU / ReLU6, max-pool) and the head (average pool, dropout, fc, cross-entropy with label smoothing or the soft
     MixUp / CutMix target, the upstream gradient);
  3. compare each block's y, dx, every parameter gradient and its running buffers after the step (the shared SE gate of
     a stage against the sum of its blocks' VJPs), and require the recorded tensors to chain bit for bit: block i's
     output is block i+1's input, block i+1's dx is block i's dy, and likewise at the stem and the head;
  4. inside the blocks, teacher-force every unit (_replay_units): each BatchNorm backward (dz, g, d gamma / d beta) on
     the engine's own z and dy (the ReLU6 gate 0 < pre < 6 as the kernels decide it), the running statistics on the
     engine's own z (plus MobileNet-v1's depthwise bias), each convolution's dgrad and wgrad (depthwise: groups = C) on
     the engine's own x and dz.  A whole bottleneck block is ill-conditioned (see LOOSE), a single unit is not: these bounds
     are tight on every configuration.

Every bound and the worst value measured per quantity are printed (``-s``) with configuration and block.  Mutants
(test_mutant_is_caught) plant one wiring fault each and must fail the replay in the block and quantity they touch.
The state is "state B" of test_gpu_engine._pair: a few fp32 SGD steps, so that no last-BN gamma is zero."""
import time

import numpy as np
import pytest
import torch

import dropout_oracle
import l1_oracle
from test_gpu_engine import _pair, _rel, _setup

pytestmark = pytest.mark.gpu

BATCH = 32

# configuration -> model family, factory arguments, input size, classes, train_step variant
CONFIGS = {
    'resnet20': dict(family='resnet', cfg=dict(dataset='cifar10', depth=20), px=32, classes=10),
    'resnext20': dict(family='resnext', cfg=dict(dataset='cifar10', depth=20), px=32, classes=10),
    'resnet20_l1': dict(family='resnet', cfg=dict(dataset='cifar10', depth=20, bn_norm='L1'), px=32, classes=10),
    'wrn16_4_dropout': dict(family='resnet', cfg=dict(dataset='cifar10', depth=16, width=[64, 128, 256], dropout=0.3),
                            px=32, classes=10),
    'resnet18': dict(family='resnet', cfg=dict(dataset='imagenet', depth=18), px=128, classes=1000),
    'resnet18_l1': dict(family='resnet', cfg=dict(dataset='imagenet', depth=18, bn_norm='L1'), px=128, classes=1000),
    'resnet50': dict(family='resnet', cfg=dict(dataset='imagenet', depth=50), px=128, classes=1000),
    'resnext50': dict(family='resnext', cfg=dict(dataset='imagenet', depth=50), px=64, classes=1000),
    'resnet_se50': dict(family='resnet_se', cfg=dict(dataset='imagenet', depth=50), px=64, classes=1000),
    'resnext_se50': dict(family='resnext_se', cfg=dict(dataset='imagenet', depth=50), px=64, classes=1000),
    # train_step variants
    'resnet20_smooth': dict(family='resnet', cfg=dict(dataset='cifar10', depth=20), px=32, classes=10, smooth=0.1),
    'resnet18_upstream8': dict(family='resnet', cfg=dict(dataset='imagenet', depth=18), px=128, classes=1000,
                               upstream=8.0),
    'resnet18_mixup': dict(family='resnet', cfg=dict(dataset='imagenet', depth=18), px=128, classes=1000,
                           mix=('mixup', 0.37)),
    'resnet20_cutmix': dict(family='resnet', cfg=dict(dataset='cifar10', depth=20), px=32, classes=10,
                            mix=('cutmix', (5, 21, 8, 30))),
    # MobileNet-v2 (bench.py's config C4; 'drop': the rate of its head Dropout, set before conversion, default 0.2)
    # and MobileNet-v1.  At 112 px the last stride-2 depthwise convolution reads an odd 7 x 7 map (-> 4 x 4)
    'mobilenet_v2': dict(family='mobilenet_v2', cfg=dict(dataset='imagenet'), px=224, classes=1000),
    'mobilenet_v2_112': dict(family='mobilenet_v2', cfg=dict(dataset='imagenet'), px=112, classes=1000),
    # 'clip': BatchNorms whose gamma / beta are raised before the step so that their ReLU6 clips (see _raise_bns)
    'mobilenet_v2_relu6': dict(family='mobilenet_v2', cfg=dict(dataset='imagenet'), px=112, classes=1000, drop=0.0,
                               clip=('features.conv0.1', 'features.bottleneck2.block.1', 'features.bottleneck2.block.4',
                                     'features.bottleneck5.block.4', 'features.bottleneck14.block.1',
                                     'features.conv1.1')),
    'mobilenet_v2_drop01': dict(family='mobilenet_v2', cfg=dict(dataset='imagenet'), px=112, classes=1000, drop=0.1),
    'mobilenet_v2_smooth_upstream8': dict(family='mobilenet_v2', cfg=dict(dataset='imagenet'), px=112, classes=1000,
                                          smooth=0.1, upstream=8.0),
    'mobilenet_v2_cutmix': dict(family='mobilenet_v2', cfg=dict(dataset='imagenet'), px=112, classes=1000,
                                mix=('cutmix', (17, 70, 9, 88))),
    'mobilenet_v1': dict(family='mobilenet', cfg=dict(dataset='imagenet'), px=112, classes=1000),
    'mobilenet_v1_shallow_w05': dict(family='mobilenet', cfg=dict(dataset='imagenet', shallow=True, width=0.5), px=112,
                                     classes=1000),
}

# rel-L2 bounds per quantity class.  'affine': d gamma and d beta of one BN on ONE scale, the norm of the larger of the
# two (d gamma can cancel almost completely, as in test_gpu_engine._mobilenet_parity).  Running means are measured
# against the norm of sqrt(running_var) (a running mean can sit near zero; L1 BatchNorm: of 1 / running_var), running
# variances against their own norm.
BOUNDS = {
    'y': 5e-3, 'dx': 5e-3, 'dW': 5e-3, 'affine': 5e-3, 'SE grad': 5e-3,
    'running_mean': 2e-5, 'running_var': 2e-5,
    'stem y': 5e-3, 'stem dW': 5e-3, 'stem affine': 5e-3,
    'logits': 2e-4, 'loss': 5e-5, 'dlogits': 5e-3, 'fc grad': 5e-3, 'dh': 5e-3,
    'eval y': 5e-3, 'eval y folded': 1e-2,
    # unit level (_replay_units): one bf16 rounding of dz / of the dgrad output, fp32 sums for the rest
    'unit dz': 3e-3, 'unit g': 1e-3, 'unit affine': 1e-4, 'unit running_mean': 2e-6, 'unit running_var': 2e-6,
    'unit dgrad': 3e-3, 'unit wgrad': 1e-4, 'unit coeffs': 1e-5,
    # MobileNet-v1's depthwise bias: the engine's gradient is exactly zero (asserted); the reference's, sum(dz) over a
    # training-mode BatchNorm, is fp64 rounding noise, measured against the norm of the same convolution's dW
    'bias noise': 1e-10,
}
# The floors above hold for the CIFAR configurations (measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, worst
# over five runs: dx 1.7e-3, dW 1.3e-3, affine 1.3e-3, running statistics 9.4e-6).  The whole blocks of the ImageNet
# configurations are ill-conditioned in their own right, so their whole-block bounds (LOOSE) only catch wiring errors
# of several percent, such as a wrong tensor fed to a branch.  Measured there, worst over five runs (the fp32 warm-up is
# not bitwise reproducible, so the state moves a little): dx 2.2e-2, dW 2.6e-2, affine 3.0e-2, the shared SE gates 9.5e-3
# (ResNet-50 / ResNeXt / SE bottlenecks at 64 and 128 px, ResNet-18 and its L1 variant at 128 px); running statistics
# 4.4e-5 (L1 BatchNorm at 4 x 4 px).  The block output agrees to 9e-4 everywhere; the excess is in the gradients of the
# inner units: the same fp64 block reference evaluated in fp32 (same storage roundings, TF32 off) differs from itself by
# up to 2 % there, because single bf16 roundings of dz and of the dgrad outputs that fall the other way are amplified
# by the BatchNorm backward's cancellation at M = 128..2048 rows.  The unit-level bounds ('unit ...', _replay_units) do
# not have that problem and hold for every configuration: measured dz 1.8e-3, dgrad 1.7e-3 (one bf16 rounding each),
# d gamma / d beta 5.8e-7, wgrad 3.1e-5, BN coefficients 1.9e-7, running statistics 1.3e-7; logits 4.4e-6, loss 6.9e-6.
LOOSE = dict(dx=4e-2, dW=5e-2, affine=6e-2, running_mean=1e-4, running_var=1e-4)
LOOSE['SE grad'] = 3e-2
# The MobileNet blocks (1x1 expand, depthwise 3x3 and 1x1 project units, each re-rounded to bf16 after its BatchNorm)
# sit between the two.  Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, worst over three runs of the
# eight MobileNet configurations: dx 3.8e-3, dW 4.6e-3, affine 1.1e-2 (the BNs of the later units of a block, whose
# inputs lie one or two units past the teacher-forced block input).  The same fp64 block reference evaluated in fp32
# (same storage roundings, TF32 off) differs from itself by up to dx 1.3e-3, dW 1.4e-3, affine 2.2e-3 on the same
# blocks (MobileNet-v2 at 224 px, v1 at 112 px).  The block outputs agree to 6.4e-4, and every unit-level bound holds
# unchanged: dz 1.7e-3, dgrad 1.7e-3, wgrad 2.0e-5 (the depthwise weight gradients, up to 32 x 112 x 112 products
# per element, included), d gamma / d beta 6.7e-7, running statistics 1.4e-7.
MB_LOOSE = dict(dx=1e-2, dW=1e-2, affine=2e-2)
for _c in CONFIGS.values():
    if _c['cfg']['dataset'] == 'imagenet':
        _c['loose'] = MB_LOOSE if _c['family'].startswith('mobilenet') else LOOSE
WORST = {}          # quantity class -> (value, bound, config, where)


@pytest.fixture(scope='module', autouse=True)
def _report_at_end():
    """after the last test of this file that ran: the worst value per quantity over those tests and their wall time"""
    WORST.clear()
    t0 = time.time()
    yield
    _report('block replay, the tests of this file that ran')
    print('block replay: %.1f s wall for the tests of this file that ran' % (time.time() - t0))


def _note(cls, value, config, where, failures, quantity=None):
    bound = CONFIGS.get(config, {}).get('loose', {}).get(cls, BOUNDS[cls])
    if value > WORST.get(cls, (-1.0,))[0]:
        WORST[cls] = (value, bound, config, where)
    if not value <= bound:
        failures.append((where, quantity or cls, value, bound))


def _report(title):
    lines = ['%s: worst rel-L2 per quantity (its bound; CIFAR bound; config, block)' % title]
    for cls in BOUNDS:
        if cls in WORST:
            v, bound, config, where = WORST[cls]
            lines.append('  %-14s %.3e  (bound %.1e; CIFAR %.1e)  %s %s' % (cls, v, bound, BOUNDS[cls], config, where))
    print('\n'.join(lines))


# ---------------------------------------------------------------------------------------------------- setup
def _build(name):
    from convnet.pytorch_b200 import models
    c = CONFIGS[name]
    factory = getattr(models, c['family'])
    if 'drop' in c:
        def factory(**cfg):
            m = models.mobilenet_v2(**cfg)
            m.classifier[0].p = c['drop']
            return m
    ref, mine, x, y = _pair(factory, c['cfg'], (3, c['px'], c['px']), c['classes'], batch=BATCH)
    if 'clip' in c:
        _raise_bns(mine, c['clip'])
    return ref, mine, x, y


def _raise_bns(mine, names):
    """gamma x 4 and beta + 3 on the named BatchNorms: bn(z) = 4 z^ + 3 with z^ ~ N(0, 1) takes its ReLU6 above 6 for
    z^ > 0.75 and below 0 for z^ < -0.75, so both edges of the gate carry gradient (a few fp32 SGD steps leave almost
    no pre-activation above 6)"""
    params = dict(mine.named_parameters())
    with torch.no_grad():
        for n in names:
            params[n + '.weight'].mul_(4.0)
            params[n + '.bias'].add_(3.0)
    mine._b200.arena.sync_shadow()


def _is_mobilenet(mine):
    from convnet.pytorch_b200.engine import MobileNetRuntime
    return isinstance(mine._b200, MobileNetRuntime)


def _step_args(name, x):
    """train_step keyword arguments of the configuration, and the (t2 permutation, lam) of a mixed step"""
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import MIX_MIXUP, MIX_CUTMIX
    c = CONFIGS[name]
    kw, soft = {}, None
    if 'smooth' in c:
        kw['smooth_eps'] = c['smooth']
    if 'upstream' in c:
        kw['upstream'] = torch.tensor(c['upstream'], device='cuda', dtype=torch.float32)
    if 'mix' in c:
        kind, arg = c['mix']
        N, _, H, W = x.shape
        perm = torch.randperm(N, generator=torch.Generator().manual_seed(11))
        blk = torch.zeros(5, dtype=torch.int32)
        if kind == 'mixup':
            lam = float(np.float32(arg))
        else:
            r0, r1, c0, c1 = arg
            lam = float(np.float32(1.0 - (r1 - r0) * (c1 - c0) / float(H * W)))
            blk[1:] = torch.tensor(arg, dtype=torch.int32)
        blk[:1].view(torch.float32)[0] = lam
        kw['mix'] = ops.Mix(perm.cuda(), blk.cuda(), MIX_MIXUP if kind == 'mixup' else MIX_CUTMIX)
        soft = (perm, lam)
    return kw, soft


def _prefixes(model):
    """[(block prefix, stride)] in the order of the runtime's blocks; MobileNet: the prefix of each block's first
    convolution (stride None: oracle.ref_model.mobilenet_blocks knows it)"""
    if _is_mobilenet(model):
        return [(spec['units'][0][0].slot.name.rsplit('.', 2)[0], None) for spec in model._b200.blocks]
    out = []
    for li, lname in enumerate(('layer1', 'layer2', 'layer3', 'layer4')):
        layer = getattr(model, lname, None)
        if layer is None or isinstance(layer, torch.nn.Identity):
            continue
        for bi in range(len(layer)):
            out.append(('%s.%d' % (lname, bi), 2 if (bi == 0 and li > 0) else 1))
    return out


# ---------------------------------------------------------------------------------------------------- recording
_WRAPPED = ('_stem_fwd', '_stem_bwd', '_block_fwd', '_block_bwd', '_head_fwd', '_head_bwd', '_bn_bwd', '_conv_bwd')


class _Tap(object):
    """wraps the stem / block / head methods of one runtime instance and clones what passes through them; inside the
    blocks also every unit's BatchNorm backward (dy in, dz and g out) and convolution backward (dz and the residual in,
    dx out), in call order.  Methods already replaced on the instance (the mutants) are wrapped and restored as found."""

    def __init__(self, rt):
        self.rt = rt
        self.stem, self.head, self.units = {}, {}, []
        self.blocks = [dict() for _ in rt.blocks]
        self.index = {id(spec): i for i, spec in enumerate(rt.blocks)}

    def __enter__(self):
        rt, orig = self.rt, {n: getattr(self.rt, n) for n in _WRAPPED}

        def stem_fwd(x, training, mix=None, aug=None):
            out, st = orig['_stem_fwd'](x, training, mix, aug)
            self.stem.update(xs=st['unit'].x.clone(), y=out.clone())
            return out, st

        def stem_bwd(st, dy):
            self.stem['dy'] = dy.clone()
            return orig['_stem_bwd'](st, dy)

        def block_fwd(spec, x, training):
            y, saved = orig['_block_fwd'](spec, x, training)
            self.blocks[self.index[id(spec)]].update(x=x.clone(), y=y.clone())
            return y, saved

        def block_bwd(spec, saved, dy):
            r = self.blocks[self.index[id(spec)]]
            r['dy'] = dy.clone()
            dx = orig['_block_bwd'](spec, saved, dy)
            r['dx'] = dx.clone()
            return dx

        def head_fwd(h, training, want_tape):
            out, tape = orig['_head_fwd'](h, training, want_tape)
            self.head.update(h=h.clone(), logits=out.clone())
            if tape is not None:            # the dropout mask (None without dropout) and the masked features
                self.head.update(mask=None if tape['mask'] is None else tape['mask'].clone(), feat=tape['feat'].clone())
            return out, tape

        def head_bwd(tape, dlogits, dl_bf16=None):
            self.head['dl'] = dl_bf16.clone()
            dh = orig['_head_bwd'](tape, dlogits, dl_bf16)
            self.head['dh'] = dh.clone()
            return dh

        def bn_bwd(u, dy, y_mask, act, want_g=False):
            dz, g = orig['_bn_bwd'](u, dy, y_mask, act, want_g)
            self.units.append(dict(kind='bn', u=u, dy=dy.clone(), join=y_mask is not None, act=act, dz=dz.clone(),
                                   g=None if g is None else g.clone()))
            return dz, g

        def conv_bwd(u, dz, need_dx=True, residual=None):
            dx = orig['_conv_bwd'](u, dz, need_dx, residual)
            self.units.append(dict(kind='conv', u=u, dz=dz.clone(), res=None if residual is None else residual.clone(),
                                   dx=None if dx is None else dx.clone()))
            return dx

        self.found = {n: vars(rt).get(n) for n in _WRAPPED}
        for n, fn in zip(_WRAPPED, (stem_fwd, stem_bwd, block_fwd, block_bwd, head_fwd, head_bwd, bn_bwd, conv_bwd)):
            setattr(rt, n, fn)
        return self

    def __exit__(self, *exc):
        for n, fn in self.found.items():
            if fn is None:
                delattr(self.rt, n)
            else:
                setattr(self.rt, n, fn)


def _record(mine, x, y, kw):
    rt = mine._b200
    mine.train()
    rt.arena.zero_grad_force()
    sd = {k: v.detach().clone() for k, v in mine.state_dict().items()}     # parameters and pre-step running buffers
    with _Tap(rt) as tap:
        _, stats = rt.train_step(x, y, **kw)
    torch.cuda.synchronize()
    tap.stats = stats.clone()
    tap.grads = {n: p.grad.detach().clone() for n, p in mine.named_parameters()}
    tap.bufs = {n: b.detach().clone() for n, b in mine.named_buffers()}
    tap.key = int(rt.dropout_key.item()) if rt.dropout_key is not None else None
    tap.sd = sd
    return tap


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


def _decode_stem(xs, cin, imagenet):
    """the relayout output the stem convolution reads -> NCHW: plain padded NHWC (3x3 stem), or the 2x2 space-to-depth
    layout with its zero border (+2 low, +1 high): channel (2 bh + bw) * cin + c of bordered cell (i, j) holds input
    pixel (2 (i - 2) + bh, 2 (j - 2) + bw) -- the tap mapping of test_gpu_conv_sweep._stem_taps, inverted"""
    if not imagenet:
        assert float(xs[..., cin:].abs().max()) == 0.0, 'padding channels of the stem input are not zero'
        return _nchw(xs[..., :cin])
    N, Hb, Wb, _ = xs.shape
    Hs, Ws = Hb - 3, Wb - 3
    inner = torch.zeros_like(xs, dtype=torch.bool)
    inner[:, 2:2 + Hs, 2:2 + Ws, :4 * cin] = True
    assert float(xs.masked_fill(inner, 0).abs().max()) == 0.0, 'border or padding of the s2d stem input is not zero'
    d = xs[:, 2:2 + Hs, 2:2 + Ws, :4 * cin].double().reshape(N, Hs, Ws, 2, 2, cin)
    return d.permute(0, 5, 1, 3, 2, 4).reshape(N, cin, 2 * Hs, 2 * Ws)


# ---------------------------------------------------------------------------------------------------- replay
def _is_l1(mine):
    from convnet.pytorch_b200.models.modules.lp_norm import L1BatchNorm2d
    return any(isinstance(m, L1BatchNorm2d) for m in mine.modules())


def _block_fn(mine, prefix, masks, training=True):
    """the block function of oracle.ref_model.resnet_block_vjp for this block (None: the default)"""
    if _is_l1(mine):
        return l1_oracle._bottleneck if hasattr(mine.layer1[0], 'conv3') else l1_oracle._basic
    if masks is not None and prefix in masks:
        mask, rate = masks[prefix]
        return lambda x, sd, p, s, tr, bufs, q: dropout_oracle._basic(x, sd, p, s, tr, bufs, q, mask, rate)
    return None


def _dropout_masks(mine, key, x):
    spec = dropout_oracle.block_spec(mine, x.shape[0], *x.shape[2:])
    if not spec:
        return None
    masks = dropout_oracle.network_masks(key, spec, x.shape[0])
    return {p: (masks[p].cuda(), rate) for p, _, _, _, _, rate in spec}


def _errors(where, ref, grads, bufs, l1, prefix_cls=''):
    """{quantity: (class, rel-L2)} of parameter gradients and running buffers against the reference of one block / the
    stem; BN affine pairs on one scale"""
    out = {}
    for k, g in ref['grads'].items():
        if 'residual_block' in k or _conv_bias(k, ref['grads']):
            continue
        q = k[len(where) + 1:] if k.startswith(where + '.') else k
        if k.endswith('.weight') and g.dim() == 4:
            out[q] = (prefix_cls + 'dW', _rel(grads[k], g))
        else:
            base = k.rsplit('.', 1)[0]
            scale = max(float(ref['grads'][base + '.weight'].norm()), float(ref['grads'][base + '.bias'].norm()))
            out[q] = (prefix_cls + 'affine', float((grads[k].double() - g).norm()) / scale)
    for k, v in ref['bufs'].items():
        q = k[len(where) + 1:] if k.startswith(where + '.') else k
        if k.endswith('running_mean'):
            rv = ref['bufs'][k.replace('running_mean', 'running_var')]
            scale = float((1.0 / rv).norm() if l1 else rv.clamp(min=0).sqrt().norm())
            out[q] = ('running_mean', float((bufs[k].double() - v).norm()) / scale)
        elif k.endswith('running_var'):
            out[q] = ('running_var', _rel(bufs[k], v))
    return out


def _conv_bias(k, grads):
    """a convolution bias (MobileNet-v1's depthwise layers, in front of a training-mode BatchNorm)"""
    return k.endswith('.bias') and grads[k[:-len('bias')] + 'weight'].dim() == 4


def _check_block(name, where, r, tap, failures, l1, prefix_cls=''):
    for k, g in r['grads'].items():
        if _conv_bias(k, r['grads']):
            # its true gradient is sum(dz) = 0 exactly: the engine writes zeros, the reference sums rounding noise
            assert float(tap.grads[k].abs().max()) == 0.0, '%s %s: the gradient of %s is not zero' % (name, where, k)
            _note('bias noise', float(g.norm()) / float(r['grads'][k[:-len('bias')] + 'weight'].norm()), name, where,
                  failures, k[len(where) + 1:])
            continue
        assert float(g.norm()) > 0, '%s %s: the reference gradient of %s is zero (vacuous state)' % (name, where, k)
        assert float(tap.grads[k].norm()) > 0, '%s %s: the gradient of %s is zero' % (name, where, k)
    for k, v in r['bufs'].items():
        if k.endswith('num_batches_tracked'):
            assert int(tap.bufs[k]) == int(tap.sd[k]) + 1 == int(v), '%s %s: num_batches_tracked %s' % (name, where, k)
    for q, (cls, v) in sorted(_errors(where, r, tap.grads, tap.bufs, l1, prefix_cls).items()):
        _note(cls, v, name, where, failures, q)


def _replay(name, mine, x, y, tap, soft=None, smooth=0.0, upstream=1.0):
    """-> failures [(where, quantity, value, bound)]; the exact chaining checks assert directly"""
    from oracle import ref_model
    rt = mine._b200
    sd, failures, l1, mobile = tap.sd, [], _is_l1(mine), _is_mobilenet(mine)
    blocks = tap.blocks
    prefixes = _prefixes(mine)
    assert len(prefixes) == len(rt.blocks) == len(blocks)
    if mobile:
        assert [p for p, _ in prefixes] == [p for p, _, _ in ref_model.mobilenet_blocks(sd)]
        for (_, units, add_res), spec in zip(ref_model.mobilenet_blocks(sd), rt.blocks):
            assert [c for c, _, _, _, _ in units] == [c.slot.name[:-len('.weight')] for c, _, _ in spec['units']]
            assert add_res == spec['add_res']
    else:
        for (p, _), spec in zip(prefixes, rt.blocks):
            assert spec['convs'][0].slot.name == p + '.conv1.weight'
    # ---- exact chaining of the recorded tensors
    chain = [('stem', tap.stem['y'], tap.stem['dy'])] + [(p, b['y'], b['dy']) for (p, _), b in zip(prefixes, blocks)]
    for (p, yo, dyo), b in zip(chain, blocks + [dict(x=tap.head['h'], dx=tap.head['dh'])]):
        assert torch.equal(yo, b['x']), '%s: the recorded output is not the next input bit for bit' % p
        assert torch.equal(dyo, b['dx']), '%s: the recorded dy is not the dx of the next block bit for bit' % p
    # ---- head
    target = y
    t2 = (target[soft[0].cuda()], soft[1]) if soft is not None else None
    fc = 'classifier.1' if 'classifier.1.weight' in sd else 'fc'
    drop = _head_mask(name, rt, tap) if tap.head['mask'] is not None else None
    h = ref_model.resnet_head_vjp(sd, _nchw(tap.head['h']), target, smooth_eps=smooth, soft=t2, upstream=upstream,
                                  fc=fc, drop=drop)
    C = rt.classes
    _note('logits', _rel(tap.head['logits'], h['logits']), name, 'head', failures)
    _note('loss', abs(float(tap.stats[0]) - float(h['loss'])) / abs(float(h['loss'])), name, 'head', failures)
    assert abs(float(tap.stats[1]) - h['top1']) < 1e-3 and abs(float(tap.stats[2]) - h['top5']) < 1e-3, \
        '%s head: top-1 / top-5 %s vs %.4f / %.4f' % (name, tap.stats.tolist(), h['top1'], h['top5'])
    assert float(tap.head['dl'][:, C:].abs().max() if tap.head['dl'].shape[1] > C else 0.0) == 0.0
    _note('dlogits', _rel(tap.head['dl'][:, :C], h['dlogits']), name, 'head', failures)
    for k in (fc + '.weight', fc + '.bias'):
        assert float(tap.grads[k].norm()) > 0
        _note('fc grad', _rel(tap.grads[k], h['grads'][k]), name, 'head', failures, k)
    _note('dh', _rel(_nchw(tap.head['dh']), h['dh']), name, 'head', failures)
    # ---- blocks
    masks = _dropout_masks(mine, tap.key, x) if tap.key is not None else None
    se_ref = {}
    for (p, stride), b in zip(prefixes, blocks):
        xb, dyb = _nchw(b['x']), _nchw(b['dy'])
        if mobile:
            r = ref_model.mobilenet_block_vjp(sd, p, xb, dyb)
        else:
            r = ref_model.resnet_block_vjp(sd, p, xb, dyb, stride, block=_block_fn(mine, p, masks))
        _note('y', _rel(_nchw(b['y']), r['y']), name, p, failures)
        _note('dx', _rel(_nchw(b['dx']), r['dx']), name, p, failures)
        _check_block(name, p, r, tap, failures, l1)
        for k, g in r['grads'].items():
            if 'residual_block' in k:
                se_ref[k] = se_ref[k] + g if k in se_ref else g
    for k, g in sorted(se_ref.items()):        # one shared gate per stage: the sum of its blocks' VJPs
        assert float(g.norm()) > 0 and float(tap.grads[k].norm()) > 0, k
        _note('SE grad', _rel(tap.grads[k], g), name, k.split('.')[0], failures, k)
    # ---- stem, past the input relayout
    stem_bn = (lambda t, sd_, pfx, tr, bufs: l1_oracle.bn_l1(t, sd_, pfx, tr, bufs)) if l1 else None
    xs = _decode_stem(tap.stem['xs'], 3, rt.imagenet_stem)
    stem = {}
    if mobile:                  # 3x3/s2 conv, BN, ReLU6 (v2) / ReLU (v1), no max-pool
        conv, norm, stride, pad, act = ref_model.mobilenet_stem(sd)
        stem = dict(conv=conv, norm=norm, stride=stride, padding=pad, act='relu' if act == 'relu' else 'relu6')
    s = ref_model.resnet_stem_vjp(sd, xs, _nchw(tap.stem['dy']), bn=stem_bn, **stem)
    _note('stem y', _rel(_nchw(tap.stem['y']), s['y']), name, 'stem', failures)
    _check_block(name, 'stem', s, tap, failures, l1, prefix_cls='stem ')
    return failures


def _head_mask(name, rt, tap):
    """the head's dropout mask from the tape: exactly the two values {0, 1 / (1 - p)} (fp32), a kept fraction within
    5 sigma of 1 - p, and the kept features are the pooled bf16 mean times 1 / (1 - p) with ONE rounding to bf16 (at
    p = 0.1 and 0.2 the fp32 product rounds like the fp64 one: a bf16 value times 10 / 9 or 5 / 4 lies at least 1/18
    ulp from a rounding midpoint) -> the (0/1 keep mask, p) of oracle.ref_model.resnet_head_vjp"""
    from convnet.pytorch_b200 import ops
    p, mask, feat = rt.dropout_p, tap.head['mask'], tap.head['feat']
    N, C = feat.shape[0], feat.shape[-1]
    mask, feat = mask.reshape(N, C), feat.reshape(N, C)
    scale = float(np.float32(1.0 / (1.0 - p)))
    values = sorted(torch.unique(mask).tolist())
    assert mask.dtype == torch.float32 and values == [0.0, scale], \
        '%s head: dropout mask %s with values %s, not {0, %r}' % (name, mask.dtype, values[:4], scale)
    keep = mask != 0
    frac, sigma = float(keep.double().mean()), (p * (1.0 - p) / keep.numel()) ** 0.5
    print('%s head dropout p = %g: kept fraction %.4f (1 - p %.4f, sigma %.1e)' % (name, p, frac, 1.0 - p, sigma))
    assert abs(frac - (1.0 - p)) < 5 * sigma, '%s head: kept fraction %.4f for p = %g' % (name, frac, p)
    pooled = ops.avgpool_fwd(tap.head['h']).reshape(N, C)
    want = (pooled.double() * (1.0 / (1.0 - p))).to(torch.bfloat16)
    assert torch.equal(feat[keep], want[keep]), '%s head: %d of the kept features are not bf16(mean / (1 - p))' % (
        name, int((feat[keep] != want[keep]).sum()))
    assert float(feat[~keep].abs().max()) == 0.0, '%s head: a dropped feature is not zero' % name
    return keep.double(), p


def _unit_names(rt, mine):
    """id of each _BN / _Conv of the runtime -> (block prefix or 'stem', module name inside it), from the module names"""
    mods = {id(m): n for n, m in mine.named_modules()}
    bns, convs = {id(rt.stem_bn): ('stem', mods[id(rt.stem_bn.mod)])}, {}
    for (p, _), spec in zip(_prefixes(mine), rt.blocks):
        if 'units' in spec:
            pairs = [(c, b) for c, b, _ in spec['units']]
        else:
            pairs = list(zip(spec['convs'], spec['bns'])) + ([tuple(spec['down'])] if spec['down'] is not None else [])
        for c, b in pairs:
            convs[id(c)] = (p, c.slot.name[len(p) + 1:-len('.weight')])
            bns[id(b)] = (p, mods[id(b.mod)][len(p) + 1:])
    return bns, convs


def _replay_units(name, mine, tap, masks, failures):
    """Unit-level teacher forcing inside the blocks: every BatchNorm backward against fp64 autograd of the BN (+ ReLU,
    + dropout) on the engine's own z and dy -- dz, g = dy * act', d gamma / d beta -- and the running statistics against
    fp64 statistics of the same z; every convolution backward against fp64 dgrad / wgrad on the engine's own x and dz.
    One rounding separates the two sides, however ill-conditioned the whole block is."""
    from convnet.pytorch_b200.lib import ACT_NONE, ACT_RELU6
    from oracle import ref_model
    rt, sd, l1 = mine._b200, tap.sd, _is_l1(mine)
    bn_names, conv_names = _unit_names(rt, mine)
    assert sum(1 for r in tap.units if r['kind'] == 'bn') == len(bn_names), 'one BatchNorm backward per BN layer'
    assert sum(1 for r in tap.units if r['kind'] == 'conv') == len(conv_names), 'one backward per block convolution'
    for rec in tap.units:
        u = rec['u']
        if rec['kind'] == 'conv':
            c = u.conv
            where, local = conv_names[id(c)]
            w = sd['%s.%s.weight' % (where, local)].double()
            x, dz = _nchw(u.x), _nchw(rec['dz'])
            kw = dict(stride=c.stride, padding=c.pad, groups=c.C if c.kind == 'dw' else c.groups)
            if rec['dx'] is not None:
                dx = torch.nn.grad.conv2d_input(x.shape, w, dz, **kw)
                if rec['res'] is not None:
                    dx = dx + _nchw(rec['res'])
                _note('unit dgrad', _rel(_nchw(rec['dx']), dx), name, where, failures, local + ' dgrad')
            dw = torch.nn.grad.conv2d_weight(x, w.shape, dz, **kw)
            _note('unit wgrad', _rel(tap.grads['%s.%s.weight' % (where, local)], dw), name, where, failures,
                  local + '.weight')
            continue
        where, local = bn_names[id(u.bn)]
        full = local if where == 'stem' else where + '.' + local
        loc = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items() if k.startswith(full + '.')}
        for k in (full + '.weight', full + '.bias'):
            loc[k] = loc[k].detach().clone().requires_grad_(True)
        z = _nchw(u.z).requires_grad_(True)
        bufs = {}
        out = l1_oracle.bn_l1(z, loc, full, True, bufs) if l1 else ref_model._bn(z, loc, full, True, bufs, False)
        dy = _nchw(rec['dy'])
        if rec['act'] == ACT_NONE:
            gout = dy
        elif rec['join']:                 # the pre-activation includes the skip: its sign is that of the output
            gout = dy * (_nchw(u.y) > 0)
        else:
            # the ReLU / ReLU6 gate as the kernels decide it, from the forward's fp32 coefficients with ONE rounding,
            # fmaf(z, scale, shift) (z * scale is exact in fp64): where bn(z) sits within fp32 rounding of 0 or 6 the
            # fp64 decision differs, and a flipped gate moves d beta by a whole dy element.  Two fp32 roundings are
            # not enough either: a depthwise convolution repeats one z value over every all-zero window, and a
            # MobileNet-v2 step has shown 20 copies of a pre-activation of 1.6e-9 whose sign the unfused sum flips
            pre = (u.z.double() * u.scale.double() + u.shift.double()).float()
            gate = (pre > 0) & (pre < 6) if rec['act'] == ACT_RELU6 else pre > 0
            gate = gate.permute(0, 3, 1, 2).double()
            if where != 'stem' and local == 'bn1' and masks is not None and where in masks:
                keep, rate = masks[where]
                gate = gate * keep.double() * dropout_oracle.threshold(rate)[1]
            gout = dy * gate
        dz, dg, db = torch.autograd.grad(out, [z, loc[full + '.weight'], loc[full + '.bias']], gout)
        bias = sd.get(u.conv.slot.name[:-len('weight')] + 'bias') if u.conv is not None else None
        if bias is not None:
            # a convolution bias in front of the BN: z holds the convolution without it; the true pre-BN tensor is
            # z + b, which moves only the running mean
            bufs[full + '.running_mean'] = bufs[full + '.running_mean'] + 0.1 * bias.double()
        with torch.no_grad():           # the forward's coefficients: y = z * scale + shift
            zd = z.detach()
            mean = zd.mean((0, 2, 3))
            if l1:
                inv = 1.0 / ((zd - mean[None, :, None, None]).abs().mean((0, 2, 3)) * l1_oracle.L1_FIX + 1e-5)
            else:
                inv = torch.rsqrt(zd.var((0, 2, 3), unbiased=False) + 1e-5)
            sc = loc[full + '.weight'].detach() * inv
            coef = torch.cat([sc, loc[full + '.bias'].detach() - mean * sc])
        _note('unit coeffs', _rel(torch.cat([u.scale, u.shift]), coef), name, where, failures, local + ' scale/shift')
        _note('unit dz', _rel(_nchw(rec['dz']), dz), name, where, failures, local + ' dz')
        if rec['g'] is not None:
            _note('unit g', _rel(_nchw(rec['g']), gout), name, where, failures, local + ' g')
        scale = max(float(dg.norm()), float(db.norm()))
        for k, ref in ((full + '.weight', dg), (full + '.bias', db)):
            _note('unit affine', float((tap.grads[k].double() - ref).norm()) / scale, name, where, failures,
                  k[len(full) - len(local):])
        for k, v in bufs.items():
            if k.endswith('running_mean'):
                rv = bufs[k.replace('running_mean', 'running_var')]
                s = float((1.0 / rv).norm() if l1 else rv.clamp(min=0).sqrt().norm())
                _note('unit running_mean', float((tap.bufs[k].double() - v).norm()) / s, name, where, failures,
                      k[len(full) - len(local):])
            elif k.endswith('running_var'):
                _note('unit running_var', _rel(tap.bufs[k], v), name, where, failures, k[len(full) - len(local):])


def _run(name, mine, x, y):
    kw, soft = _step_args(name, x)
    c = CONFIGS[name]
    tap = _record(mine, x, y, kw)
    failures = _replay(name, mine, x, y, tap, soft=soft, smooth=c.get('smooth', 0.0), upstream=c.get('upstream', 1.0))
    masks = _dropout_masks(mine, tap.key, x) if tap.key is not None else None
    _replay_units(name, mine, tap, masks, failures)
    if 'clip' in c:
        _check_clipping(name, mine, tap, c['clip'])
    return failures


def _check_clipping(name, mine, tap, bns):
    """the raised BatchNorms of the configuration clip: at least 1 % of their pre-activations lie above 6"""
    bn_names = _unit_names(mine._b200, mine)[0]
    seen = {}
    for rec in tap.units:
        if rec['kind'] == 'bn':
            where, local = bn_names[id(rec['u'].bn)]
            full = local if where == 'stem' else where + '.' + local
            if full in bns:
                u = rec['u']
                seen[full] = float(((u.z.float() * u.scale + u.shift) > 6).double().mean())
    print('%s: fraction of pre-activations above 6: %s' % (name, ', '.join('%s %.3f' % kv for kv in sorted(seen.items()))))
    assert sorted(seen) == sorted(bns)
    assert min(seen.values()) >= 0.01, '%s: a raised BatchNorm does not clip: %s' % (name, seen)


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize('name', list(CONFIGS))
def test_block_replay(name):
    """one training step of the configuration, block by block against fp64"""
    _setup()
    t0 = time.time()
    ref, mine, x, y = _build(name)
    failures = _run(name, mine, x, y)
    print('\nblock replay %s: %.1f s' % (name, time.time() - t0))
    _report('after %s' % name)
    assert not failures, '%s: %s' % (name, ['%s %s %.3e > %.0e' % f for f in failures])


@pytest.mark.parametrize('name', ['resnet20', 'resnext_se50', 'mobilenet_v2_relu6', 'mobilenet_v1'])
def test_gradients_accumulate(name):
    """two train_steps on one batch without zero_grad: every arena gradient is twice the one-step gradient (the
    accumulate contract of include/b200conv.h that chunked batches rely on: the stem's space-to-depth gather, the
    grouped unpack, the SE and fc column sums, BN d gamma / d beta, the depthwise weight gradients through their shared
    workspace on the side stream), and the running buffers saw two momentum updates.  A path that overwrites instead of
    accumulating shows an error of 0.5.  MobileNet-v1's depthwise biases stay exactly zero.  (The MobileNet-v2
    configuration has no head dropout: two steps would draw two masks.)"""
    _setup()
    ref, mine, x, y = _build(name)
    rt = mine._b200
    mine.train()
    rt.arena.zero_grad_force()
    b0 = {n: b.clone() for n, b in mine.named_buffers()}
    rt.train_step(x, y)
    torch.cuda.synchronize()
    g1 = {n: p.grad.clone() for n, p in mine.named_parameters()}
    b1 = {n: b.clone() for n, b in mine.named_buffers()}
    rt.train_step(x, y)
    torch.cuda.synchronize()
    worst = (0.0, '')
    for n, p in mine.named_parameters():
        if _conv_bias(n, g1):
            assert float(g1[n].abs().max()) == 0.0 and float(p.grad.abs().max()) == 0.0, n
            continue
        assert float(g1[n].norm()) > 0, n
        worst = max(worst, (_rel(p.grad, 2 * g1[n]), n))
    bworst = (0.0, '')
    for n, b in mine.named_buffers():
        if n.endswith('num_batches_tracked'):
            assert int(b) == int(b0[n]) + 2, n
            continue
        want = 1.9 * b1[n].double() - 0.9 * b0[n].double()      # r2 = 0.9 r1 + 0.1 s with s = (r1 - 0.9 r0) / 0.1
        scale = b1[n.replace('running_mean', 'running_var')].double().sqrt().norm() if 'mean' in n else want.norm()
        bworst = max(bworst, (float((b.double() - want).norm() / scale), n))
    print('\naccumulation %s: worst gradient rel-L2 %.3e (%s), running buffers %.3e (%s)' % ((name,) + worst + bworst))
    assert worst[0] <= 1e-6, worst
    assert bworst[0] <= 1e-6, bworst


@pytest.mark.parametrize('name', ['resnet18', 'resnext20', 'resnet_se50', 'resnet20_l1', 'mobilenet_v2',
                                  'mobilenet_v1'])
def test_eval_blocks(name):
    """eval-mode forwards, BatchNorm folded into the convolutions and not folded: every block against the fp64 block in
    eval mode on the running statistics.  The folded weights carry one more bf16 rounding, of w * gamma / sigma.  The
    MobileNet runtimes never fold (fold_bn_eval = False): both settings must give the same logits bit for bit, and
    MobileNet-v1's depthwise bias enters the BatchNorm shift."""
    from oracle import ref_model
    from convnet.pytorch_b200 import engine
    _setup()
    ref, mine, x, y = _build(name)
    rt = mine._b200
    sd = {k: v.detach().clone() for k, v in mine.state_dict().items()}
    prefixes = _prefixes(mine)
    mine.eval()
    failures, logits = [], []
    saved = engine.FOLD_BN_EVAL
    try:
        for fold in (False, True):
            engine.FOLD_BN_EVAL = fold
            with _Tap(rt) as tap, torch.no_grad():
                logits.append(mine(x))
            torch.cuda.synchronize()
            folded = fold and rt.fold_bn_eval
            for (p, stride), b in zip(prefixes, tap.blocks):
                if _is_mobilenet(mine):
                    r = ref_model.mobilenet_block_vjp(sd, p, _nchw(b['x']), None, training=False)
                else:
                    r = ref_model.resnet_block_vjp(sd, p, _nchw(b['x']), None, stride, block=_block_fn(mine, p, None),
                                                   training=False)
                _note('eval y folded' if folded else 'eval y', _rel(_nchw(b['y']), r['y']), name, p, failures)
    finally:
        engine.FOLD_BN_EVAL = saved
    if not rt.fold_bn_eval:
        assert torch.equal(logits[0], logits[1]), '%s: FOLD_BN_EVAL changed the eval forward of a non-folding runtime' % name
    _report('after eval %s' % name)
    assert not failures, '%s: %s' % (name, ['%s %s %.3e > %.0e' % f for f in failures])


# ---------------------------------------------------------------------------------------------------- mutants
def _spec(rt, mine, prefix):
    return rt.blocks[[p for p, _ in _prefixes(mine)].index(prefix)]


def _wrap_bn_bwd(monkeypatch, rt, fn):
    orig = rt._bn_bwd
    monkeypatch.setattr(rt, '_bn_bwd', lambda u, dy, y_mask, act, want_g=False: fn(orig, u, dy, y_mask, act, want_g),
                        raising=False)


def _mutant_skip_dy(monkeypatch, rt, mine):
    """identity block layer1.1: the skip gradient is dy instead of g = dy * (out > 0)"""
    last = _spec(rt, mine, 'layer1.1')['bns'][-1]

    def fn(orig, u, dy, y_mask, act, want_g):
        dz, g = orig(u, dy, y_mask, act, want_g)
        return (dz, dy) if (want_g and u.bn is last) else (dz, g)
    _wrap_bn_bwd(monkeypatch, rt, fn)
    return 'layer1.1', lambda q: q in ('dx', 'bn2 g')


def _mutant_down_dy(monkeypatch, rt, mine):
    """layer2.0: the downsample BN's backward receives dy instead of g"""
    spec = _spec(rt, mine, 'layer2.0')
    last, down, seen = spec['bns'][-1], spec['down'][1], {}

    def fn(orig, u, dy, y_mask, act, want_g):
        if want_g and u.bn is last:
            seen['dy'] = dy
        if u.bn is down:
            dy = seen['dy']
        return orig(u, dy, y_mask, act, want_g)
    _wrap_bn_bwd(monkeypatch, rt, fn)
    return 'layer2.0', lambda q: q.startswith('downsample')


def _mutant_dgamma(monkeypatch, rt, mine):
    """mid-network bottleneck layer2.2.bn2: the d gamma increment scaled by 1 + 2^-6"""
    bn = _spec(rt, mine, 'layer2.2')['bns'][1]

    def fn(orig, u, dy, y_mask, act, want_g):
        if u.bn is not bn:
            return orig(u, dy, y_mask, act, want_g)
        before = bn.dgamma.clone()
        out = orig(u, dy, y_mask, act, want_g)
        bn.dgamma.copy_(before + (bn.dgamma - before) * (1 + 2 ** -6))
        return out
    _wrap_bn_bwd(monkeypatch, rt, fn)
    return 'layer2.2', lambda q: q == 'bn2.weight'


def _mutant_momentum(monkeypatch, rt, mine):
    """layer2.1.bn1 updates its running statistics with momentum 0.1 * (1 + 2^-7)"""
    monkeypatch.setattr(_spec(rt, mine, 'layer2.1')['bns'][0].mod, 'momentum', 0.1 * (1 + 2 ** -7))
    return 'layer2.1', lambda q: q.startswith('bn1.running')


def _mutant_se_scratch(monkeypatch, rt, mine):
    """layer3.1 writes its gate gradients to scratch instead of accumulating them into the stage's shared gate"""
    se = _spec(rt, mine, 'layer3.1')['se']
    for lin in (se.l1, se.l2):
        for a in ('gw', 'gb'):
            monkeypatch.setattr(lin, a, torch.zeros_like(getattr(lin, a)))
    return 'layer3', lambda q: 'residual_block' in q


def _mutant_drop_layer(monkeypatch, rt, mine):
    """layer2.0 draws its dropout mask with layer index n + 1"""
    spec = _spec(rt, mine, 'layer2.0')
    monkeypatch.setitem(spec, 'drop', (spec['drop'][0] + 1, spec['drop'][1]))
    return 'layer2.0', lambda q: q in ('bn1 dz', 'conv1.weight', 'conv2.weight', 'bn1.weight')


def _mutant_sign_sum(monkeypatch, rt, mine):
    """the L1 unit of layer2.1.bn1 has its sign_sum zeroed before its backward"""
    bn = _spec(rt, mine, 'layer2.1')['bns'][0]

    def fn(orig, u, dy, y_mask, act, want_g):
        if u.bn is bn:
            print('sign_sum of layer2.1.bn1: |sum| / M mean %.3e' % float(u.sign_sum.abs().mean() / (u.z.numel() // u.z.shape[-1])))
            u.sign_sum.zero_()
        return orig(u, dy, y_mask, act, want_g)
    _wrap_bn_bwd(monkeypatch, rt, fn)
    return 'layer2.1', lambda q: q in ('bn1 dz', 'dx', 'conv1.weight')


def _mutant_upstream_bias(monkeypatch, rt, mine):
    """the fc bias gradient is the column sum of an unscaled copy of the bf16 dlogits (upstream 8 dropped)"""
    from convnet.pytorch_b200 import ops
    orig = ops.colsum_bf16

    def colsum(m, out):
        if out.data_ptr() == rt.fc.gb.data_ptr():
            m = (m.float() / 8.0).to(torch.bfloat16)
        return orig(m, out)
    monkeypatch.setattr(ops, 'colsum_bf16', colsum)
    return 'head', lambda q: q == 'fc.bias'


def _mutant_mb_skip(monkeypatch, rt, mine):
    """MobileNet-v2 identity block bottleneck2: its first unit's dgrad gets no residual (the skip gradient is dropped)"""
    first = _spec(rt, mine, 'features.bottleneck2.block')['units'][0][0]
    orig = rt._conv_bwd

    def conv_bwd(u, dz, need_dx=True, residual=None):
        return orig(u, dz, need_dx, None if u.conv is first else residual)
    monkeypatch.setattr(rt, '_conv_bwd', conv_bwd, raising=False)
    return 'features.bottleneck2.block', lambda q: q == 'dx'


def _mutant_relu6_as_relu(monkeypatch, rt, mine):
    """the clipping depthwise BN of bottleneck2 (mobilenet_v2_relu6) runs its backward with ReLU's gate"""
    from convnet.pytorch_b200.lib import ACT_RELU
    bn = _spec(rt, mine, 'features.bottleneck2.block')['units'][1][1]

    def fn(orig, u, dy, y_mask, act, want_g):
        return orig(u, dy, y_mask, ACT_RELU if u.bn is bn else act, want_g)
    _wrap_bn_bwd(monkeypatch, rt, fn)
    return 'features.bottleneck2.block', lambda q: q == '4 dz'


def _mutant_dw_bias_mean(monkeypatch, rt, mine):
    """MobileNet-v1 features.5: the depthwise convolution's bias is left out of its BN's running-mean update"""
    monkeypatch.setattr(_spec(rt, mine, 'features.5.components')['units'][0][0], 'bias32', None)
    return 'features.5.components', lambda q: q == '1.running_mean'


def _mutant_head_mask_bwd(monkeypatch, rt, mine):
    """MobileNet-v2: the head's backward does not apply the dropout mask to d feat"""
    orig = rt._head_bwd
    monkeypatch.setattr(rt, '_head_bwd', lambda tape, dlogits, dl_bf16=None: orig(dict(tape, mask=None), dlogits,
                                                                                  dl_bf16), raising=False)
    return 'head', lambda q: q == 'dh'


MUTANTS = {
    'skip_dy': ('resnet20', _mutant_skip_dy),
    'down_dy': ('resnet18', _mutant_down_dy),
    'dgamma': ('resnet50', _mutant_dgamma),
    'momentum': ('resnet20', _mutant_momentum),
    'se_scratch': ('resnet_se50', _mutant_se_scratch),
    'drop_layer': ('wrn16_4_dropout', _mutant_drop_layer),
    'sign_sum': ('resnet20_l1', _mutant_sign_sum),
    'upstream_bias': ('resnet18_upstream8', _mutant_upstream_bias),
    'mb_skip': ('mobilenet_v2_112', _mutant_mb_skip),
    'relu6_as_relu': ('mobilenet_v2_relu6', _mutant_relu6_as_relu),
    'dw_bias_mean': ('mobilenet_v1', _mutant_dw_bias_mean),
    'head_mask_bwd': ('mobilenet_v2_112', _mutant_head_mask_bwd),
}


@pytest.mark.parametrize('mutant', list(MUTANTS))
def test_mutant_is_caught(mutant, monkeypatch):
    """One wiring fault planted in the Python engine code (every launch stays valid): the replay fails, in the block and
    quantity the fault touches and nowhere else; test_block_replay runs the same configuration unmutated.

    The d gamma mutant (1.6 % on one tensor, in a ResNet-50 bottleneck) is caught by the unit-level replay; the
    whole-block bounds of the bottlenecks (LOOSE) are wider than that.  It also runs through
    test_gpu_engine._check_against_bf16_oracle and the outcome is printed: that check did not notice it when this test
    was written (scaling a gradient tensor leaves its cosine to the oracle's at 1, and moves the global gradient by far
    less than the oracle's self-sensitivity)."""
    _setup()
    name, plant = MUTANTS[mutant]
    ref, mine, x, y = _build(name)
    where, quantity = plant(monkeypatch, mine._b200, mine)
    saved = dict(WORST)
    failures = _run(name, mine, x, y)
    WORST.clear()
    WORST.update(saved)                    # the mutant's errors stay out of the worst-value table
    print('\nmutant %s on %s: %s' % (mutant, name, ['%s %s %.3e > %.0e' % f for f in failures]))
    assert failures, 'mutant %s passed the replay' % mutant
    assert all(f[0] == where for f in failures), 'mutant %s failed outside %s: %s' % (mutant, where, failures)
    assert any(quantity(f[1]) for f in failures), 'mutant %s did not fail the expected quantity: %s' % (mutant, failures)
    if mutant == 'dgamma':
        # the network-level check starts from the state before the replayed step: its running buffers
        from test_gpu_engine import _check_against_bf16_oracle
        with torch.no_grad():
            for (_, b), (_, c) in zip(mine.named_buffers(), ref.named_buffers()):
                b.copy_(c)
        try:
            _check_against_bf16_oracle(mine, ref, x, y)
            print('the network-level T2 check did not notice the d gamma mutant')
        except AssertionError as e:
            print('the network-level T2 check noticed the d gamma mutant: %s' % e)
