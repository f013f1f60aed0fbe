"""B200 execution engine: parameter arenas + the fused forward/backward pipeline of the ResNet family.

``convert_b200(model)`` takes a model built by the registry (ordinary ``torch.nn`` layers, reference
attribute names) and
  * moves every parameter into flat device arenas -- fp32 master ``p32``, fp32 gradient ``g32``, bf16
    compute shadow ``p16`` -- conv weights physically [K][R*S][C] (the layout the wgmma kernels read)
    while ``param.shape`` / ``state_dict()`` stay the reference's logical OIHW (SURVEY.md section 5,
    checkpoint row);
  * installs a runtime whose ``forward`` replaces ``model.forward`` (models/resnet.py:196-213 in the
    reference) by the kernel pipeline
        conv (wgmma implicit GEMM) -> BN statistics -> BN apply + ReLU (+ residual) ...
    and whose backward (one autograd node for the whole net) runs BN backward, dgrad and wgrad kernels
    and writes parameter gradients straight into ``g32`` (``param.grad`` are views of it).
Nothing here computes on the CPU or through cuDNN/cuBLAS: a missing library or an unsupported layer
raises ``B200Error``.
"""
import torch
import torch.nn as nn

from . import ops
from .lib import B200Error, ACT_NONE, ACT_RELU, ACT_RELU6

_ALIGN = 64  # elements; keeps every slot 128B-aligned in the bf16 shadow (TMA needs 16B)
FOLD_BN_EVAL = True   # inference: BN folded into conv weights + epilogue bias (tests turn it off to compare)


def _round_up(n, m):
    return (n + m - 1) // m * m


class _Slot(object):
    __slots__ = ('name', 'param', 'kind', 'offset', 'numel', 'alloc', 'shape', 'group', 'module')


class Arena(object):
    """Flat fp32 master / fp32 grad / bf16 shadow storage for all parameters of one model."""

    def __init__(self, model, device):
        self.device = device
        self.convs = []          # every engine._Conv built on this arena (batched dgrad-weight transposes)
        self.version = 0         # bumped whenever parameters or BN running statistics may have changed
        self.grads_zero = False  # True while g32 is known to be all zeros (the fused SGD kernel cleared it in its pass)
        slots = []
        seen = set()
        for mod_name, mod in model.named_modules():
            for p_name, p in mod.named_parameters(recurse=False):
                if id(p) in seen:
                    continue
                seen.add(id(p))
                s = _Slot()
                s.name = (mod_name + '.' if mod_name else '') + p_name
                s.param, s.module, s.shape = p, mod, tuple(p.shape)
                s.numel = p.numel()
                s.alloc = s.numel
                if isinstance(mod, nn.Conv2d) and p_name == 'weight':
                    depthwise = mod.groups > 1 and mod.groups == mod.in_channels and mod.in_channels == mod.out_channels
                    if mod.groups > 1 and not depthwise and (mod.in_channels % mod.groups or mod.out_channels % mod.groups):
                        raise B200Error('grouped convolution %s: channels not divisible by groups' % s.name)
                    s.kind = 'dw' if depthwise else 'conv'   # grouped weights [K, C/g, R, S] use the same KRSC view
                    s.group = 1 if depthwise else 0
                elif isinstance(mod, nn.Linear) and p_name == 'weight':
                    s.kind, s.group = 'fc', 0
                    s.alloc = _round_up(p.shape[0], 8) * p.shape[1]  # zero rows: class count padded to 8
                elif isinstance(mod, nn.Linear) and p_name == 'bias':
                    s.kind, s.group = 'vec', 2
                    s.alloc = _round_up(p.shape[0], 8)
                else:
                    s.kind, s.group = 'vec', 2
                slots.append(s)
        slots.sort(key=lambda s: s.group)  # stable: [dense conv + fc | depthwise | everything else]
        off = 0
        self.group_end = [0, 0, 0]
        for s in slots:
            s.offset = off
            off += _round_up(s.alloc, _ALIGN)
            self.group_end[s.group] = off
        self.group_end[1] = max(self.group_end[1], self.group_end[0])
        self.group_end[2] = off
        self.total = off
        self.slots = slots
        self.by_param = {id(s.param): s for s in slots}
        self.p32 = torch.zeros(off, device=device, dtype=torch.float32)
        self.g32 = torch.zeros(off, device=device, dtype=torch.float32)
        self.p16 = torch.zeros(off, device=device, dtype=torch.bfloat16)
        with torch.no_grad():
            for s in slots:
                src = s.param.detach().to(device=device, dtype=torch.float32)
                view = self.logical_view(self.p32, s)
                view.copy_(src)
                s.param.data = view
                s.param.grad = self.logical_view(self.g32, s)
        self.sync_shadow()

    # logical (reference-shaped) view of a slot inside a flat buffer
    def logical_view(self, flat, s):
        seg = flat[s.offset:s.offset + s.numel]
        if s.kind == 'conv':
            K, C, R, S = s.shape
            return seg.view(K, R, S, C).permute(0, 3, 1, 2)
        if s.kind == 'dw':
            C, _, R, S = s.shape
            return seg.view(R, S, C).permute(2, 0, 1).unsqueeze(1)
        return seg.view(s.shape)

    def kernel_view(self, flat, s):
        """physical layout consumed by the kernels."""
        if s.kind == 'conv':
            K, C, R, S = s.shape
            return flat[s.offset:s.offset + s.numel].view(K, R * S, C)
        if s.kind == 'dw':
            C, _, R, S = s.shape
            return flat[s.offset:s.offset + s.numel].view(R * S, C)
        if s.kind == 'fc':
            K, C = s.shape
            return flat[s.offset:s.offset + s.alloc].view(_round_up(K, 8), 1, C)
        return flat[s.offset:s.offset + s.alloc]

    def slot(self, param):
        return self.by_param[id(param)]

    def sync_shadow(self):
        """bf16 shadow <- fp32 master (whole arena, one kernel)."""
        ops.cast_bf16(self.p32, self.p16)
        self.version += 1

    def zero_grad(self):
        """g32 <- 0.  A no-op when the fused SGD kernel already cleared the arena while consuming the gradients
        (B200SGD.fold_zero_grad) and nothing has been accumulated since."""
        if not self.grads_zero:
            self.g32.zero_()
            self.grads_zero = True

    def zero_grad_force(self):
        self.grads_zero = False
        self.zero_grad()

    def rebind_grads(self):
        for s in self.slots:
            if s.param.grad is None or s.param.grad.data_ptr() != self.g32.data_ptr() + 4 * s.offset:
                s.param.grad = self.logical_view(self.g32, s)


# ----------------------------------------------------------------------------------------------------
class _Conv(object):
    def __init__(self, arena, mod):
        s = arena.slot(mod.weight)
        self.kind = s.kind
        self.K, self.C = mod.out_channels, mod.in_channels
        self.R, self.S = mod.kernel_size
        self.stride = mod.stride[0]
        self.pad = mod.padding[0]
        if mod.stride[0] != mod.stride[1] or mod.padding[0] != mod.padding[1] or mod.dilation != (1, 1):
            raise B200Error('conv %s: only square stride/padding and dilation 1 are supported' % s.name)
        # A bias in front of a BatchNorm (MobileNet-v1's depthwise convolutions, models/mobilenet.py:44-46 of the
        # reference) is absorbed analytically: training-mode BN removes it from the output and makes its gradient
        # exactly zero; it only shifts the running mean and the eval-mode BN shift (see Runtime._bn_coeffs)
        self.bias32 = None
        if mod.bias is not None:
            if s.kind != 'dw':
                raise B200Error('conv %s: bias is only supported on depthwise convolutions followed by BatchNorm' % s.name)
            self.bias32 = arena.kernel_view(arena.p32, arena.slot(mod.bias))
        self.groups = mod.groups if s.kind == 'conv' else 1
        # grouped convolutions (ResNeXt) run block-diagonally: 64-channel windows for fprop / dgrad, 128 for wgrad
        # (b200_conv_desc.window); shapes outside that fall back to the dense block-diagonal expansion (window == C)
        cg = self.C // max(self.groups, 1)
        self.window = 64 if (self.groups > 1 and self.C == self.K and self.C % 128 == 0 and 64 % cg == 0) else 0
        self.slot = s
        self.wt = None           # [C, R*S, K] view of the runtime's transposed shadow (dgrad operand), set by Runtime
        arena.convs.append(self)
        self.w16 = arena.kernel_view(arena.p16, s)
        self.w32 = arena.kernel_view(arena.p32, s)
        self.g32 = arena.kernel_view(arena.g32, s)

    def desc(self, N, H, W, wgrad=False):
        return ops.make_desc(N, H, W, self.C, self.K, self.R, self.S, self.stride, self.pad,
                             algo_macs=self.K * self.R * self.S * self.C // self.groups,
                             window=(128 if wgrad else 64) if self.window else 0)

    def kernel_weights(self, w32=None):
        """bf16 operand of the convolution kernels: the arena shadow [K, R*S, C], or for a grouped convolution the
        block-diagonal packing of the fp32 master at window granularity ([K, R*S, 64]; dense [K, R*S, C] fallback)."""
        if self.groups == 1:
            return self.w16
        return ops.group_weight_pack(self.w32 if w32 is None else w32, self.K, self.R * self.S, self.C, self.groups,
                                     self.window or self.C)

    def dgrad_weights(self):
        """grouped convolutions: [C, R*S, 64] operand of dgrad (dense [C, R*S, K] fallback), packed from the fp32
        master."""
        return ops.group_weight_pack(self.w32, self.K, self.R * self.S, self.C, self.groups, self.window or self.C,
                                     transpose=True)


class _BN(object):
    """one BatchNorm layer: nn.BatchNorm2d, or L1BatchNorm2d (``l1``: mean-absolute-deviation scale, csrc/bn_l1.cu)"""

    def __init__(self, arena, mod):
        from .models.modules.lp_norm import L1BatchNorm2d
        if not mod.affine or not mod.track_running_stats:
            raise B200Error('BatchNorm2d without affine/running stats is not supported')
        self.mod = mod
        self.l1 = isinstance(mod, L1BatchNorm2d)
        self.C = mod.num_features
        sw, sb = arena.slot(mod.weight), arena.slot(mod.bias)
        self.gamma = arena.kernel_view(arena.p32, sw)
        self.beta = arena.kernel_view(arena.p32, sb)
        self.dgamma = arena.kernel_view(arena.g32, sw)
        self.dbeta = arena.kernel_view(arena.g32, sb)


class _SE(object):
    """squeeze-and-excitation gate (models/modules/se.py:6-25 of the reference): two tiny linear layers whose
    parameters live in the arena like the classifier's (bf16 [K,1,C] kernel views, fp32 biases)."""

    def __init__(self, arena, mod):
        from .models.modules.se import SEBlock
        if not isinstance(mod, SEBlock):
            raise B200Error('residual_block of type %s is outside the B200 hot path' % type(mod).__name__)
        l1, l2 = mod.transform[0], mod.transform[2]
        self.C, self.hidden = l1.in_features, l1.out_features
        if self.C % 8 or self.hidden % 8 or l2.out_features != self.C:
            raise B200Error('SE gate: channel counts must be multiples of 8 (got %d -> %d)' % (self.C, self.hidden))
        sw1, sb1, sw2, sb2 = (arena.slot(p) for p in (l1.weight, l1.bias, l2.weight, l2.bias))
        self.w1, self.gw1 = arena.kernel_view(arena.p16, sw1), arena.kernel_view(arena.g32, sw1)
        self.b1, self.gb1 = arena.kernel_view(arena.p32, sb1), arena.kernel_view(arena.g32, sb1)
        self.w2, self.gw2 = arena.kernel_view(arena.p16, sw2), arena.kernel_view(arena.g32, sw2)
        self.b2, self.gb2 = arena.kernel_view(arena.p32, sb2), arena.kernel_view(arena.g32, sb2)

    def fwd(self, r):
        """r' = r * sigmoid(W2 relu(W1 mean(r) + b1) + b2); returns (r', tape)."""
        N = r.shape[0]
        mean = ops.se_pool(r)                                                        # [N,1,1,C] bf16
        d1 = ops.make_desc(N, 1, 1, self.C, self.hidden, 1, 1, 1, 0)
        d2 = ops.make_desc(N, 1, 1, self.hidden, self.C, 1, 1, 1, 0)
        h = ops.conv_fprop(mean, self.w1, d1, bias=self.b1, act=ACT_RELU)            # [N,1,1,C/ratio] bf16
        logit = ops.conv_fprop(h, self.w2, d2, bias=self.b2, out_fp32=True).view(N, self.C)
        return ops.se_scale_fwd(r, logit), (r, mean, h, logit, d1, d2)

    def bwd(self, rt, tape, g):
        """g = dL/dr' -> dL/dr; the gate's parameter gradients accumulate into the arena."""
        r, mean, h, logit, d1, d2 = tape
        N = r.shape[0]
        dlogit = ops.se_bwd_reduce(g, r, logit)                                      # [N,1,1,C] bf16
        ops.colsum_bf16(dlogit.view(N, self.C), self.gb2)
        rt._wgrad_async(lambda: ops.conv_wgrad(h, dlogit, d2, self.gw2), h, dlogit)
        dh = ops.conv_dgrad(dlogit, ops.weight_transpose(self.w2), d2)
        dh = ops.act_bwd(dh, h, ACT_RELU)
        ops.colsum_bf16(dh.view(N, self.hidden), self.gb1)
        rt._wgrad_async(lambda: ops.conv_wgrad(mean, dh, d1, self.gw1), mean, dh)
        dmean = ops.conv_dgrad(dh, ops.weight_transpose(self.w1), d1)
        return ops.se_bwd_dx(g, logit, dmean)


class _Unit(object):
    """saved state of one conv+BN unit for backward."""
    __slots__ = ('x', 'z', 'y', 'w', 'desc', 'mean', 'invstd', 'scale', 'shift', 'sums', 'conv', 'bn', 'act', 'mask',
                 'sign_sum', 'drop')


class Runtime(object):
    """Kernel pipeline for one converted model.  ``forward(x)`` takes the reference's NCHW fp32 input."""

    def __init__(self, model, device):
        self.model = model
        self.device = device
        self.arena = Arena(model, device)
        for name, buf in model.named_buffers():
            buf.data = buf.data.to(device)
        self._anchor = self.arena.slots[0].param
        from .models.modules.lp_norm import L1BatchNorm2d
        self._max_c = max([m.num_features for m in model.modules() if isinstance(m, (nn.BatchNorm2d, L1BatchNorm2d))]
                          + [8])
        self._ws = torch.zeros(ops.bn_workspace_floats(self._max_c), device=device, dtype=torch.float32)
        self._wg_stream = torch.cuda.Stream(device=device)   # weight gradients on a second CUDA stream
        self._wg_keep = []
        self._fold_cache = {}
        self._want_tape = True
        self.loss_scale_inv = 1.0
        self.grad_bucket_hook = None # Trainer (data parallel): .bucket(lo, hi, wg_stream) when g32[lo:hi) is complete,
                                     # .finish() at the end of the backward pass
        self._bucket_hi = None
        self._bucket_min = 1 << 20
        # SyncBatchNorm (main.py:190-191 of the reference: nn.SyncBatchNorm.convert_sync_batchnorm): with sync_bn set
        # (engine.enable_sync_batchnorm) the per-channel sum / sum^2 accumulated by the conv epilogue are all-reduced over
        # the ranks before the statistics are finalised, and d gamma / d beta sums before the BN input gradient
        self.sync_bn_group = None
        self.sync_bn_world = 1
        self._fused_dl = None        # bf16 dlogits handed from _FusedCE.backward to run_backward (side channel)
        self._ce_dummy = torch.zeros((), device=device, dtype=torch.float32)
        # activation checkpointing: while a checkpointed segment runs forward, _conv_and_coeffs records each unit's
        # coefficient vectors here; while it is recomputed in the backward pass, it hands them back in the same order
        self._coeffs_record = None
        self._coeffs_replay = None
        self._build()
        self._setup_transposes()

    def _setup_transposes(self):
        """dgrad reads weights as [C][R*S][K]: one batched launch per step transposes the bf16 shadow of every dense
        (groups == 1) convolution into a second arena; grouped convolutions transpose their expanded weights per
        unit."""
        self._p16t, self._wt_jobs, self._wt_tiles = None, None, 0
        convs = [c for c in self.arena.convs if c.kind == 'conv' and c.groups == 1]
        if not convs:
            return
        self._p16t = torch.empty_like(self.arena.p16)
        spec = []
        for c in convs:
            off, n = c.slot.offset, c.slot.numel
            spec.append((off, off, c.K, c.R * c.S, c.C))
            c.wt = self._p16t[off:off + n].view(c.C, c.R * c.S, c.K)
        self._wt_jobs, self._wt_tiles = ops.transpose_jobs(spec, self.device)

    def _transpose_weights(self):
        if self._wt_jobs is not None:
            ops.weight_transpose_batched(self.arena.p16, self._p16t, self._wt_jobs, self._wt_tiles)

    # ---- program construction (overridden per model family) -------------------------------------
    def _build(self):
        raise NotImplementedError

    # ---- small helpers ----------------------------------------------------------------------------
    def _coeffs(self, n):
        return torch.empty(n, device=self.device, dtype=torch.float32)

    # network input: the reference's contract is a normalised NCHW fp32 batch (trainer.py:116-117).  Additionally a
    # uint8 NHWC batch [N, H, W, C] -- what an image decoder yields BEFORE ToTensor/Normalize (preprocess.py:20-24) --
    # is accepted and normalised inside the relayout kernel (SURVEY.md section 8(f) row 2: device input pipeline).
    input_mean = (0.485, 0.456, 0.406)
    input_std = (0.229, 0.224, 0.225)

    def _input(self, x, mix=None, aug=None):
        """-> (tensor, relayout function, (N, C, H, W)).  ``mix`` (ops.Mix): MixUp / CutMix applied by the relayout
        kernel itself (the reference mixes the fp32 batch before the forward pass, trainer.py:119-135).  ``aug``
        (ops.Aug): x holds the B un-augmented uint8 images and the relayout writes their B*D augmented copies; with
        ops.Rrc or ops.ScaleCropTables x is a flat uint8 region buffer and the relayout resamples it."""
        if isinstance(aug, ops.Rrc):
            # x is the flat uint8 region buffer; the relayout resamples the B*D crops (mode 0 or the mode-2 stem)
            if mix is not None:
                raise B200Error('the resized crop on the device is not combined with MixUp / CutMix')
            if x.dtype != torch.uint8 or x.dim() != 1:
                raise B200Error('the resized crop on the device needs the flat uint8 region buffer; got %s %s'
                                % (x.dtype, tuple(x.shape)))
            OH, OW = aug.size
            return x, (lambda t, cpad, **kw: ops.input_prep_u8_rrc(t, cpad, aug, **kw)), \
                (aug.rows, aug.lut.shape[0], OH, OW)
        if isinstance(aug, ops.ScaleCropTables):
            # x is the flat uint8 region buffer; the relayout resamples each image's centre-crop window (evaluation)
            if mix is not None:
                raise B200Error('the scale crop on the device is not combined with MixUp / CutMix')
            if x.dtype != torch.uint8 or x.dim() != 1:
                raise B200Error('the scale crop on the device needs the flat uint8 region buffer; got %s %s'
                                % (x.dtype, tuple(x.shape)))
            OH, OW = aug.size
            return x, (lambda t, cpad, **kw: ops.input_prep_u8_scale_crop(t, cpad, aug, **kw)), \
                (aug.index.shape[0], aug.lut.shape[0], OH, OW)
        if x.dtype == torch.uint8:
            if x.dim() != 4 or x.shape[-1] > 4:
                raise B200Error('uint8 network inputs must be NHWC [N, H, W, C<=4]; got %s' % (tuple(x.shape),))
            N, H, W, C = x.shape
            if aug is not None:
                if mix is not None:
                    raise B200Error('batch augmentation on the device is not combined with MixUp / CutMix')

                def prep_aug(t, cpad, s2d=False, border=False, **kw):
                    if s2d:
                        raise B200Error('batch augmentation on the device needs the CIFAR-style 3x3 stem '
                                        '(the space-to-depth stem layouts are not supported)')
                    return ops.input_prep_u8_aug(t, cpad, aug, **kw)
                OH, OW = aug.out_hw or (H, W)       # the stem sees the resized copies, not the uint8 images' size
                return x.contiguous(), prep_aug, (aug.rows, C, OH, OW)
            mean = getattr(self.model, 'input_mean', self.input_mean)
            std = getattr(self.model, 'input_std', self.input_std)
            return x.contiguous(), (lambda t, cpad, **kw: ops.input_prep_u8(t, cpad, mean[:C], std[:C], mix=mix, **kw)), \
                (N, C, H, W)
        if aug is not None:
            raise B200Error('batch augmentation on the device needs the uint8 NHWC images; got %s' % (x.dtype,))
        N, C, H, W = x.shape
        return x.float().contiguous(), (lambda t, cpad, **kw: ops.input_prep(t, cpad, mix=mix, **kw)), (N, C, H, W)

    # ---- inference: BatchNorm folded into the convolution (reference utils/absorb_bn.py:18-48) ----------------
    # w' = w * gamma/sqrt(var+eps) per output channel, b' = beta - mean*gamma/sqrt(var+eps) (L1 BN: running_var is
    # the scale itself, w' = w * gamma*running_var, b' = beta - running_mean*gamma*running_var): one kernel computes
    # act(conv(x, w') + b' [+ residual]) -- no z tensor, no separate BN pass.  Folded weights are cached until the
    # parameters or the running statistics change (arena.version).
    def _folded(self, conv, bn):
        key = (id(conv), id(bn))
        hit = self._fold_cache.get(key)
        if hit is not None and hit[0] == self.arena.version:
            return hit[1], hit[2]
        m = bn.mod
        coef = self._coeffs(2 * bn.C)
        scale, shift = coef[:bn.C], coef[bn.C:]
        self._eval_coeffs(bn, scale, shift)
        w32 = conv.w32 * scale.view(-1, 1, 1)                      # [K, T, C/g] fp32, once per version (not per step)
        if conv.groups == 1:
            wf = w32.to(torch.bfloat16).contiguous()
        else:
            wf = conv.kernel_weights(w32.contiguous())
        self._fold_cache[key] = (self.arena.version, wf, shift)
        return wf, shift

    def _unit_fwd_folded(self, x, conv, bn, act, residual=None, other=None):
        N, H, W, _ = x.shape
        u = _Unit()
        u.conv, u.bn, u.act, u.x = conv, bn, act, x
        u.desc = conv.desc(N, H, W)
        wf, bf = self._folded(conv, bn)
        if other is not None:                # downsample branch: r = conv_ds'(x_block) + b_ds', added below
            residual = other.y
        u.z, u.mask = None, None
        u.y = ops.conv_fprop(x, wf, u.desc, bias=bf, residual=residual, act=act)
        return u

    def _unit_fwd(self, x, conv, bn, act, training, tape, residual=None, other=None, drop=None):
        """z = conv(x); BN statistics (train) / running-stat coefficients (eval);
        y = act(bn(z) + residual | + bn_other(z_other)).  Returns y and (if tape) the saved unit.
        drop = (layer, p): in training y = dropout(relu(bn(z))) with the mask of (self.dropout_key, layer); ignored in
        eval mode."""
        if not training and FOLD_BN_EVAL and not self._want_tape:
            return self._unit_fwd_folded(x, conv, bn, act, residual=residual, other=other)
        N, H, W, _ = x.shape
        u = _Unit()
        u.conv, u.bn, u.act, u.x = conv, bn, act, x
        u.desc = conv.desc(N, H, W)
        u.w = conv.kernel_weights()
        self._conv_and_coeffs(u, x, u.w, training)
        u.drop = drop if training else None
        if u.drop is not None:
            # the kept-and-positive bits are the only record of the mask: the backward reads them, never the stream
            u.mask = torch.empty(ops.bn_act_mask_bytes(u.z.numel() // u.z.shape[-1], u.z.shape[-1]), device=self.device,
                                 dtype=torch.uint8)
            u.y = ops.bn_apply_dropout(u.z, u.scale, u.shift, self.dropout_key, drop[0], drop[1], u.mask)
            return u
        # a join (something is added before the activation) cannot recompute act'(.) from z alone: keep one bit per
        # element instead of re-reading the bf16 output in both backward kernels (row-quad words, one extra load per
        # thread and iteration; -0.74 ms/step on ResNet-50)
        u.mask = None
        if tape and training and act != ACT_NONE and (other is not None or residual is not None):
            u.mask = torch.empty(ops.bn_act_mask_bytes(u.z.numel() // u.z.shape[-1], u.z.shape[-1]), device=self.device,
                                 dtype=torch.uint8)
        if other is not None:
            u.y = ops.bn_apply(u.z, u.scale, u.shift, act, z2=other.z, scale2=other.scale, shift2=other.shift,
                               act_mask=u.mask)
        else:
            u.y = ops.bn_apply(u.z, u.scale, u.shift, act, residual=residual, act_mask=u.mask)
        return u

    def _conv_and_coeffs(self, u, x, w16, training):
        """z = conv(x) and the BN coefficients; in training the statistics are accumulated by the conv epilogue
        itself whenever the output width allows it (saves one full read of z).  L1 BN needs the mean before it can
        sum |z - mean|, so its statistics always come from bn_l1_stats."""
        if training and not u.bn.l1 and ops.can_fuse_bn_stats(u.desc.K):
            u.z = ops.conv_fprop(x, w16, u.desc, bn_stats_ws=self._ws)
            self._bn_coeffs(u, training, fused=True)
        else:
            u.z = ops.conv_fprop(x, w16, u.desc)
            self._bn_coeffs(u, training)
        if self._coeffs_record is not None:
            self._coeffs_record.append((u.mean, u.invstd, u.scale, u.shift, u.sums, u.sign_sum))
        elif self._coeffs_replay is not None:
            # recompute of a checkpointed segment: the statistics just computed went to scratch (their running-
            # statistics update is the reference's second one); z is bitwise the forward's, and y is applied with the
            # forward's coefficients so that it and every gradient are too
            u.mean, u.invstd, u.scale, u.shift, u.sums, u.sign_sum = self._coeffs_replay.pop(0)

    def _eval_coeffs(self, bn, scale, shift):
        m = bn.mod
        if bn.l1:
            ops.bn_l1_eval_coeffs(bn.gamma, bn.beta, m.running_mean, m.running_var, scale, shift)
        else:
            ops.bn_eval_coeffs(bn.gamma, bn.beta, m.running_mean, m.running_var, m.eps, scale, shift)

    def _bn_coeffs(self, u, training, fused=False):
        bn = u.bn
        C = bn.C
        buf = self._coeffs((7 if bn.l1 else 6) * C)
        u.mean, u.invstd, u.scale, u.shift, u.sums = buf[0:C], buf[C:2 * C], buf[2 * C:3 * C], buf[3 * C:4 * C], \
            buf[4 * C:6 * C]
        u.sign_sum = buf[6 * C:7 * C] if bn.l1 else None
        m = bn.mod
        if training and self.sync_bn_world > 1 and bn.l1:
            raise B200Error('SyncBatchNorm is not implemented for L1 BatchNorm')
        if training and self.sync_bn_world > 1 and not fused:
            raise B200Error('SyncBatchNorm on the B200 path needs the conv-epilogue statistics (output channels % 64 == 0)')
        if training and bn.l1:
            # invstd holds the L1 scale s: bn_apply and the backward reduction use it like 1/std
            ops.bn_l1_stats(u.z, bn.gamma, bn.beta, m.eps, m.momentum, m.running_mean, m.running_var, u.mean,
                            u.invstd, u.sign_sum, u.scale, u.shift, self._ws)
        elif training and fused:
            M = u.z.numel() // C
            if self.sync_bn_world > 1:
                # the epilogue accumulators are fp64 [16 replicas][2][C] at the start of the BN workspace: ONE small
                # all-reduce makes them global sums; the statistics then are those of the global batch
                import torch.distributed as dist
                dist.all_reduce(self._ws.view(torch.float64)[:16 * 2 * C], group=self.sync_bn_group)
                M *= self.sync_bn_world
            ops.bn_finalize(M, C, bn.gamma, bn.beta, m.eps, m.momentum, m.running_mean, m.running_var,
                            m.num_batches_tracked, u.mean, u.invstd, u.scale, u.shift, self._ws)
        elif training:
            ops.bn_stats(u.z, bn.gamma, bn.beta, m.eps, m.momentum, m.running_mean, m.running_var,
                         m.num_batches_tracked, u.mean, u.invstd, u.scale, u.shift, self._ws)
        else:
            self._eval_coeffs(bn, u.scale, u.shift)
        bias = getattr(u.conv, 'bias32', None) if u.conv is not None else None
        if bias is not None:            # conv bias in front of this BN (never on the ResNet / MobileNet-v2 paths)
            if training:                # the true pre-BN tensor is z + b: only the running mean sees it
                if m.momentum is None:
                    m.running_mean.add_(bias / m.num_batches_tracked.to(torch.float32))
                else:
                    m.running_mean.add_(bias, alpha=float(m.momentum))
            else:
                u.shift.add_(u.scale * bias)

    def _stats_only(self, x, conv, bn, training):
        """conv + BN coefficients without the apply (used for the downsample branch, fused into the main apply)."""
        if not training and FOLD_BN_EVAL and not self._want_tape:
            return self._unit_fwd_folded(x, conv, bn, ACT_NONE)       # y = bn_ds(conv_ds(x)) in one kernel
        N, H, W, _ = x.shape
        u = _Unit()
        u.conv, u.bn, u.act, u.x = conv, bn, ACT_NONE, x
        u.desc = conv.desc(N, H, W)
        u.w = conv.kernel_weights()
        self._conv_and_coeffs(u, x, u.w, training)
        u.y = None
        return u

    def _sync_bn_sums(self, sums):
        """SyncBatchNorm backward: the input gradient needs the GLOBAL d gamma / d beta sums divided by the global pixel
        count; the kernel divides by the local count, so the reduced sums are pre-scaled by 1/world (equal per-rank
        batches).  The arena gradients received the local sums and are averaged with all other gradients later."""
        import torch.distributed as dist
        dist.all_reduce(sums, group=self.sync_bn_group)
        sums.mul_(1.0 / self.sync_bn_world)

    def _bn_bwd(self, u, dy, y_mask, act, want_g=False):
        """BN (+activation) backward of unit u: returns dz (and g = dy*act'(.) when want_g).
        y_mask=None with an activation: the mask is recomputed from z inside the kernels (no read of y)."""
        bn = u.bn
        drop = getattr(u, 'drop', None)
        if drop is not None:        # dropout(relu(bn(z))): g = bit ? dy * c : 0 from the forward's mask bits
            ops.bn_bwd_reduce_dropout(dy, u.z, u.mask, drop[1], u.mean, u.invstd, u.sums, bn.dgamma, bn.dbeta, self._ws)
            if self.sync_bn_world > 1:
                self._sync_bn_sums(u.sums)
            return ops.bn_bwd_dx_dropout(dy, u.z, u.mask, drop[1], u.mean, u.invstd, bn.gamma, u.sums), None
        mask = getattr(u, 'mask', None) if y_mask is not None else None
        ops.bn_bwd_reduce(dy, y_mask, u.z, act, u.mean, u.invstd, bn.gamma, bn.beta, u.sums, bn.dgamma, bn.dbeta,
                          self._ws, act_mask=mask)
        if self.sync_bn_world > 1:
            self._sync_bn_sums(u.sums)
        g = torch.empty_like(dy) if want_g else None
        if bn.l1:     # sums = {sum g*(z-mean)*s, sum g}: the reduction above ran with invstd = s
            dz = ops.bn_l1_bwd_dx(dy, y_mask, u.z, act, u.mean, u.invstd, u.sign_sum, bn.gamma, bn.beta, u.sums,
                                  g_out=g, act_mask=mask)
        else:
            dz = ops.bn_bwd_dx(dy, y_mask, u.z, act, u.mean, u.invstd, bn.gamma, bn.beta, u.sums, g_out=g,
                               act_mask=mask)
        return dz, g

    # ---- weight gradients on a side stream ----------------------------------------------------------------
    # wgrad(conv_i) only feeds the optimiser; the critical path of the backward pass is BN-backward -> dgrad of the
    # units before it.  Launching the wgrads on a second stream lets the tensor/L2-bound wgrad CTAs share the SMs
    # with the HBM-bound BN kernels of the next unit (inside a captured step the fork/join become graph edges).
    def _wgrad_async(self, fn, *operands):
        if self._wg_stream is None:
            fn()
            return
        ev = torch.cuda.Event()
        ev.record()
        self._wg_stream.wait_event(ev)
        with torch.cuda.stream(self._wg_stream):
            fn()
        self._wg_keep.append(operands)   # main-stream allocations: keep them alive (un-reused) until the join

    def _wgrad_join(self):
        if self._wg_stream is not None and self._wg_keep:
            torch.cuda.current_stream().wait_stream(self._wg_stream)
            self._wg_keep = []

    # ---- gradient buckets for the data-parallel all-reduce ------------------------------------------------------
    # Dense conv / fc weights sit in the arena in forward (module) order and the backward pass completes them in
    # reverse, so "every dense weight gradient at offset >= lo is final" holds at block boundaries.  Whenever at
    # least _bucket_min elements have become final, the hook (Trainer: an NCCL all-reduce on a communication stream)
    # is called for that arena range while the rest of the backward pass keeps running -- the reference gets the same
    # overlap from DistributedDataParallel's 25 MB buckets (trainer.py:79-82).  The remainder (early layers, depthwise
    # weights, BN / bias vectors) goes out in a final call at the end of the pass.
    def _buckets_begin(self):
        self._bucket_hi = self.arena.group_end[0] if self.grad_bucket_hook is not None else None

    def _bucket_point(self, lo, force=False):
        """gradients of every dense weight at arena offset >= lo are complete (their wgrads are enqueued)."""
        if self._bucket_hi is None:
            return
        if lo < self._bucket_hi and (force or self._bucket_hi - lo >= self._bucket_min):
            self.grad_bucket_hook.bucket(lo, self._bucket_hi, self._wg_stream)
            self._bucket_hi = lo

    def _buckets_end(self):
        if self._bucket_hi is None:
            return
        self._bucket_point(0, force=True)
        a = self.arena
        if a.total > a.group_end[0]:
            self.grad_bucket_hook.bucket(a.group_end[0], a.total, None)   # depthwise weights, biases, BN affine
        self.grad_bucket_hook.finish()
        self._bucket_hi = None

    @staticmethod
    def _spec_lo(convs):
        return min(c.slot.offset for c in convs)

    def _conv_bwd(self, u, dz, need_dx=True, residual=None):
        """wgrad into the gradient arena and (optionally) dgrad."""
        conv = u.conv
        if conv.groups == 1:
            self._wgrad_async(lambda: ops.conv_wgrad(u.x, dz, u.desc, conv.g32), u.x, dz)
        else:  # windowed (block-diagonal) wgrad into a scratch [K, T, window], then keep each channel's group
            def grouped():
                T = conv.R * conv.S
                N, H, W, _ = u.x.shape
                win = 128 if conv.window else conv.C
                scratch = torch.zeros((conv.K, T, win), device=self.device, dtype=torch.float32)
                ops.conv_wgrad(u.x, dz, conv.desc(N, H, W, wgrad=True), scratch)
                ops.group_wgrad_unpack(scratch, conv.K, T, conv.C, conv.groups, win, conv.g32)
            self._wgrad_async(grouped, u.x, dz)
        if not need_dx:
            return None
        if conv.groups > 1:
            wt = conv.dgrad_weights()
        else:
            wt = conv.wt
        return ops.conv_dgrad(dz, wt, u.desc, residual=residual)

    # ---- classifier head: global average pool -> (dropout) -> linear as a 1x1 conv on a 1x1 map ----------
    def _head_build(self, fc, dropout_p=0.0):
        a = self.arena
        sw, sb = a.slot(fc.weight), a.slot(fc.bias)
        self.classes = fc.out_features
        self.classes_pad = _round_up(self.classes, 8)
        self.fc_in = fc.in_features
        self.fc_w16 = a.kernel_view(a.p16, sw)       # [Kpad,1,C]
        self.fc_gw = a.kernel_view(a.g32, sw)
        self.fc_b = a.kernel_view(a.p32, sb)         # [Kpad]
        self.fc_gb = a.kernel_view(a.g32, sb)
        self.dropout_p = float(dropout_p)

    def _head_fwd(self, h, training, want_tape):
        N = h.shape[0]
        feat = ops.avgpool_fwd(h)                                        # [N,1,1,C]
        mask = None
        if training and self.dropout_p > 0:
            # the Bernoulli draw uses torch's CUDA generator (RNG glue on a [N, C] tensor; mobilenet_v2.py:126)
            keep = 1.0 - self.dropout_p
            mask = (torch.rand(feat.shape, device=self.device) < keep).to(torch.bfloat16) / keep
            feat = feat * mask
        desc = ops.make_desc(N, 1, 1, self.fc_in, self.classes_pad, 1, 1, 1, 0, algo_macs=self.fc_in * self.classes)
        logits = ops.conv_fprop(feat, self.fc_w16, desc, bias=self.fc_b, out_fp32=True).view(N, self.classes_pad)
        out = logits if self.classes_pad == self.classes else logits[:, :self.classes]
        tape = {'feat': feat, 'mask': mask, 'last_shape': tuple(h.shape), 'fc_desc': desc,
                'logits_pad': logits} if want_tape else None
        return out, tape

    def _head_bwd(self, tape, dlogits, dl_bf16=None):
        N = dlogits.shape[0]
        if dl_bf16 is not None:              # written by the fused softmax-CE kernel: bf16, padded, pad columns zero
            dl = dl_bf16
        elif self.classes_pad == self.classes:
            dl = torch.empty((N, self.classes_pad), device=self.device, dtype=torch.bfloat16)
            ops.cast_bf16(dlogits.contiguous().float(), dl)
        else:
            dl = torch.zeros((N, self.classes_pad), device=self.device, dtype=torch.bfloat16)
            dl[:, :self.classes].copy_(dlogits)
        desc = tape['fc_desc']
        dl4 = dl.view(N, 1, 1, self.classes_pad)
        ops.colsum_bf16(dl, self.fc_gb)
        feat = tape['feat']
        self._wgrad_async(lambda: ops.conv_wgrad(feat, dl4, desc, self.fc_gw), feat, dl4)
        wt = ops.weight_transpose(self.fc_w16)
        dfeat = ops.conv_dgrad(dl4, wt, desc)
        if tape['mask'] is not None:
            dfeat = dfeat * tape['mask']
        return ops.avgpool_bwd(dfeat, tape['last_shape'])

    # ---- autograd glue ----------------------------------------------------------------------------
    def forward(self, x):
        if x.device.type != 'cuda':
            raise B200Error('B200 runtime needs CUDA inputs (no CPU fallback); got %s' % x.device)
        training = self.model.training
        if torch.is_grad_enabled() and training:
            out = _NetFn.apply(x, self._anchor, self, training)
            out._b200_head = _HeadHandle(self, self._last_logits_pad)   # lets CrossEntropyLoss take the fused kernel
            return out
        # eval mode never tapes (BatchNorm backward with running statistics is not implemented): the logits carry no
        # autograd history, so a backward() through them fails loudly instead of using batch-statistics formulas
        logits, _ = self.run_forward(x, training, False)
        return logits

    def run_forward(self, x, training, want_tape, mix=None, aug=None):
        raise NotImplementedError

    def run_backward(self, tape, dlogits, dl_bf16=None):
        raise NotImplementedError

    def train_step(self, x, target, smooth_eps=0.0, upstream=None, mix=None, aug=None, reduce=True):
        """forward + mean softmax cross-entropy (label smoothing ``smooth_eps``) + backward of one batch as a straight
        sequence of library calls -- no autograd graph, no autograd worker thread, no ATen kernels: what Trainer runs
        (and captures into a CUDA graph) when the criterion is the plain CrossEntropyLoss of the reference
        (trainer.py:132-162 with utils/cross_entropy.py:20-24,46-52).  ``upstream``: optional 0-dim fp32 device tensor
        multiplied into the gradients (loss scale x grad scale).  Gradients accumulate into the arena.
        ``mix`` (ops.Mix): MixUp / CutMix of the batch (trainer.py:119-135 with utils/mixup.py of the reference) -- the
        relayout kernel mixes the input and the loss is the soft-target cross-entropy against lam*onehot(target) +
        (1-lam)*onehot(target[perm]); ``smooth_eps`` is then ignored, as the reference's cross_entropy ignores it for
        soft targets (utils/cross_entropy.py:38-54).  Top-1 / top-5 still count against ``target``.
        ``aug`` (ops.Aug): x is the uint8 NHWC batch of B images and the step trains on its B*D augmented copies
        (row b*D + d); ``target`` then has B*D entries, or aug.window's n.
        ``reduce``: False keeps the data-parallel gradient buckets (grad_bucket_hook) out of this backward pass -- a
        chunk of an accumulated batch whose summed gradients are all-reduced once, after its last chunk.
        Returns (logits, stats): logits detached, stats = fp32[3] device tensor {mean loss, top-1 %, top-5 %}."""
        if x.device.type != 'cuda':
            raise B200Error('B200 runtime needs CUDA inputs (no CPU fallback); got %s' % x.device)
        n_rows = aug.rows if aug is not None else x.shape[0]
        if target.dtype != torch.int64 or target.dim() != 1 or target.shape[0] != n_rows or not target.is_cuda:
            raise B200Error('train_step: target must be a CUDA int64 vector with one class index per sample')
        logits, tape = self.run_forward(x, True, True, mix=mix, aug=aug)
        pad = tape['head']['logits_pad']
        dev = pad.device
        stats = torch.empty(3, device=dev, dtype=torch.float32)
        rows = torch.empty(2 * pad.shape[0], device=dev, dtype=torch.float32)
        dl = torch.empty(pad.shape, device=dev, dtype=torch.bfloat16)
        up = None
        if upstream is not None:
            up = upstream.reshape(1)
        if mix is not None:
            ops.softmax_ce_mix(pad, target.contiguous(), mix, self.classes, loss=stats, row_loss=rows, dlogits=dl,
                               grad_scale_dev=up)
        else:
            ops.softmax_ce(pad, target.contiguous(), self.classes, smooth_eps, loss=stats, row_loss=rows, dlogits=dl,
                           grad_scale_dev=up)
        self.arena.rebind_grads()
        self.arena.grads_zero = False
        hook = self.grad_bucket_hook
        if not reduce:
            self.grad_bucket_hook = None
        try:
            self.run_backward(tape, logits, dl_bf16=dl)
        finally:
            self.grad_bucket_hook = hook
        return logits, stats


class _HeadHandle(object):
    """Tag on the logits of a taped forward: the padded fp32 logits storage + the runtime that produced them."""
    __slots__ = ('rt', 'logits_pad', 'stats')

    def __init__(self, rt, logits_pad):
        self.rt, self.logits_pad, self.stats = rt, logits_pad, None

    def loss(self, logits, target, smooth_eps=0.0):
        return _FusedCE.apply(logits, target, float(smooth_eps or 0.0), self)


class _FusedCE(torch.autograd.Function):
    """mean softmax cross-entropy with label smoothing (reference utils/cross_entropy.py:20-24,46-52) on the fused
    kernel.  backward writes bf16 dlogits (already multiplied by the upstream gradient, read on the device) straight
    into the buffer the classifier's dgrad/wgrad kernels consume; autograd only carries a zero-stride placeholder."""

    @staticmethod
    def forward(ctx, logits, target, eps, head):
        pad, rt = head.logits_pad, head.rt
        if logits.data_ptr() != pad.data_ptr() or logits.shape != (pad.shape[0], rt.classes) or \
                target.shape != (pad.shape[0],) or target.dtype != torch.int64 or not target.is_cuda:
            raise B200Error('fused cross-entropy: logits/target do not belong to this forward pass')
        target = target.contiguous()
        stats = torch.empty(3, device=pad.device, dtype=torch.float32)          # loss, top-1 %, top-5 %
        rows = torch.empty(2 * pad.shape[0], device=pad.device, dtype=torch.float32)
        ops.softmax_ce(pad, target, rt.classes, eps, loss=stats, row_loss=rows)
        ctx.head, ctx.eps = head, eps
        ctx.save_for_backward(target)
        head.stats = stats
        return stats[0]

    @staticmethod
    def backward(ctx, gout):
        head, (target,) = ctx.head, ctx.saved_tensors
        pad, rt = head.logits_pad, head.rt
        up = gout.reshape(1)
        if up.dtype != torch.float32 or not up.is_contiguous():
            up = up.float().contiguous()
        dl = torch.empty(pad.shape, device=pad.device, dtype=torch.bfloat16)
        ops.softmax_ce(pad, target, rt.classes, ctx.eps, dlogits=dl, grad_scale_dev=up)
        rt._fused_dl = dl
        return rt._ce_dummy.expand(pad.shape[0], rt.classes), None, None, None


class _NetFn(torch.autograd.Function):
    """One autograd node for the whole network: backward writes parameter gradients into the arena."""

    @staticmethod
    def forward(ctx, x, anchor, rt, training):
        logits, tape = rt.run_forward(x.detach(), training, True)
        ctx.rt, ctx.tape = rt, tape
        rt._last_logits_pad = tape['head']['logits_pad']
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        rt, tape = ctx.rt, ctx.tape
        ctx.tape = None
        rt.arena.rebind_grads()
        rt.arena.grads_zero = False
        side, rt._fused_dl = rt._fused_dl, None
        if side is not None and (side.shape[0] != dlogits.shape[0] or side.device != dlogits.device):
            side = None
        if side is not None and not (dlogits.data_ptr() == rt._ce_dummy.data_ptr() and dlogits.stride() == (0, 0)):
            # the logits had another consumer besides the fused loss: add its gradient (rare; torch glue)
            dlogits = dlogits + side[:, :rt.classes].float()
            side = None
        rt.run_backward(tape, dlogits, dl_bf16=side)
        return None, None, None, None


# ----------------------------------------------------------------------------------------------------
class ResNetRuntime(Runtime):
    """Pipeline for models.resnet.ResNet_imagenet / ResNet_cifar (BasicBlock or Bottleneck)."""

    def _build(self):
        from .models.resnet import BasicBlock, Bottleneck
        from .models.modules.lp_norm import L1BatchNorm2d
        from .models.modules.checkpoint import CheckpointModule
        m, a = self.model, self.arena
        self.imagenet_stem = m.conv1.kernel_size == (7, 7)
        if self.imagenet_stem:
            if m.conv1.stride != (2, 2) or m.conv1.padding != (3, 3) or m.conv1.in_channels != 3:
                raise B200Error('unsupported 7x7 stem geometry')
        elif m.conv1.kernel_size != (3, 3) or m.conv1.stride != (1, 1) or m.conv1.in_channels > 16:
            raise B200Error('unsupported stem geometry')
        self.stem_conv = m.conv1
        s = a.slot(m.conv1.weight)
        self.stem_w32 = a.p32[s.offset:s.offset + s.numel]      # [K][R][S][C] fp32
        self.stem_g32 = a.g32[s.offset:s.offset + s.numel]
        self.stem_bn = _BN(a, m.bn1)
        self.has_maxpool = isinstance(m.maxpool, nn.MaxPool2d)
        self.blocks = []
        # checkpoint_segments: [start, end) ranges of self.blocks whose activations the forward pass does not keep;
        # the backward pass recomputes each range just before it needs it
        self.segments = []
        n_drop = 0
        for lname in ('layer1', 'layer2', 'layer3', 'layer4'):
            layer = getattr(m, lname)
            if isinstance(layer, nn.Identity):
                continue
            if isinstance(layer, CheckpointModule):
                base = len(self.blocks)
                self.segments += [(base + a, base + b) for a, b in layer.segments()]
                layer = layer.module
            for blk in layer:
                p = float(blk.dropout.p) if isinstance(blk.dropout, nn.Dropout) else 0.0
                if p != 0 and not isinstance(blk, BasicBlock):
                    raise B200Error('dropout inside residual blocks is not supported on the B200 path')
                spec = {'kind': 'bottleneck' if isinstance(blk, Bottleneck) else 'basic'}
                if not isinstance(blk, (BasicBlock, Bottleneck)):
                    raise B200Error('unknown block type %s' % type(blk).__name__)
                # BasicBlock dropout after relu(bn1(conv1(x))): fused into that unit's apply and backward (dropout.cu),
                # layer index = position among the network's dropout layers (part of the mask's Philox counter)
                spec['drop'] = None
                if p != 0:
                    if not 0.0 < p < 1.0:
                        raise B200Error('dropout rate %r inside residual blocks: the B200 path needs 0 < p < 1' % p)
                    if isinstance(blk.bn1, L1BatchNorm2d):
                        raise B200Error('dropout with L1 BatchNorm is not supported on the B200 path')
                    spec['drop'] = (n_drop, p)
                    n_drop += 1
                names = ('conv1', 'conv2', 'conv3') if spec['kind'] == 'bottleneck' else ('conv1', 'conv2')
                spec['convs'] = [_Conv(a, getattr(blk, n)) for n in names]
                spec['bns'] = [_BN(a, getattr(blk, n.replace('conv', 'bn'))) for n in names]
                spec['down'] = None
                if blk.downsample is not None:
                    spec['down'] = (_Conv(a, blk.downsample[0]), _BN(a, blk.downsample[1]))
                # squeeze-excitation on the residual branch (resnet_se / resnext_se): one gate per stage, shared
                spec['se'] = _SE(a, blk.residual_block) if blk.residual_block is not None else None
                self.blocks.append(spec)
        self._head_build(m.fc)
        # one 64-bit Philox key per training step, drawn on the device with torch's CUDA generator (a captured step
        # draws a fresh one on every replay; torch.manual_seed makes runs reproducible)
        self.dropout_key = torch.zeros(1, device=self.device, dtype=torch.int64) if n_drop else None

    # ---- stem ---------------------------------------------------------------------------------------
    def _stem_fwd(self, x, training, mix=None, aug=None):
        x, prep, (N, Cin, H, W) = self._input(x, mix, aug)
        K = self.stem_conv.out_channels
        st = {}
        if self.imagenet_stem:
            ws = torch.empty((K, 16, 16), device=self.device, dtype=torch.bfloat16)
            ops.stem_weight_to_s2d(self.stem_w32, K, Cin, 16, ws)
            Hs, Ws = H // 2, W // 2
            # 7x7/s2 -> space-to-depth 4x4/s1 on 16 channels -> 4x1 on "wide pixels": 4 neighbouring 32-byte
            # pixels of the zero-bordered tensor are read as ONE 64-channel (128 B) pixel, so every tap row is a
            # full 128B-swizzle TMA tile (4 loads per tile instead of 16 quarter-width ones).
            xs = prep(x, 16, s2d=True, border=True)                # [N, Hs+3, Ws+3, 16], data at (+2,+2)
            desc = ops.make_desc(N, Hs + 3, Ws, 64, K, 4, 1, 1, 0, P=Hs, Q=Ws,
                                 x_strides=(16, (Ws + 3) * 16, (Hs + 3) * (Ws + 3) * 16), algo_macs=K * 49 * Cin)
            if Ws + 3 <= 128:
                # same bordered tensor described as the dense 4x4 / pad-0 convolution it is: the library runs it
                # on the halo kernel (one 32-byte-row tile load per output row, weights stationary in smem)
                desc = ops.make_desc(N, Hs + 3, Ws + 3, 16, K, 4, 4, 1, 0, P=Hs, Q=Ws, algo_macs=K * 49 * Cin)
        else:
            xs = prep(x, 16, s2d=False)
            ws = torch.zeros((K, 9, 16), device=self.device, dtype=torch.bfloat16)
            ws[:, :, :Cin].copy_(self.stem_w32.view(K, 9, Cin))       # 432-element pad+cast of the 3-channel stem
            desc = ops.make_desc(N, H, W, 16, K, 3, 3, 1, 1, algo_macs=K * 9 * Cin)
        u = _Unit()
        u.conv, u.bn, u.act, u.x, u.desc = None, self.stem_bn, ACT_RELU, xs, desc
        self._conv_and_coeffs(u, xs, ws, training)
        st['unit'] = u
        if self.has_maxpool:
            # bn1 -> relu -> maxpool in one pass: the [N, 112, 112, 64] activation is never written
            u.y = None
            out, st['argmax'] = ops.bn_apply_maxpool(u.z, u.scale, u.shift, ACT_RELU)
        else:
            u.y = ops.bn_apply(u.z, u.scale, u.shift, ACT_RELU)
            out = u.y
        st['cin'] = Cin
        return out, st

    def _stem_bwd(self, st, dy):
        u = st['unit']
        if self.has_maxpool:
            dy = ops.maxpool_bwd(dy, st['argmax'], tuple(u.z.shape))
        dz, _ = self._bn_bwd(u, dy, None, ACT_RELU)   # mask recomputed from z: the activation is not needed
        K, Cin = self.stem_conv.out_channels, st['cin']
        def stem_wgrad():   # every wgrad shares the split-K workspace: all of them go through _wgrad_async
            if self.imagenet_stem:
                dws = torch.zeros((K, 16, 16), device=self.device, dtype=torch.float32)
                ops.conv_wgrad(u.x, dz, u.desc, dws)
                ops.stem_wgrad_from_s2d(dws, K, Cin, 16, self.stem_g32)
            else:
                dws = torch.zeros((K, 9, 16), device=self.device, dtype=torch.float32)
                ops.conv_wgrad(u.x, dz, u.desc, dws)
                self.stem_g32.view(K, 9, Cin).add_(dws[:, :, :Cin])
        self._wgrad_async(stem_wgrad, u.x, dz)

    # ---- residual blocks ----------------------------------------------------------------------------
    def _block_fwd(self, spec, x, training):
        convs, bns = spec['convs'], spec['bns']
        units = []
        h = x
        for i in range(len(convs) - 1):
            u = self._unit_fwd(h, convs[i], bns[i], ACT_RELU, training, True, drop=spec['drop'] if i == 0 else None)
            units.append(u)
            h = u.y
        down, se_tape = None, None
        if spec.get('se') is not None:
            # residual = SE(downsample(x) | x): the gate needs the materialised residual, so the downsample branch
            # gets its own BN-apply pass here instead of being folded into the join
            r = x
            if spec['down'] is not None:
                down = self._unit_fwd(x, spec['down'][0], spec['down'][1], ACT_NONE, training, True)
                r = down.y
            r, se_tape = spec['se'].fwd(r)
            last = self._unit_fwd(h, convs[-1], bns[-1], ACT_RELU, training, True, residual=r)
        elif spec['down'] is not None:
            down = self._stats_only(x, spec['down'][0], spec['down'][1], training)
            last = self._unit_fwd(h, convs[-1], bns[-1], ACT_RELU, training, True, other=down)
        else:
            last = self._unit_fwd(h, convs[-1], bns[-1], ACT_RELU, training, True, residual=x)
        units.append(last)
        return last.y, {'units': units, 'down': down, 'se': se_tape}

    def _block_bwd(self, spec, saved, dy):
        units, down = saved['units'], saved['down']
        last = units[-1]
        # out = relu(bn_last(z) + skip): g = dy * (out > 0) feeds both branches
        dz, g = self._bn_bwd(last, dy, last.y, ACT_RELU, want_g=True)
        if saved.get('se') is not None:
            g = spec['se'].bwd(self, saved['se'], g)          # through the gate: dL/d(residual before SE)
        if down is not None:
            dzd, _ = self._bn_bwd(down, g, None, ACT_NONE)
            skip = self._conv_bwd(down, dzd)
        else:
            skip = g
        d = self._conv_bwd(last, dz)
        for u in reversed(units[1:-1]):
            dz, _ = self._bn_bwd(u, d, None, ACT_RELU)
            d = self._conv_bwd(u, dz)
        u = units[0]
        dz, _ = self._bn_bwd(u, d, None, ACT_RELU)
        return self._conv_bwd(u, dz, residual=skip)

    # ---- whole network ------------------------------------------------------------------------------
    def run_forward(self, x, training, want_tape, mix=None, aug=None):
        self._want_tape = want_tape
        if training:
            self.arena.version += 1          # running statistics change: folded inference weights become stale
            if self.dropout_key is not None:
                self.dropout_key.random_(-2 ** 63, None)         # the full 64-bit range
        h, stem = self._stem_fwd(x, training, mix, aug)
        saved = []
        # eval and tapeless training forwards (calibrate_bn) keep nothing to recompute: only a backward pass needs it
        ckpt = {a: b for a, b in self.segments} if (training and want_tape) else {}
        i = 0
        while i < len(self.blocks):
            if i in ckpt:
                # checkpointed segment: keep its input and each unit's coefficients; z, y and the masks are dropped
                seg_in, coeffs = h, []
                try:
                    for spec in self.blocks[i:ckpt[i]]:
                        self._coeffs_record = []
                        h, _ = self._block_fwd(spec, h, training)
                        coeffs.append(self._coeffs_record)
                finally:
                    self._coeffs_record = None
                saved.append({'segment': (i, ckpt[i]), 'x': seg_in, 'coeffs': coeffs})
                saved += [None] * (ckpt[i] - i - 1)
                i = ckpt[i]
                continue
            h, s = self._block_fwd(self.blocks[i], h, training)
            saved.append(s if want_tape else None)
            i += 1
        out, head = self._head_fwd(h, training, want_tape)
        tape = {'stem': stem, 'blocks': saved, 'head': head} if want_tape else None
        return out, tape

    def _recompute(self, seg):
        """the block tapes of a checkpointed segment, rebuilt from its input by the forward's own launches"""
        h, tapes = seg['x'], []
        a, b = seg['segment']
        try:
            for spec, coeffs in zip(self.blocks[a:b], seg['coeffs']):
                self._coeffs_replay = list(coeffs)
                h, s = self._block_fwd(spec, h, True)
                tapes.append(s)
        finally:
            self._coeffs_replay = None
        return tapes

    def run_backward(self, tape, dlogits, dl_bf16=None):
        self._transpose_weights()
        self._buckets_begin()
        d = self._head_bwd(tape['head'], dlogits, dl_bf16)
        blocks = list(tape['blocks'])
        seg_start = {s['segment'][1] - 1: i for i, s in enumerate(blocks) if s is not None and 'segment' in s}
        for i in range(len(self.blocks) - 1, -1, -1):
            spec = self.blocks[i]
            if i in seg_start:
                a = seg_start[i]
                blocks[a:i + 1] = self._recompute(blocks[a])
            d = self._block_bwd(spec, blocks[i], d)
            blocks[i] = None
            convs = spec['convs'] + ([spec['down'][0]] if spec['down'] is not None else [])
            self._bucket_point(self._spec_lo(convs))
            if i in seg_start.values():
                # end of a recomputed segment's backward: the side-stream wgrads still read its tensors; joining here
                # lets the allocator hand them to the next segment instead of keeping every segment to the end
                self._wgrad_join()
        self._stem_bwd(tape['stem'], d)
        self._wgrad_join()
        self._buckets_end()


class MobileNetRuntime(Runtime):
    """Pipeline for models.mobilenet_v2.MobileNet_v2: 1x1 expand / depthwise 3x3 / 1x1 project units with
    BN + ReLU6, identity skips, dropout + linear head (reference: models/mobilenet_v2.py:39-156)."""

    def _build(self):
        m, a = self.model, self.arena
        f = m.features
        conv0 = f.conv0[0]
        if conv0.kernel_size != (3, 3) or conv0.in_channels > 16 or conv0.groups != 1:
            raise B200Error('unsupported MobileNet stem')
        self.stem_conv = conv0
        s = a.slot(conv0.weight)
        self.stem_w32 = a.p32[s.offset:s.offset + s.numel]
        self.stem_g32 = a.g32[s.offset:s.offset + s.numel]
        self.stem_bn = _BN(a, f.conv0[1])
        self.blocks = []
        for name, mod in f.named_children():
            if not name.startswith('bottleneck'):
                continue
            if mod.residual_block is not None:
                raise B200Error('residual_block is outside the B200 hot path')
            self.blocks.append({'add_res': mod.add_res, 'units': self._parse_units(list(mod.block))})
        self.blocks.append({'add_res': False, 'units': self._parse_units(list(f.conv1))})
        drop, fc = m.classifier[0], m.classifier[1]
        self._head_build(fc, dropout_p=drop.p if isinstance(drop, nn.Dropout) else 0.0)
        max_c = max(u[1].C for b in self.blocks for u in b['units'] if u[0] == 'dw')
        self._dw_ws = torch.empty(592 * 9 * max_c, device=self.device, dtype=torch.float32)

    def _parse_units(self, layers):
        units, i = [], 0
        while i < len(layers):
            conv, bn = layers[i], layers[i + 1]
            has_act = i + 2 < len(layers) and isinstance(layers[i + 2], (nn.ReLU6, nn.ReLU))
            act = ACT_NONE
            if has_act:
                act = ACT_RELU6 if isinstance(layers[i + 2], nn.ReLU6) else ACT_RELU
            kind = 'dw' if conv.groups > 1 else 'dense'
            units.append((kind, _Conv(self.arena, conv), _BN(self.arena, bn), act))
            i += 3 if has_act else 2
        return units

    def _mb_unit_fwd(self, x, kind, conv, bn, act, training, residual=None):
        N, H, W, _ = x.shape
        u = _Unit()
        u.conv, u.bn, u.act, u.x = conv, bn, act, x
        u.desc = conv.desc(N, H, W)
        if kind == 'dw':
            u.w = None
            u.z = ops.dwconv_fprop(x, conv.w16, u.desc)
            self._bn_coeffs(u, training)
        else:
            u.w = conv.kernel_weights()
            self._conv_and_coeffs(u, x, u.w, training)
        u.y = ops.bn_apply(u.z, u.scale, u.shift, act, residual=residual)
        return u

    def _mb_conv_bwd(self, kind, u, dz, need_dx=True, residual=None):
        if kind == 'dw':
            # like the dense weight gradients: on the side stream (all depthwise wgrads share _dw_ws, the stream orders
            # them), off the BN-backward -> dgrad chain
            self._wgrad_async(lambda: ops.dwconv_wgrad(u.x, dz, u.desc, u.conv.g32, self._dw_ws), u.x, dz)
            return ops.dwconv_dgrad(dz, u.conv.w16, u.desc) if need_dx else None
        return self._conv_bwd(u, dz, need_dx=need_dx, residual=residual)

    def _stem_fwd(self, x, training, mix=None, aug=None):
        x, prep, (N, Cin, H, W) = self._input(x, mix, aug)
        K = self.stem_conv.out_channels
        xs = prep(x, 16, s2d=False)
        ws = torch.zeros((K, 9, 16), device=self.device, dtype=torch.bfloat16)
        ws[:, :, :Cin].copy_(self.stem_w32.view(K, 9, Cin))
        st, pad = self.stem_conv.stride[0], self.stem_conv.padding[0]
        act = getattr(self, 'stem_act', ACT_RELU6)
        u = _Unit()
        u.conv, u.bn, u.act, u.x = None, self.stem_bn, act, xs
        u.desc = ops.make_desc(N, H, W, 16, K, 3, 3, st, pad, algo_macs=K * 9 * Cin)
        u.z = ops.conv_fprop(xs, ws, u.desc)
        self._bn_coeffs(u, training)
        u.y = ops.bn_apply(u.z, u.scale, u.shift, act)
        return u.y, {'unit': u, 'cin': Cin}

    def _stem_bwd(self, st, dy):
        u = st['unit']
        dz, _ = self._bn_bwd(u, dy, None, u.act)
        K, Cin = self.stem_conv.out_channels, st['cin']
        def stem_wgrad():
            dws = torch.zeros((K, 9, 16), device=self.device, dtype=torch.float32)
            ops.conv_wgrad(u.x, dz, u.desc, dws)
            self.stem_g32.view(K, 9, Cin).add_(dws[:, :, :Cin])
        self._wgrad_async(stem_wgrad, u.x, dz)

    def run_forward(self, x, training, want_tape, mix=None, aug=None):
        self._want_tape = want_tape
        if training:
            self.arena.version += 1
        h, stem = self._stem_fwd(x, training, mix, aug)
        saved = []
        for spec in self.blocks:
            xin, units = h, []
            for j, (kind, conv, bn, act) in enumerate(spec['units']):
                last = j == len(spec['units']) - 1
                u = self._mb_unit_fwd(h, kind, conv, bn, act, training,
                                      residual=xin if (last and spec['add_res']) else None)
                units.append(u)
                h = u.y
            saved.append(units if want_tape else None)
        out, head = self._head_fwd(h, training, want_tape)
        tape = {'stem': stem, 'blocks': saved, 'head': head} if want_tape else None
        return out, tape

    def run_backward(self, tape, dlogits, dl_bf16=None):
        self._transpose_weights()
        self._buckets_begin()
        d = self._head_bwd(tape['head'], dlogits, dl_bf16)
        for spec, units in zip(reversed(self.blocks), reversed(tape['blocks'])):
            skip = d if spec['add_res'] else None   # out = bn(z) + x (no activation): the skip gradient is dy itself
            for j in range(len(units) - 1, -1, -1):
                kind, _, _, act = spec['units'][j]
                u = units[j]
                dz, _ = self._bn_bwd(u, d, None, act)
                d = self._mb_conv_bwd(kind, u, dz, residual=skip if j == 0 else None)
            dense = [c for k, c, _, _ in spec['units'] if k != 'dw']
            if dense:
                self._bucket_point(self._spec_lo(dense))
        self._stem_bwd(tape['stem'], d)
        self._wgrad_join()
        self._buckets_end()


class MobileNetV1Runtime(MobileNetRuntime):
    """Pipeline for models.mobilenet.MobileNet (v1): stem conv + BN + ReLU, 13 x [depthwise 3x3 (+bias) + BN + ReLU,
    1x1 + BN + ReLU], global average pool, linear (reference: models/mobilenet.py:39-156) -- the unit kernels of
    MobileNetRuntime with ReLU instead of ReLU6 and no skips."""

    def _build(self):
        m, a = self.model, self.arena
        layers = list(m.features)
        conv0, bn0 = layers[0], layers[1]
        if conv0.kernel_size != (3, 3) or conv0.in_channels > 16 or conv0.groups != 1 or conv0.bias is not None:
            raise B200Error('unsupported MobileNet stem')
        self.stem_conv = conv0
        s = a.slot(conv0.weight)
        self.stem_w32 = a.p32[s.offset:s.offset + s.numel]
        self.stem_g32 = a.g32[s.offset:s.offset + s.numel]
        self.stem_bn = _BN(a, bn0)
        self.stem_act = ACT_RELU6 if isinstance(layers[2], nn.ReLU6) else ACT_RELU
        self.blocks = []
        for mod in layers[3:]:
            self.blocks.append({'add_res': False, 'units': self._parse_units(list(mod.components))})
        self._head_build(m.fc, dropout_p=0.0)
        max_c = max(u[1].C for b in self.blocks for u in b['units'] if u[0] == 'dw')
        self._dw_ws = torch.empty(592 * 9 * max_c, device=self.device, dtype=torch.float32)


def enable_sync_batchnorm(model, process_group=None):
    """SyncBatchNorm for a converted model (``--sync-bn``, main.py:82-83,190-191 of the reference): batch statistics and
    the BN backward sums are taken over all ranks of ``process_group`` (equal per-rank batches assumed, as with
    DistributedSampler).  Two small all-reduces per BN layer and step; every layer's output width must allow the fused
    conv-epilogue statistics (multiples of 64 channels)."""
    import torch.distributed as dist
    rt = getattr(model, '_b200', None)
    if rt is None:
        raise B200Error('enable_sync_batchnorm needs a model converted by convert_b200')
    if not (dist.is_available() and dist.is_initialized()):
        raise B200Error('enable_sync_batchnorm needs an initialised process group')
    from .models.modules.lp_norm import L1BatchNorm2d
    if any(isinstance(m, L1BatchNorm2d) for m in model.modules()):
        raise NotImplementedError('SyncBatchNorm is not implemented for L1 BatchNorm (bn_norm=\'L1\')')
    if getattr(rt, 'segments', None):
        raise NotImplementedError('SyncBatchNorm is not implemented with checkpoint_segments: the recompute would '
                                  'all-reduce every checkpointed layer\'s statistics a second time')
    rt.sync_bn_group = process_group
    rt.sync_bn_world = dist.get_world_size(process_group)
    return model


def convert_b200(model, device=None):
    """Convert a registry model for the B200 kernel path (in place) and return it."""
    from .models.resnet import ResNet
    from .models.mobilenet_v2 import MobileNet_v2
    from .models.mobilenet import MobileNet
    from . import lib
    lib.load()  # fail loudly when the CUDA extension is missing
    if not torch.cuda.is_available():
        raise B200Error('convert_b200 needs a CUDA device: the B200 path has no CPU fallback')
    device = torch.device(device if device is not None else 'cuda:%d' % torch.cuda.current_device())
    if getattr(model, '_b200', None) is not None:
        return model
    if isinstance(model, ResNet):
        rt = ResNetRuntime(model, device)
    elif isinstance(model, MobileNet_v2):
        rt = MobileNetRuntime(model, device)
    elif isinstance(model, MobileNet):
        rt = MobileNetV1Runtime(model, device)
    else:
        raise B200Error('no B200 runtime for model type %s yet' % type(model).__name__)
    object.__setattr__(model, '_b200', rt)
    # checkpoints load into the fp32 masters (arena views); refresh the bf16 compute shadow afterwards
    model.register_load_state_dict_post_hook(lambda module, incompatible: rt.arena.sync_shadow())
    return model
