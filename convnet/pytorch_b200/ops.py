"""Tensor-level wrappers over the C ABI (one Python function per entry point of include/b200conv.h).

Tensors are torch CUDA tensors used purely as device-memory handles: activations are contiguous
[N,H,W,C] bf16, conv weights [K, R*S, C] bf16, statistics / master weights / gradients fp32.
Every call is asynchronous on the current torch CUDA stream.
"""
import ctypes

import torch

from . import lib as _l
from .lib import ACT_NONE, ACT_RELU, ACT_RELU6, ConvDesc, Epilogue  # noqa: F401

bf16 = torch.bfloat16


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- optional per-call device timing (bench.py's kernel-class breakdown): CUDA events on the launch stream
_TIMING = None


class _T(object):
    __slots__ = ('name', 'flops', 'nbytes', 'e0')

    def __init__(self, name, flops=0, nbytes=0):
        self.name, self.flops, self.nbytes = name, flops, nbytes

    def __enter__(self):
        if _TIMING is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if _TIMING is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            _TIMING.append((self.name, self.flops, self.nbytes, self.e0, e1))
        return False


def start_timing():
    global _TIMING
    _TIMING = []


def stop_timing():
    """-> {class: {'ms', 'calls', 'flops', 'bytes'}} for the calls since start_timing()."""
    global _TIMING
    rec, _TIMING = _TIMING, None
    torch.cuda.synchronize()
    out = {}
    for name, flops, nbytes, e0, e1 in rec or []:
        c = out.setdefault(name, {'ms': 0.0, 'calls': 0, 'flops': 0, 'bytes': 0})
        c['ms'] += e0.elapsed_time(e1)
        c['calls'] += 1
        c['flops'] += flops
        c['bytes'] += nbytes
    return out


def _conv_flops(d):
    """ALGORITHMIC FLOPs of the convolution the reference runs (bench.py's roofline numerators): descriptors of
    padded / re-laid problems (space-to-depth stem 7x7x3 -> 4x4x16, class count padded to 8, grouped convolutions
    executed on a block-diagonal dense weight) carry the true MACs per output pixel in ``algo_macs``."""
    macs = getattr(d, 'algo_macs', None)
    if macs is None:
        macs = d.K * d.R * d.S * d.C
    return 2 * d.N * d.P * d.Q * macs


def _conv_bytes(x, w, out, residual=None):
    """ALGORITHMIC bytes of one convolution launch: every operand tensor once (input, weights, output, residual)."""
    n = x.numel() * x.element_size() + w.numel() * w.element_size() + out.numel() * out.element_size()
    if residual is not None:
        n += residual.numel() * residual.element_size()
    return n


def _chk(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise _l.B200Error("%s must be a CUDA tensor (no CPU fallback exists)" % name)
    if t.dtype != dtype:
        raise _l.B200Error("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise _l.B200Error("%s must be contiguous" % name)


def out_size(h, r, stride, pad_lo, pad_hi=None):
    pad_hi = pad_lo if pad_hi is None else pad_hi
    return (h + pad_lo + pad_hi - r) // stride + 1


def make_desc(N, H, W, C, K, R, S, stride, pad, P=None, Q=None, x_strides=(0, 0, 0), algo_macs=None, window=0):
    pad_h, pad_w = (pad, pad) if isinstance(pad, int) else pad
    P = out_size(H, R, stride, pad_h) if P is None else P
    Q = out_size(W, S, stride, pad_w) if Q is None else Q
    d = ConvDesc(N, H, W, C, K, R, S, stride, pad_h, pad_w, P, Q, *x_strides, int(window))
    if algo_macs is not None:
        d.algo_macs = int(algo_macs)      # python-side annotation only (not part of the C struct)
    return d


# ------------------------------------------------------------------------------------ convolution
def can_fuse_bn_stats(K):
    """b200_conv_fprop can accumulate BN statistics in its epilogue for this K on every path it may take.  The halo
    kernel (3x3 stride 1, conv3x3.cu) splits K into equal 64/128/256-wide tiles and is the stricter of the two; the
    implicit-GEMM kernel (conv.cu) accepts any K % 64 == 0."""
    n_tiles = (K + 255) // 256
    block_n = ((K + n_tiles - 1) // n_tiles + 15) // 16 * 16
    return K % 64 == 0 and K % block_n == 0 and 256 % block_n == 0


def conv_fprop(x, w, desc, out=None, bias=None, residual=None, act=ACT_NONE, out_fp32=False, bn_stats_ws=None):
    """x [N,H,W,C] bf16, w [K,R*S,C] bf16 -> y [N,P,Q,K] (bf16, or fp32 if out_fp32).
    bn_stats_ws: BN workspace into which the epilogue accumulates per-channel sum / sum^2 (finish: bn_finalize)."""
    _chk(x, bf16, "x"); _chk(w, bf16, "w"); _chk(bias, torch.float32, "bias"); _chk(residual, bf16, "residual")
    if out is None:
        out = torch.empty((desc.N, desc.P, desc.Q, desc.K), device=x.device,
                          dtype=torch.float32 if out_fp32 else bf16)
    ep = Epilogue(_l.ptr(bias), _l.ptr(residual), int(act), int(bool(out_fp32)), _l.ptr(bn_stats_ws))
    with _T('conv_fprop', _conv_flops(desc), _conv_bytes(x, w, out, residual)):
        _l.check(_l.load().b200_conv_fprop(ctypes.byref(desc), x.data_ptr(), w.data_ptr(), out.data_ptr(),
                                           ctypes.byref(ep), _stream()), "b200_conv_fprop")
    return out


def conv_dgrad(dy, wt, desc, out=None, residual=None):
    """dy [N,P,Q,K] bf16, wt [C,R*S,K] bf16 -> dx [N,H,W,C] bf16 (+ residual)."""
    _chk(dy, bf16, "dy"); _chk(wt, bf16, "wt"); _chk(residual, bf16, "residual")
    if out is None:
        out = torch.empty((desc.N, desc.H, desc.W, desc.C), device=dy.device, dtype=bf16)
    with _T('conv_dgrad', _conv_flops(desc), _conv_bytes(dy, wt, out, residual)):
        _l.check(_l.load().b200_conv_dgrad(ctypes.byref(desc), dy.data_ptr(), wt.data_ptr(), out.data_ptr(),
                                           _l.ptr(residual), _stream()), "b200_conv_dgrad")
    return out


_WGRAD_WS = {}


def _wgrad_workspace(device):
    """per-device split-K scratch (allocated once; the library states its size)."""
    ws = _WGRAD_WS.get(device)
    if ws is None:
        ws = torch.empty(int(_l.load().b200_conv_wgrad_workspace_bytes()), device=device, dtype=torch.uint8)
        _WGRAD_WS[device] = ws
    return ws


def conv_wgrad(x, dy, desc, dw):
    """dw [K,R*S,C] fp32 += dy^T (*) x."""
    _chk(x, bf16, "x"); _chk(dy, bf16, "dy"); _chk(dw, torch.float32, "dw")
    ws = _wgrad_workspace(x.device)
    with _T('conv_wgrad', _conv_flops(desc), _conv_bytes(x, dy, dw)):
        _l.check(_l.load().b200_conv_wgrad(ctypes.byref(desc), x.data_ptr(), dy.data_ptr(), dw.data_ptr(),
                                           ws.data_ptr(), ws.numel(), _stream()), "b200_conv_wgrad")
    return dw


def dwconv_fprop(x, w, desc, out=None):
    _chk(x, bf16, "x"); _chk(w, bf16, "w")
    if out is None:
        out = torch.empty((desc.N, desc.P, desc.Q, desc.K), device=x.device, dtype=bf16)
    with _T('dw_fprop', 0, _conv_bytes(x, w, out)):       # HBM-bound class (name does not start with conv_)
        _l.check(_l.load().b200_dwconv_fprop(ctypes.byref(desc), x.data_ptr(), w.data_ptr(), out.data_ptr(), _stream()),
                 "b200_dwconv_fprop")
    return out


def dwconv_dgrad(dy, w, desc, out=None):
    _chk(dy, bf16, "dy"); _chk(w, bf16, "w")
    if out is None:
        out = torch.empty((desc.N, desc.H, desc.W, desc.C), device=dy.device, dtype=bf16)
    with _T('dw_dgrad', 0, _conv_bytes(dy, w, out)):
        _l.check(_l.load().b200_dwconv_dgrad(ctypes.byref(desc), dy.data_ptr(), w.data_ptr(), out.data_ptr(), _stream()),
                 "b200_dwconv_dgrad")
    return out


def dwconv_wgrad(x, dy, desc, dw, workspace):
    _chk(x, bf16, "x"); _chk(dy, bf16, "dy"); _chk(dw, torch.float32, "dw"); _chk(workspace, torch.float32, "ws")
    with _T('dw_wgrad', 0, _conv_bytes(x, dy, dw)):
        _l.check(_l.load().b200_dwconv_wgrad(ctypes.byref(desc), x.data_ptr(), dy.data_ptr(), dw.data_ptr(),
                                             workspace.data_ptr(), workspace.numel() * 4, _stream()), "b200_dwconv_wgrad")
    return dw


# ------------------------------------------------------------------------------------ batch norm
def bn_workspace_floats(C):
    return int(_l.load().b200_bn_workspace_floats(int(C)))


def bn_act_mask_bytes(M, C):
    """bytes of the 1-bit activation mask of an [M, C] tensor (rows padded to 8: the kernels read whole row-quad words)"""
    return (int(M) + 7) // 8 * 8 * (int(C) // 8)


def bn_stats(z, gamma, beta, eps, momentum, running_mean, running_var, nbt, mean, invstd, scale, shift, workspace):
    C = z.shape[-1]
    M = z.numel() // C
    _chk(z, bf16, "z")
    mom = -1.0 if momentum is None else float(momentum)
    with _T('bn_stats', 0, 2 * z.numel()):
        _l.check(_l.load().b200_bn_stats(z.data_ptr(), M, C, _l.ptr(gamma), _l.ptr(beta), float(eps), mom,
                                         _l.ptr(running_mean), _l.ptr(running_var), _l.ptr(nbt), mean.data_ptr(),
                                         invstd.data_ptr(), scale.data_ptr(), shift.data_ptr(), workspace.data_ptr(),
                                         _stream()), "b200_bn_stats")


def bn_finalize(M, C, gamma, beta, eps, momentum, running_mean, running_var, nbt, mean, invstd, scale, shift, workspace):
    mom = -1.0 if momentum is None else float(momentum)
    with _T('bn_stats', 0, 0):
        _l.check(_l.load().b200_bn_finalize(int(M), int(C), _l.ptr(gamma), _l.ptr(beta), float(eps), mom,
                                            _l.ptr(running_mean), _l.ptr(running_var), _l.ptr(nbt), mean.data_ptr(),
                                            invstd.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                            workspace.data_ptr(), _stream()), "b200_bn_finalize")


def bn_eval_coeffs(gamma, beta, running_mean, running_var, eps, scale, shift):
    C = running_mean.numel()
    _l.check(_l.load().b200_bn_eval_coeffs(C, _l.ptr(gamma), _l.ptr(beta), running_mean.data_ptr(),
                                           running_var.data_ptr(), float(eps), scale.data_ptr(), shift.data_ptr(),
                                           _stream()), "b200_bn_eval_coeffs")


def bn_apply(z, scale, shift, act=ACT_NONE, residual=None, z2=None, scale2=None, shift2=None, out=None, act_mask=None):
    """act_mask: optional uint8 tensor of z.numel()/8 bytes receiving one act'(.) bit per element (bn_bwd_* read it
    instead of y)."""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(z, bf16, "z"); _chk(residual, bf16, "residual"); _chk(z2, bf16, "z2"); _chk(act_mask, torch.uint8, "act_mask")
    if act_mask is not None and act_mask.numel() != bn_act_mask_bytes(M, C):
        raise _l.B200Error("act_mask must hold bn_act_mask_bytes(M, C) bytes")
    if out is None:
        out = torch.empty_like(z)
    with _T('bn_apply', 0, 2 * z.numel() * (2 + (residual is not None) + (z2 is not None))):
        _l.check(_l.load().b200_bn_apply(z.data_ptr(), M, C, scale.data_ptr(), shift.data_ptr(), _l.ptr(residual),
                                         _l.ptr(z2), _l.ptr(scale2), _l.ptr(shift2), int(act), out.data_ptr(),
                                         _l.ptr(act_mask), _stream()),
                 "b200_bn_apply")
    return out


def bn_bwd_reduce(dy, y, z, act, mean, invstd, gamma, beta, sums, dgamma_acc, dbeta_acc, workspace, act_mask=None):
    """y=None and act_mask=None: the activation mask is recomputed from z (valid when nothing was added before the
    activation); act_mask (bits written by bn_apply) takes precedence over y."""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(dy, bf16, "dy"); _chk(y, bf16, "y"); _chk(z, bf16, "z"); _chk(act_mask, torch.uint8, "act_mask")
    with _T('bn_bwd_reduce', 0, 2 * z.numel() * (2 + (y is not None and act_mask is None))):
        _l.check(_l.load().b200_bn_bwd_reduce(dy.data_ptr(), _l.ptr(y), _l.ptr(act_mask), z.data_ptr(), M, C, int(act),
                                              mean.data_ptr(),
                                              invstd.data_ptr(), _l.ptr(gamma), _l.ptr(beta), sums.data_ptr(),
                                              _l.ptr(dgamma_acc), _l.ptr(dbeta_acc), workspace.data_ptr(), _stream()),
                 "b200_bn_bwd_reduce")


def bn_bwd_dx(dy, y, z, act, mean, invstd, gamma, beta, sums, dz=None, g_out=None, act_mask=None):
    C = z.shape[-1]
    M = z.numel() // C
    if dz is None:
        dz = torch.empty_like(z)
    with _T('bn_bwd_dx', 0, 2 * z.numel() * (3 + (y is not None and act_mask is None) + (g_out is not None))):
        _l.check(_l.load().b200_bn_bwd_dx(dy.data_ptr(), _l.ptr(y), _l.ptr(act_mask), z.data_ptr(), M, C, int(act),
                                          mean.data_ptr(),
                                          invstd.data_ptr(), _l.ptr(gamma), _l.ptr(beta), sums.data_ptr(),
                                          dz.data_ptr(), _l.ptr(g_out), _stream()), "b200_bn_bwd_dx")
    return dz


# ------------------------------------------------------------------------------------ L1 batch norm
def bn_l1_stats(z, gamma, beta, eps, momentum, running_mean, running_var, mean, invstd, sign_sum, scale, shift,
                workspace):
    """L1 batch statistics of z [.., C]: mean, invstd = s = 1/(mean|z-mean|*sqrt(pi/2) + eps), sign_sum =
    sum sign(z - mean), scale/shift for bn_apply; running buffers (optional) updated with the reference's momentum
    convention.  Two reads of z."""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(z, bf16, "z")
    with _T('bn_l1_stats', 0, 2 * 2 * z.numel()):
        _l.check(_l.load().b200_bn_l1_stats(z.data_ptr(), M, C, _l.ptr(gamma), _l.ptr(beta), float(eps),
                                            float(momentum), _l.ptr(running_mean), _l.ptr(running_var),
                                            mean.data_ptr(), invstd.data_ptr(), sign_sum.data_ptr(), scale.data_ptr(),
                                            shift.data_ptr(), workspace.data_ptr(), _stream()), "b200_bn_l1_stats")


def bn_l1_eval_coeffs(gamma, beta, running_mean, running_var, scale, shift):
    """eval-mode L1 BN: scale = gamma * running_var (the running scale s), shift = beta - running_mean * scale."""
    C = running_mean.numel()
    _l.check(_l.load().b200_bn_l1_eval_coeffs(C, _l.ptr(gamma), _l.ptr(beta), running_mean.data_ptr(),
                                              running_var.data_ptr(), scale.data_ptr(), shift.data_ptr(), _stream()),
             "b200_bn_l1_eval_coeffs")


def bn_l1_bwd_dx(dy, y, z, act, mean, invstd, sign_sum, gamma, beta, sums, dz=None, g_out=None, act_mask=None):
    """L1 BN input gradient; sums from bn_bwd_reduce called with invstd = s.  y / act_mask / g_out as bn_bwd_dx."""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(dy, bf16, "dy"); _chk(y, bf16, "y"); _chk(z, bf16, "z"); _chk(act_mask, torch.uint8, "act_mask")
    if dz is None:
        dz = torch.empty_like(z)
    with _T('bn_l1_bwd_dx', 0, 2 * z.numel() * (3 + (y is not None and act_mask is None) + (g_out is not None))):
        _l.check(_l.load().b200_bn_l1_bwd_dx(dy.data_ptr(), _l.ptr(y), _l.ptr(act_mask), z.data_ptr(), M, C, int(act),
                                             mean.data_ptr(), invstd.data_ptr(), sign_sum.data_ptr(), _l.ptr(gamma),
                                             _l.ptr(beta), sums.data_ptr(), dz.data_ptr(), _l.ptr(g_out), _stream()),
                 "b200_bn_l1_bwd_dx")
    return dz


# ------------------------------------------------------------------------------------ dropout in residual blocks
def dropout_threshold(p):
    """(T, c) of dropout rate 0 <= p < 1: an element is kept iff its 16-bit Philox uniform is < T = round((1-p)*65536)
    (computed in double; keep probability T/65536), and kept values are scaled by c = fp32(1/(1-p)) as in torch."""
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise _l.B200Error('dropout rate must be in [0, 1), got %r' % p)
    return int(round((1.0 - p) * 65536.0)), float(ctypes.c_float(1.0 / (1.0 - p)).value)


def bn_apply_dropout(z, scale, shift, key, layer, p, act_mask, out=None):
    """y = dropout(relu(z*scale + shift)) with the Philox mask of (key, layer) (csrc/dropout.cu); act_mask receives
    keep && pre > 0 for bn_bwd_*_dropout.  key: int64 device tensor of one element, read by the kernel."""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(z, bf16, "z"); _chk(key, torch.int64, "key"); _chk(act_mask, torch.uint8, "act_mask")
    if act_mask is None or act_mask.numel() != bn_act_mask_bytes(M, C):
        raise _l.B200Error("act_mask must hold bn_act_mask_bytes(M, C) bytes")
    T, c = dropout_threshold(p)
    if out is None:
        out = torch.empty_like(z)
    with _T('bn_apply_dropout', 0, 2 * 2 * z.numel() + act_mask.numel()):
        _l.check(_l.load().b200_bn_apply_dropout(z.data_ptr(), M, C, scale.data_ptr(), shift.data_ptr(), key.data_ptr(),
                                                 int(layer), T, c, out.data_ptr(), act_mask.data_ptr(), _stream()),
                 "b200_bn_apply_dropout")
    return out


def bn_bwd_reduce_dropout(dy, z, act_mask, p, mean, invstd, sums, dgamma_acc, dbeta_acc, workspace):
    """bn_bwd_reduce of a bn_apply_dropout unit: g = bit ? dy*c : 0"""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(dy, bf16, "dy"); _chk(z, bf16, "z"); _chk(act_mask, torch.uint8, "act_mask")
    _, c = dropout_threshold(p)
    with _T('bn_bwd_reduce_dropout', 0, 2 * 2 * z.numel() + act_mask.numel()):
        _l.check(_l.load().b200_bn_bwd_reduce_dropout(dy.data_ptr(), act_mask.data_ptr(), z.data_ptr(), M, C, c,
                                                      mean.data_ptr(), invstd.data_ptr(), sums.data_ptr(),
                                                      _l.ptr(dgamma_acc), _l.ptr(dbeta_acc), workspace.data_ptr(),
                                                      _stream()), "b200_bn_bwd_reduce_dropout")


def bn_bwd_dx_dropout(dy, z, act_mask, p, mean, invstd, gamma, sums, dz=None):
    """bn_bwd_dx of a bn_apply_dropout unit: g = bit ? dy*c : 0"""
    C = z.shape[-1]
    M = z.numel() // C
    _chk(dy, bf16, "dy"); _chk(z, bf16, "z"); _chk(act_mask, torch.uint8, "act_mask")
    _, c = dropout_threshold(p)
    if dz is None:
        dz = torch.empty_like(z)
    with _T('bn_bwd_dx_dropout', 0, 2 * 3 * z.numel() + act_mask.numel()):
        _l.check(_l.load().b200_bn_bwd_dx_dropout(dy.data_ptr(), act_mask.data_ptr(), z.data_ptr(), M, C, c,
                                                  mean.data_ptr(), invstd.data_ptr(), _l.ptr(gamma), sums.data_ptr(),
                                                  dz.data_ptr(), _stream()), "b200_bn_bwd_dx_dropout")
    return dz


# ------------------------------------------------------------------------------------ pooling
def _out(out, shape, dtype, device, name):
    """a caller-supplied output (checked: dtype, contiguity, shape) or a new tensor"""
    if out is None:
        return torch.empty(shape, device=device, dtype=dtype)
    _chk(out, dtype, name)
    if tuple(out.shape) != tuple(shape):
        raise _l.B200Error("%s has shape %s, expected %s" % (name, tuple(out.shape), tuple(shape)))
    return out


def maxpool_fwd(x, want_argmax=True, out=None, argmax_out=None):
    N, H, W, C = x.shape
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = _out(out, (N, OH, OW, C), bf16, x.device, "out")
    am = _out(argmax_out, (N, OH, OW, C), torch.uint8, x.device, "argmax_out") if want_argmax else None
    with _T('maxpool_fwd', 0, 2 * x.numel() + 3 * y.numel()):
        _l.check(_l.load().b200_maxpool3x3s2_fwd(x.data_ptr(), N, H, W, C, y.data_ptr(), _l.ptr(am), _stream()),
                 "b200_maxpool3x3s2_fwd")
    return y, am


def maxpool_bwd(dy, argmax, in_shape, out=None):
    N, H, W, C = in_shape
    dx = _out(out, in_shape, bf16, dy.device, "out")
    with _T('maxpool_bwd', 0, 2 * dx.numel() + 3 * dy.numel()):
        _l.check(_l.load().b200_maxpool3x3s2_bwd(dy.data_ptr(), argmax.data_ptr(), N, H, W, C, dx.data_ptr(), _stream()),
                 "b200_maxpool3x3s2_bwd")
    return dx


def bn_apply_maxpool(z, scale, shift, act=ACT_RELU, want_argmax=True, out=None, argmax_out=None):
    """maxpool3x3s2(bf16(act(z*scale+shift))) in one pass (the ImageNet stem tail); returns (pooled, argmax bytes)."""
    N, H, W, C = z.shape
    _chk(z, bf16, "z")
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    y = _out(out, (N, OH, OW, C), bf16, z.device, "out")
    am = _out(argmax_out, (N, OH, OW, C), torch.uint8, z.device, "argmax_out") if want_argmax else None
    with _T('bn_apply', 0, 2 * z.numel() + 3 * y.numel()):
        _l.check(_l.load().b200_bn_apply_maxpool3x3s2(z.data_ptr(), N, H, W, C, scale.data_ptr(), shift.data_ptr(),
                                                      int(act), y.data_ptr(), _l.ptr(am), _stream()),
                 "b200_bn_apply_maxpool3x3s2")
    return y, am


def avgpool_fwd(x, out=None):
    N, H, W, C = x.shape
    y = _out(out, (N, 1, 1, C), bf16, x.device, "out")
    with _T('avgpool', 0, 2 * x.numel()):
        _l.check(_l.load().b200_avgpool_fwd(x.data_ptr(), N, H * W, C, y.data_ptr(), _stream()), "b200_avgpool_fwd")
    return y


def avgpool_bwd(dy, in_shape, out=None):
    N, H, W, C = in_shape
    dx = _out(out, in_shape, bf16, dy.device, "out")
    with _T('avgpool', 0, 2 * dx.numel()):
        _l.check(_l.load().b200_avgpool_bwd(dy.data_ptr(), N, H * W, C, dx.data_ptr(), _stream()), "b200_avgpool_bwd")
    return dx


# ------------------------------------------------------------------------------------ squeeze-and-excitation
def se_pool(r, out=None):
    N, H, W, C = r.shape
    out = _out(out, (N, 1, 1, C), bf16, r.device, "out")
    with _T('se', 0, 2 * r.numel()):
        _l.check(_l.load().b200_se_pool(r.data_ptr(), N, H * W, C, out.data_ptr(), _stream()), "b200_se_pool")
    return out


def se_scale_fwd(r, logit, out=None):
    N, H, W, C = r.shape
    _chk(logit, torch.float32, "logit")
    out = _out(out, r.shape, bf16, r.device, "out")
    with _T('se', 0, 4 * r.numel()):
        _l.check(_l.load().b200_se_scale_fwd(r.data_ptr(), logit.data_ptr(), N, H * W, C, out.data_ptr(), _stream()),
                 "b200_se_scale_fwd")
    return out


def se_bwd_reduce(g, r, logit, out=None):
    N, H, W, C = r.shape
    out = _out(out, (N, 1, 1, C), bf16, r.device, "out")
    with _T('se', 0, 4 * r.numel()):
        _l.check(_l.load().b200_se_bwd_reduce(g.data_ptr(), r.data_ptr(), logit.data_ptr(), N, H * W, C, out.data_ptr(),
                                              _stream()), "b200_se_bwd_reduce")
    return out


def se_bwd_dx(g, logit, dmean, out=None):
    N, H, W, C = g.shape
    out = _out(out, g.shape, bf16, g.device, "out")
    with _T('se', 0, 4 * g.numel()):
        _l.check(_l.load().b200_se_bwd_dx(g.data_ptr(), logit.data_ptr(), dmean.data_ptr(), N, H * W, C, out.data_ptr(),
                                          _stream()), "b200_se_bwd_dx")
    return out


def act_bwd(dy, y, act, out=None):
    out = _out(out, dy.shape, bf16, dy.device, "out")
    _l.check(_l.load().b200_act_bwd(dy.data_ptr(), y.data_ptr(), dy.numel(), int(act), out.data_ptr(), _stream()),
             "b200_act_bwd")
    return out


# ------------------------------------------------------------------------------------ layout / casts
class Mix(object):
    """Device-side draws of one MixUp / CutMix step for the mixing kernels: ``perm`` int64 [N], ``params`` the
    b200_mix_params block (int32 [5] on the device: lambda as fp32 bits, then r0, r1, c0, c1), ``kind`` MIX_MIXUP or
    MIX_CUTMIX.  The kernels read perm and params at run time, so a captured graph follows new values in place."""
    __slots__ = ('perm', 'params', 'kind')

    def __init__(self, perm, params, kind):
        self.perm, self.params, self.kind = perm, params, int(kind)

    @property
    def lam(self):
        """fp32 [1] device view of lambda (the first field of the parameter block)."""
        return self.params[:1].view(torch.float32)


def _check_mix(mix, n):
    _chk(mix.perm, torch.int64, "perm"); _chk(mix.params, torch.int32, "mix params")
    if mix.perm.numel() != n or mix.params.numel() < 5 or mix.kind not in (_l.MIX_MIXUP, _l.MIX_CUTMIX):
        raise _l.B200Error("mix: perm must have one entry per sample, params 5 int32, kind MIXUP or CUTMIX")


def _prep_out(N, H, W, cpad, s2d, border, device, out):
    if s2d and border:
        shape = (N, H // 2 + 3, W // 2 + 3, cpad)
    else:
        shape = (N, H // 2, W // 2, cpad) if s2d else (N, H, W, cpad)
    if out is None:
        return torch.empty(shape, device=device, dtype=bf16)
    _chk(out, bf16, "out")
    if tuple(out.shape) != shape:
        raise _l.B200Error("input_prep: out has shape %s, expected %s" % (tuple(out.shape), shape))
    return out


def input_prep(x_nchw, cpad, s2d=False, border=False, mix=None, out=None):
    """NCHW fp32 -> NHWC bf16 (channels zero-padded to cpad) or its 2x2 space-to-depth form (optionally with
    the physical zero border of mode 2: +2 low / +1 high in H and W).  ``mix`` (a Mix): MixUp / CutMix in the pass."""
    _chk(x_nchw, torch.float32, "x")
    N, C, H, W = x_nchw.shape
    out = _prep_out(N, H, W, cpad, s2d, border, x_nchw.device, out)
    mode = (2 if border else 1) if s2d else 0
    if mix is None:
        with _T('input_prep', 0, 4 * x_nchw.numel() + 2 * out.numel()):
            _l.check(_l.load().b200_input_prep(x_nchw.data_ptr(), N, C, H, W, cpad, mode, out.data_ptr(),
                                               _stream()), "b200_input_prep")
        return out
    _check_mix(mix, N)
    reads = 2 if mix.kind == _l.MIX_MIXUP else 1
    with _T('input_prep', 0, 4 * reads * x_nchw.numel() + 2 * out.numel()):
        _l.check(_l.load().b200_input_prep_mix(x_nchw.data_ptr(), N, C, H, W, cpad, mode, mix.perm.data_ptr(),
                                               mix.params.data_ptr(), mix.kind, out.data_ptr(), _stream()),
                 "b200_input_prep_mix")
    return out


def u8_norm_coeffs(mean, std):
    """fp32 scale / bias of the uint8 normalisation: value = u8 * scale + bias = (u8/255 - mean)/std."""
    scale = [1.0 / (255.0 * float(s)) for s in std]
    bias = [-float(m) / float(s) for m, s in zip(mean, std)]
    return scale, bias


def input_prep_u8(x_nhwc_u8, cpad, mean, std, s2d=False, border=False, mix=None, out=None):
    """uint8 NHWC [N,H,W,C] -> the layouts of input_prep, normalised as (u8/255 - mean)/std in the same pass."""
    _chk(x_nhwc_u8, torch.uint8, "x")
    N, H, W, C = x_nhwc_u8.shape
    out = _prep_out(N, H, W, cpad, s2d, border, x_nhwc_u8.device, out)
    sc, bi = u8_norm_coeffs(mean, std)
    scale = (ctypes.c_float * C)(*sc)
    bias = (ctypes.c_float * C)(*bi)
    mode = (2 if border else 1) if s2d else 0
    if mix is None:
        with _T('input_prep', 0, x_nhwc_u8.numel() + 2 * out.numel()):
            _l.check(_l.load().b200_input_prep_u8(x_nhwc_u8.data_ptr(), N, C, H, W, cpad, mode, scale, bias,
                                                  out.data_ptr(), _stream()), "b200_input_prep_u8")
        return out
    _check_mix(mix, N)
    reads = 2 if mix.kind == _l.MIX_MIXUP else 1
    with _T('input_prep', 0, reads * x_nhwc_u8.numel() + 2 * out.numel()):
        _l.check(_l.load().b200_input_prep_u8_mix(x_nhwc_u8.data_ptr(), N, C, H, W, cpad, mode, scale, bias,
                                                  mix.perm.data_ptr(), mix.params.data_ptr(), mix.kind, out.data_ptr(),
                                                  _stream()), "b200_input_prep_u8_mix")
    return out


class Aug(object):
    """Device-side draws of one batch-augmentation step (utils/augment.py): ``params`` int16 [N*D, 3 + 4*holes] rows
    {oy, ox, flip, y1, y2, x1, x2, ...}, ``lut`` fp32 [C, 256] (ToTensor + Normalize of each uint8 value), ``duplicates``
    D, ``pad`` the crop padding, ``out_hw`` (OH, OW) when the crop is resized (the Mix&Match CIFAR regimes; None: the
    copies keep the images' size).  The kernel reads params at run time, so a captured graph follows new draws in place.
    ``window`` (p, n): the step trains on rows [p, p + n) of these images' copies (a chunk of a larger batch, see
    row_range); None: on all of them."""
    __slots__ = ('params', 'lut', 'duplicates', 'pad', 'out_hw', 'window')

    def __init__(self, params, lut, duplicates, pad, out_hw=None, window=None):
        self.params, self.lut, self.duplicates, self.pad = params, lut, int(duplicates), int(pad)
        self.out_hw = (int(out_hw[0]), int(out_hw[1])) if out_hw is not None else None
        self.window = window

    @property
    def holes(self):
        return (self.params.shape[-1] - 3) // 4

    @property
    def rows(self):
        return self.window[1] if self.window is not None else self.params.shape[0]

    @property
    def key(self):
        """what a captured step depends on besides the input's shape (the draws are refreshed in place)"""
        return ('aug', tuple(self.params.shape), self.duplicates, self.pad, self.lut.data_ptr(), self.out_hw,
                self.window)

    @property
    def tables(self):
        return (self.params,)

    def with_tables(self, tables):
        return Aug(tables[0], self.lut, self.duplicates, self.pad, self.out_hw, self.window)

    def row_range(self, r0, r1):
        """-> (Aug, b0, b1): rows [r0, r1) of the B*D copies as a step over images [b0, b1) (x_nhwc[b0:b1]), whose
        relayout computes the copies of those whole images and hands on the window of the chunk's rows."""
        b0, b1, p = _image_range(r0, r1, self.duplicates)
        D = self.duplicates
        return Aug(self.params[b0 * D:b1 * D], self.lut, D, self.pad, self.out_hw, (p, r1 - r0)), b0, b1


class Rrc(object):
    """Device-side tables of one resized-crop step (utils/augment.py ResizedCropBatch): ``index`` int64 [B, 3] {byte
    offset, h, w} of each image's region in the uint8 region buffer, ``draws`` int32 [B*D, 5] {y, x, h, w, flip} of each
    copy's crop box inside its region, ``lut`` fp32 [C, 256], ``size`` (OH, OW).  ``host`` holds CPU copies of index and
    draws plus the number of region bytes in use: input_prep_u8_rrc validates them before any launch, without a device
    read-back.  The kernel reads the tables at run time, so a captured graph follows new values in place.
    ``window`` (p, n): as for Aug."""
    __slots__ = ('index', 'draws', 'lut', 'duplicates', 'size', 'host', 'window')

    def __init__(self, index, draws, lut, duplicates, size, host, window=None):
        self.index, self.draws, self.lut, self.duplicates = index, draws, lut, int(duplicates)
        self.size, self.host = (int(size[0]), int(size[1])), host
        self.window = window

    @property
    def rows(self):
        return self.window[1] if self.window is not None else self.draws.shape[0]

    @property
    def key(self):
        return ('rrc', tuple(self.index.shape), self.duplicates, self.size, self.lut.data_ptr(), self.window)

    @property
    def tables(self):
        return (self.index, self.draws)

    def with_tables(self, tables):
        return Rrc(tables[0], tables[1], self.lut, self.duplicates, self.size, self.host, self.window)

    def row_range(self, r0, r1):
        """-> (Rrc, b0, b1): rows [r0, r1) of the B*D crops as a step over the regions of images [b0, b1) (the region
        buffer is shared: the index holds absolute offsets); see Aug.row_range."""
        b0, b1, p = _image_range(r0, r1, self.duplicates)
        D = self.duplicates
        h_index, h_draws, nbytes = self.host
        return Rrc(self.index[b0:b1], self.draws[b0 * D:b1 * D], self.lut, D, self.size,
                   (h_index[b0:b1], h_draws[b0 * D:b1 * D], nbytes), (p, r1 - r0)), b0, b1


def chunk_rows(rows, chunks):
    """[(r0, r1), ...]: the row ranges of torch.chunk(chunks) over ``rows`` rows -- ceil(rows / chunks) rows each, the
    last one fewer, and fewer than ``chunks`` ranges when the rows run out first."""
    if rows < 1 or chunks < 1:
        raise ValueError('chunk_rows: rows and chunks must be >= 1; got %d, %d' % (rows, chunks))
    step = -(-rows // chunks)
    return [(r, min(r + step, rows)) for r in range(0, rows, step)]


def _image_range(r0, r1, D):
    """rows [r0, r1) of a batch whose image b owns rows [b*D, (b+1)*D) -> (b0, b1, p): the images [b0, b1) that cover
    them and the offset p of row r0 in their rows.  A chunk boundary may split one image's copies: both chunks then
    compute that image's D copies and each keeps its own (at most 2 (D - 1) extra rows per chunk)."""
    if not 0 <= r0 < r1:
        raise _l.B200Error('row range [%d, %d) is empty' % (r0, r1))
    b0, b1 = r0 // D, -(-r1 // D)
    return b0, b1, r0 - b0 * D


def check_rrc_tables(index, draws, nbytes, C, D):
    """Host-side validation of resized-crop tables (CPU int64 [B, 3] index, int32 [B*D, 5] draws): every region lies
    inside the first ``nbytes`` bytes of the buffer and every crop box inside its region.  Raises B200Error."""
    if index.dim() != 2 or index.shape[1] != 3 or draws.dim() != 2 or draws.shape[1] != 5 \
            or draws.shape[0] != index.shape[0] * D:
        raise _l.B200Error("input_prep_u8_rrc: index must be [B, 3] and draws [B*D, 5]; got %s, %s (D=%d)"
                           % (tuple(index.shape), tuple(draws.shape), D))
    off, h, w = (index[:, k].long() for k in range(3))
    if bool(((off < 0) | (h < 1) | (w < 1) | (h > 65535) | (w > 65535) | (off + h * w * C > nbytes)).any()):
        raise _l.B200Error("input_prep_u8_rrc: a region lies outside the %d-byte buffer" % nbytes)
    d = draws.long()
    rh, rw = h.repeat_interleave(D), w.repeat_interleave(D)
    if bool(((d[:, 0] < 0) | (d[:, 1] < 0) | (d[:, 2] < 1) | (d[:, 3] < 1) | (d[:, 0] + d[:, 2] > rh)
             | (d[:, 1] + d[:, 3] > rw) | (d[:, 4] < 0) | (d[:, 4] > 1)).any()):
        raise _l.B200Error("input_prep_u8_rrc: a crop box lies outside its region")


def input_prep_u8_rrc(regions, cpad, rrc, s2d=False, border=False, out=None):
    """uint8 region buffer -> bf16 [B*D, OH, OW, cpad] (or the bordered space-to-depth layout): RandomResizedCrop with
    Pillow's bilinear resample, flip and normalisation through rrc.lut; row b*D + d = copy d of image b.  With
    rrc.window = (p, n): rows [p, p + n) of that output."""
    _chk(regions, torch.uint8, "regions"); _chk(rrc.index, torch.int64, "index"); _chk(rrc.draws, torch.int32, "draws")
    _chk(rrc.lut, torch.float32, "lut")
    if s2d and not border:
        raise _l.B200Error("input_prep_u8_rrc: the space-to-depth layout needs the border (mode 2)")
    if regions.dim() != 1 or rrc.lut.dim() != 2 or rrc.lut.shape[1] != 256:
        raise _l.B200Error("input_prep_u8_rrc: regions must be a flat uint8 buffer and lut fp32 [C, 256]")
    C, D = rrc.lut.shape[0], rrc.duplicates
    (OH, OW), B = rrc.size, rrc.index.shape[0]
    h_index, h_draws, nbytes = rrc.host
    if nbytes > regions.numel() or tuple(h_index.shape) != tuple(rrc.index.shape) \
            or tuple(h_draws.shape) != tuple(rrc.draws.shape):
        raise _l.B200Error("input_prep_u8_rrc: host tables do not describe the device tables and buffer")
    check_rrc_tables(h_index, h_draws, nbytes, C, D)
    out = _prep_out(B * D, OH, OW, cpad, s2d, border, regions.device, out)
    mode = 2 if s2d else 0
    nbytes_read = int((h_index[:, 1].long() * h_index[:, 2].long()).sum()) * C
    with _T('input_prep', 0, nbytes_read + 8 * rrc.index.numel() + 4 * rrc.draws.numel() + 2 * out.numel()):
        _l.check(_l.load().b200_input_prep_u8_rrc(regions.data_ptr(), regions.numel(), rrc.index.data_ptr(),
                                                  rrc.draws.data_ptr(), B, D, C, OH, OW, cpad, mode,
                                                  rrc.lut.data_ptr(), out.data_ptr(), _stream()),
                 "b200_input_prep_u8_rrc")
    return _window(out, rrc.window)


def _window(out, window):
    """rows [p, p + n) of a relayout output (a contiguous view: rows are its outermost dimension)"""
    if window is None:
        return out
    p, n = window
    if p < 0 or n < 1 or p + n > out.shape[0]:
        raise _l.B200Error('relayout window (%d, %d) outside its %d rows' % (p, n, out.shape[0]))
    return out[p:p + n]


class ScaleCropTables(object):
    """Device-side tables of one scale-crop (evaluation) batch (utils/augment.py ScaleCropBatch): ``index`` int64 [B, 3]
    {byte offset, h, w} of each image's support region in the uint8 region buffer, ``geom`` int32 [B, 8] {y0, x0, H, W,
    RH, RW, top, left}, ``lut`` fp32 [C, 256], ``size`` (OH, OW).  ``host`` holds CPU copies of index and geom plus the
    number of region bytes in use: input_prep_u8_scale_crop validates them before the launch, without a device
    read-back."""
    __slots__ = ('index', 'geom', 'lut', 'size', 'host')

    def __init__(self, index, geom, lut, size, host):
        self.index, self.geom, self.lut = index, geom, lut
        self.size, self.host = (int(size[0]), int(size[1])), host


def check_scale_crop_tables(index, geom, nbytes, C, size):
    """Host-side validation of scale-crop tables (CPU int64 [B, 3] index, int32 [B, 8] geom) for an OH x OW ``size``:
    every region lies inside the first ``nbytes`` bytes of the buffer and inside its image, and covers every source
    pixel the crop window's taps read.  Raises B200Error."""
    from .utils.augment import crop_support
    if index.dim() != 2 or index.shape[1] != 3 or geom.dim() != 2 or geom.shape[1] != 8 \
            or geom.shape[0] != index.shape[0]:
        raise _l.B200Error("input_prep_u8_scale_crop: index must be [B, 3] and geom [B, 8]; got %s, %s"
                           % (tuple(index.shape), tuple(geom.shape)))
    off, h, w = (index[:, k].long() for k in range(3))
    if bool(((off < 0) | (h < 1) | (w < 1) | (h > 65535) | (w > 65535) | (off + h * w * C > nbytes)).any()):
        raise _l.B200Error("input_prep_u8_scale_crop: a region lies outside the %d-byte buffer" % nbytes)
    OH, OW = size
    for b, (y0, x0, H, W, RH, RW, top, left) in enumerate(geom.tolist()):
        rh, rw = int(h[b]), int(w[b])
        if not (1 <= H <= 65535 and 1 <= W <= 65535 and 1 <= RH <= 65535 and 1 <= RW <= 65535):
            raise _l.B200Error("input_prep_u8_scale_crop: image %d has sizes %dx%d -> %dx%d outside 1..65535"
                               % (b, H, W, RH, RW))
        if y0 < 0 or x0 < 0 or y0 + rh > H or x0 + rw > W:
            raise _l.B200Error("input_prep_u8_scale_crop: the region of image %d lies outside its %dx%d image"
                               % (b, H, W))
        for n, nr, start, n_out, lo, ext in ((H, RH, top, OH, y0, rh), (W, RW, left, OW, x0, rw)):
            s = crop_support(n, nr, start, n_out)
            if s is not None and (s[0] < lo or s[1] > lo + ext):
                raise _l.B200Error("input_prep_u8_scale_crop: the region of image %d misses source pixels the crop "
                                   "window reads" % b)


def input_prep_u8_scale_crop(regions, cpad, sc, s2d=False, border=False, out=None):
    """uint8 region buffer -> bf16 [B, OH, OW, cpad] (or the bordered space-to-depth layout): Resize + CenterCrop with
    Pillow's bilinear resample of each whole image, and normalisation through sc.lut (a ScaleCropTables)."""
    _chk(regions, torch.uint8, "regions"); _chk(sc.index, torch.int64, "index"); _chk(sc.geom, torch.int32, "geom")
    _chk(sc.lut, torch.float32, "lut")
    if s2d and not border:
        raise _l.B200Error("input_prep_u8_scale_crop: the space-to-depth layout needs the border (mode 2)")
    if regions.dim() != 1 or sc.lut.dim() != 2 or sc.lut.shape[1] != 256:
        raise _l.B200Error("input_prep_u8_scale_crop: regions must be a flat uint8 buffer and lut fp32 [C, 256]")
    C, (OH, OW), B = sc.lut.shape[0], sc.size, sc.index.shape[0]
    h_index, h_geom, nbytes = sc.host
    if nbytes > regions.numel() or tuple(h_index.shape) != tuple(sc.index.shape) \
            or tuple(h_geom.shape) != tuple(sc.geom.shape):
        raise _l.B200Error("input_prep_u8_scale_crop: host tables do not describe the device tables and buffer")
    check_scale_crop_tables(h_index, h_geom, nbytes, C, sc.size)
    out = _prep_out(B, OH, OW, cpad, s2d, border, regions.device, out)
    mode = 2 if s2d else 0
    nbytes_read = int((h_index[:, 1].long() * h_index[:, 2].long()).sum()) * C
    with _T('input_prep', 0, nbytes_read + 8 * sc.index.numel() + 4 * sc.geom.numel() + 2 * out.numel()):
        _l.check(_l.load().b200_input_prep_u8_scale_crop(regions.data_ptr(), regions.numel(), sc.index.data_ptr(),
                                                         sc.geom.data_ptr(), B, C, OH, OW, cpad, mode,
                                                         sc.lut.data_ptr(), out.data_ptr(), _stream()),
                 "b200_input_prep_u8_scale_crop")
    return out


def input_prep_u8_aug(x_nhwc_u8, cpad, aug, out=None):
    """uint8 NHWC [N,H,W,C] -> bf16 NHWC [N*D, H, W, cpad]: the D augmented copies of every image (crop, flip, Cutout)
    normalised through aug.lut, row n*D + d = copy d of image n.  With aug.out_hw = (OH, OW) every crop is resized
    (Pillow's bilinear resample) before the flip: bf16 [N*D, OH, OW, cpad], Cutout boxes in output coordinates.  With
    aug.window = (p, n): rows [p, p + n) of that output."""
    _chk(x_nhwc_u8, torch.uint8, "x"); _chk(aug.params, torch.int16, "aug params"); _chk(aug.lut, torch.float32, "lut")
    N, H, W, C = x_nhwc_u8.shape
    D = aug.duplicates
    if aug.params.dim() != 2 or aug.params.shape[0] != N * D or (aug.params.shape[1] - 3) % 4 != 0 \
            or tuple(aug.lut.shape) != (C, 256):
        raise _l.B200Error("input_prep_u8_aug: params must be int16 [N*D, 3+4*holes] and lut fp32 [C, 256]; got %s, %s"
                           % (tuple(aug.params.shape), tuple(aug.lut.shape)))
    if aug.out_hw is not None:
        OH, OW = aug.out_hw
        out = _prep_out(N * D, OH, OW, cpad, False, False, x_nhwc_u8.device, out)
        with _T('input_prep', 0, D * x_nhwc_u8.numel() + 2 * aug.params.numel() + 2 * out.numel()):
            _l.check(_l.load().b200_input_prep_u8_aug_resize(x_nhwc_u8.data_ptr(), N, D, C, H, W, OH, OW, cpad, aug.pad,
                                                             aug.lut.data_ptr(), aug.params.data_ptr(), aug.holes,
                                                             out.data_ptr(), _stream()),
                     "b200_input_prep_u8_aug_resize")
        return _window(out, aug.window)
    out = _prep_out(N * D, H, W, cpad, False, False, x_nhwc_u8.device, out)
    with _T('input_prep', 0, x_nhwc_u8.numel() + 2 * aug.params.numel() + 2 * out.numel()):
        _l.check(_l.load().b200_input_prep_u8_aug(x_nhwc_u8.data_ptr(), N, D, C, H, W, cpad, aug.pad,
                                                  aug.lut.data_ptr(), aug.params.data_ptr(), aug.holes,
                                                  out.data_ptr(), _stream()), "b200_input_prep_u8_aug")
    return _window(out, aug.window)


def weight_transpose(w, out=None):
    """bf16 [K,T,C] -> [C,T,K]."""
    K, T, C = w.shape
    if out is None:
        out = torch.empty((C, T, K), device=w.device, dtype=bf16)
    with _T('weight_transpose', 0, 4 * w.numel()):
        _l.check(_l.load().b200_weight_transpose(w.data_ptr(), out.data_ptr(), K, T, C, _stream()),
                 "b200_weight_transpose")
    return out


def transpose_jobs(shapes_and_offsets, device):
    """[(src_off, dst_off, K, T, C), ...] -> (int32 device tensor [n, 6], total_tiles) for weight_transpose_batched."""
    rows, tiles = [], 0
    for src_off, dst_off, K, T, C in shapes_and_offsets:
        rows.append([src_off, dst_off, K, T, C, tiles])
        tiles += T * ((K + 31) // 32) * ((C + 31) // 32)
    return torch.tensor(rows, dtype=torch.int32, device=device), tiles


def weight_transpose_batched(src_base, dst_base, jobs, total_tiles):
    """every job: bf16 [K,T,C] at src_base[src_off:] -> [C,T,K] at dst_base[dst_off:], one launch."""
    _chk(src_base, bf16, "src_base"); _chk(dst_base, bf16, "dst_base"); _chk(jobs, torch.int32, "jobs")
    with _T('weight_transpose', 0, 4 * src_base.numel()):
        _l.check(_l.load().b200_weight_transpose_batched(src_base.data_ptr(), dst_base.data_ptr(), jobs.data_ptr(),
                                                         int(jobs.shape[0]), int(total_tiles), _stream()),
                 "b200_weight_transpose_batched")
    return dst_base


def stem_weight_to_s2d(w_f32, K, C, cpad, out):
    _l.check(_l.load().b200_stem_weight_to_s2d(w_f32.data_ptr(), K, C, cpad, out.data_ptr(), _stream()),
             "b200_stem_weight_to_s2d")
    return out


def stem_wgrad_from_s2d(dw_s2d, K, C, cpad, dw):
    _l.check(_l.load().b200_stem_wgrad_from_s2d(dw_s2d.data_ptr(), K, C, cpad, dw.data_ptr(), _stream()),
             "b200_stem_wgrad_from_s2d")
    return dw


def group_weight_pack(w32_grouped, K, T, C, groups, window, transpose=False, out=None):
    """fp32 [K,T,C/g] -> bf16 [K,T,window] (or [C,T,window] transposed): the block-diagonal operand of a grouped
    convolution at window granularity.  window == C is the dense expansion for any C and K: [K,T,C] (or [C,T,K])."""
    shape = (C, T, K if window == C else window) if transpose else (K, T, window)
    if out is None:
        out = torch.empty(shape, device=w32_grouped.device, dtype=bf16)
    _chk(out, bf16, "out")
    if tuple(out.shape) != shape:
        raise _l.B200Error("group_weight_pack: out must be %s, got %s" % (shape, tuple(out.shape)))
    with _T('weight_transpose', 0, 2 * out.numel()):
        _l.check(_l.load().b200_group_weight_pack(w32_grouped.data_ptr(), K, T, C, groups, int(window), int(bool(transpose)),
                                                  out.data_ptr(), _stream()), "b200_group_weight_pack")
    return out


def group_wgrad_unpack(dw_win, K, T, C, groups, window, dw_grouped):
    with _T('weight_transpose', 0, 4 * dw_grouped.numel()):
        _l.check(_l.load().b200_group_wgrad_unpack(dw_win.data_ptr(), K, T, C, groups, int(window), dw_grouped.data_ptr(),
                                                   _stream()), "b200_group_wgrad_unpack")
    return dw_grouped


def cast_bf16(src, dst):
    with _T('cast', 0, 6 * src.numel()):
        _l.check(_l.load().b200_cast_f32_to_bf16(src.data_ptr(), dst.data_ptr(), src.numel(), _stream()),
                 "b200_cast_f32_to_bf16")
    return dst


# ------------------------------------------------------------------------------------ loss / optimizer
def softmax_ce(logits, target, classes, smooth_eps, loss=None, row_loss=None, dlogits=None, grad_scale=1.0,
               grad_scale_dev=None):
    """logits fp32 [B, ld] (ld >= classes), target int64 [B].  loss fp32[3] (+ row_loss fp32[2B] scratch): mean loss,
    top-1 %, top-5 % -- overwritten; dlogits bf16 [B, ld] = grad_scale * (*grad_scale_dev) / B * dloss/dlogits (pad
    columns zeroed)."""
    if loss is not None and (loss.numel() < 3 or row_loss is None or row_loss.numel() < 2 * logits.shape[0]):
        raise _l.B200Error("softmax_ce: loss needs 3 floats and row_loss 2*B floats")
    B, ld = logits.shape
    _chk(logits, torch.float32, "logits"); _chk(target, torch.int64, "target"); _chk(dlogits, bf16, "dlogits")
    _chk(loss, torch.float32, "loss"); _chk(row_loss, torch.float32, "row_loss")
    _chk(grad_scale_dev, torch.float32, "grad_scale_dev")
    with _T('softmax_ce', 0, 4 * logits.numel()):
        _l.check(_l.load().b200_softmax_ce(logits.data_ptr(), target.data_ptr(), B, int(classes), int(ld),
                                           float(smooth_eps or 0.0), float(grad_scale), _l.ptr(grad_scale_dev),
                                           _l.ptr(loss), _l.ptr(row_loss), _l.ptr(dlogits), _stream()),
                 "b200_softmax_ce")


def softmax_ce_mix(logits, target, mix, classes, loss=None, row_loss=None, dlogits=None, grad_scale=1.0,
                   grad_scale_dev=None):
    """softmax_ce with the soft MixUp / CutMix target lam*onehot(t) + (1-lam)*onehot(t[perm]); ``mix`` is an ops.Mix
    (perm and lambda are read on the device).  Top-1 / top-5 count against ``target`` itself; no label smoothing."""
    if loss is not None and (loss.numel() < 3 or row_loss is None or row_loss.numel() < 2 * logits.shape[0]):
        raise _l.B200Error("softmax_ce_mix: loss needs 3 floats and row_loss 2*B floats")
    B, ld = logits.shape
    _chk(logits, torch.float32, "logits"); _chk(target, torch.int64, "target"); _chk(dlogits, bf16, "dlogits")
    _chk(loss, torch.float32, "loss"); _chk(row_loss, torch.float32, "row_loss")
    _chk(grad_scale_dev, torch.float32, "grad_scale_dev")
    _check_mix(mix, B)
    with _T('softmax_ce', 0, 4 * logits.numel()):
        _l.check(_l.load().b200_softmax_ce_mix(logits.data_ptr(), target.data_ptr(), mix.perm.data_ptr(),
                                               mix.lam.data_ptr(), B, int(classes), int(ld), float(grad_scale),
                                               _l.ptr(grad_scale_dev), _l.ptr(loss), _l.ptr(row_loss), _l.ptr(dlogits),
                                               _stream()), "b200_softmax_ce_mix")


def colsum_bf16(m, out):
    B, K = m.shape
    _l.check(_l.load().b200_colsum_bf16(m.data_ptr(), B, K, out.data_ptr(), _stream()), "b200_colsum_bf16")


def fused_sgd(p32, g32, m32, p16, n, wd_count, lr, momentum, dampening, weight_decay, inv_scale, clip_coef,
              first_step, zero_grad=False):
    with _T('fused_sgd', 0, (26 if zero_grad else 22) * int(n)):   # 12 B read + 10 B written (+4 B memset) per parameter
        _l.check(_l.load().b200_fused_sgd(p32.data_ptr(), g32.data_ptr(), _l.ptr(m32), _l.ptr(p16), int(n),
                                          int(wd_count), float(lr), float(momentum), float(dampening),
                                          float(weight_decay), float(inv_scale), _l.ptr(clip_coef), int(bool(first_step)),
                                          int(bool(zero_grad)), _stream()), "b200_fused_sgd")


def sumsq(g, n, out, workspace):
    _l.check(_l.load().b200_sumsq(g.data_ptr(), int(n), out.data_ptr(), workspace.data_ptr(), _stream()),
             "b200_sumsq")


def grad_coef(sumsq_t, inv_scale, mode, max_norm, momentum, state, coef_out, norm_out):
    _l.check(_l.load().b200_grad_coef(sumsq_t.data_ptr(), float(inv_scale), int(mode), float(max_norm),
                                      float(momentum), _l.ptr(state), coef_out.data_ptr(), _l.ptr(norm_out),
                                      _stream()), "b200_grad_coef")
