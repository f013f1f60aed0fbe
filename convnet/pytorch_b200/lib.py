"""ctypes binding of libb200conv.so (the C ABI declared in include/b200conv.h).

This is the only place the shared library is opened.  There is deliberately no fallback: if the
library is missing or a call fails, a ``B200Error`` is raised (the reference silently relies on
whatever torch dispatches to; see SURVEY.md section 8b).
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200_LIB_PATH") or os.path.join(_HERE, "libb200conv.so")   # override: A/B builds in tools/

ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2
MIX_NONE, MIX_MIXUP, MIX_CUTMIX = 0, 1, 2      # B200_MIX_* (input mixing of b200_input_prep_mix)


class B200Error(RuntimeError):
    pass


class ConvDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in
                ("N", "H", "W", "C", "K", "R", "S", "stride", "pad_h", "pad_w", "P", "Q",
                 "x_pixel_stride", "x_row_stride", "x_image_stride", "window")]


class Epilogue(ctypes.Structure):
    _fields_ = [("bias", ctypes.c_void_p), ("residual", ctypes.c_void_p),
                ("act", ctypes.c_int), ("out_fp32", ctypes.c_int), ("bn_stats_workspace", ctypes.c_void_p)]


_vp, _i, _ll, _f, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_size_t
_dp = ctypes.POINTER(ConvDesc)
_ep = ctypes.POINTER(Epilogue)

# name -> argtypes (restype is int unless listed in _RESTYPES)
SIGNATURES = {
    "b200_conv_fprop": [_dp, _vp, _vp, _vp, _ep, _vp],
    "b200_conv_dgrad": [_dp, _vp, _vp, _vp, _vp, _vp],
    "b200_conv_wgrad": [_dp, _vp, _vp, _vp, _vp, _sz, _vp],
    "b200_conv_wgrad_workspace_bytes": [],
    "b200_dwconv_fprop": [_dp, _vp, _vp, _vp, _vp],
    "b200_dwconv_dgrad": [_dp, _vp, _vp, _vp, _vp],
    "b200_dwconv_wgrad": [_dp, _vp, _vp, _vp, _vp, _sz, _vp],
    "b200_bn_workspace_floats": [_i],
    "b200_bn_act_mask_bytes": [_ll, _i],
    "b200_bn_stats": [_vp, _ll, _i, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_finalize": [_ll, _i, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_eval_coeffs": [_i, _vp, _vp, _vp, _vp, _f, _vp, _vp, _vp],
    "b200_bn_apply": [_vp, _ll, _i, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp],
    "b200_bn_bwd_reduce": [_vp, _vp, _vp, _vp, _ll, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_bwd_dx": [_vp, _vp, _vp, _vp, _ll, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_l1_stats": [_vp, _ll, _i, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_l1_eval_coeffs": [_i, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_l1_bwd_dx": [_vp, _vp, _vp, _vp, _ll, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_apply_dropout": [_vp, _ll, _i, _vp, _vp, _vp, _i, ctypes.c_uint, _f, _vp, _vp, _vp],
    "b200_bn_bwd_reduce_dropout": [_vp, _vp, _vp, _ll, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_bn_bwd_dx_dropout": [_vp, _vp, _vp, _ll, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp],
    "b200_maxpool3x3s2_fwd": [_vp, _i, _i, _i, _i, _vp, _vp, _vp],
    "b200_maxpool3x3s2_bwd": [_vp, _vp, _i, _i, _i, _i, _vp, _vp],
    "b200_bn_apply_maxpool3x3s2": [_vp, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp],
    "b200_avgpool_fwd": [_vp, _i, _i, _i, _vp, _vp],
    "b200_avgpool_bwd": [_vp, _i, _i, _i, _vp, _vp],
    "b200_input_prep": [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp],
    "b200_input_prep_u8": [_vp, _i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float),
                           _vp, _vp],
    "b200_input_prep_mix": [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp],
    "b200_input_prep_u8_mix": [_vp, _i, _i, _i, _i, _i, _i, ctypes.POINTER(ctypes.c_float),
                               ctypes.POINTER(ctypes.c_float), _vp, _vp, _i, _vp, _vp],
    "b200_input_prep_u8_aug": [_vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp],
    "b200_input_prep_u8_aug_resize": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _i, _vp, _vp],
    "b200_input_prep_u8_rrc": [_vp, _ll, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp],
    "b200_input_prep_u8_scale_crop": [_vp, _ll, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp],
    "b200_jpeg_decode": [_vp, _ll, _vp, _i, _vp, _i, _vp, _ll, _vp, _ll, _ll, _vp, _ll, _vp, _vp],
    "b200_weight_transpose": [_vp, _vp, _i, _i, _i, _vp],
    "b200_weight_transpose_batched": [_vp, _vp, _vp, _i, _i, _vp],
    "b200_stem_weight_to_s2d": [_vp, _i, _i, _i, _vp, _vp],
    "b200_stem_wgrad_from_s2d": [_vp, _i, _i, _i, _vp, _vp],
    "b200_cast_f32_to_bf16": [_vp, _vp, _ll, _vp],
    "b200_group_weight_pack": [_vp, _i, _i, _i, _i, _i, _i, _vp, _vp],
    "b200_group_wgrad_unpack": [_vp, _i, _i, _i, _i, _i, _vp, _vp],
    "b200_se_pool": [_vp, _i, _i, _i, _vp, _vp],
    "b200_se_scale_fwd": [_vp, _vp, _i, _i, _i, _vp, _vp],
    "b200_se_bwd_reduce": [_vp, _vp, _vp, _i, _i, _i, _vp, _vp],
    "b200_se_bwd_dx": [_vp, _vp, _vp, _i, _i, _i, _vp, _vp],
    "b200_act_bwd": [_vp, _vp, _ll, _i, _vp, _vp],
    "b200_softmax_ce": [_vp, _vp, _i, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _vp],
    "b200_softmax_ce_mix": [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp],
    "b200_colsum_bf16": [_vp, _i, _i, _vp, _vp],
    "b200_fused_sgd": [_vp, _vp, _vp, _vp, _ll, _ll, _f, _f, _f, _f, _f, _vp, _i, _i, _vp],
    "b200_sumsq": [_vp, _ll, _vp, _vp, _vp],
    "b200_grad_coef": [_vp, _f, _i, _f, _f, _vp, _vp, _vp, _vp],
    "b200_last_error": [],
    "b200_version": [],
    "b200_launch_count": [],
}
_RESTYPES = {"b200_last_error": ctypes.c_char_p, "b200_launch_count": ctypes.c_longlong,
             "b200_conv_wgrad_workspace_bytes": ctypes.c_size_t,
             "b200_bn_workspace_floats": ctypes.c_size_t, "b200_bn_act_mask_bytes": ctypes.c_size_t}

_lib = None
_lock = threading.Lock()


def available():
    return os.path.exists(LIB_PATH)


def load():
    """Open libb200conv.so (once) and bind every symbol of include/b200conv.h."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise B200Error(
                "libb200conv.so not found at %s -- build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` or `make -C convnet/pytorch_b200/csrc`. There is no CPU/cuDNN fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the ABI and the binding disagree
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, ctypes.c_int)
        _lib = lib
    return _lib


def check(rc, what):
    if rc != 0:
        msg = load().b200_last_error()
        raise B200Error("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def launch_count():
    return int(load().b200_launch_count())


def ptr(t):
    """device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()
