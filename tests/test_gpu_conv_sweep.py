"""Generated sweep of the convolution kernels (implicit-GEMM fprop/dgrad, split-K wgrad, halo shift-GEMM fprop/dgrad
and wgrad) against fp64 torch, element by element.

The shapes are generated from the device's SM count, so that each intended schedule (one tile per CTA, warpgroup 1
computing tiles, five or more tiles per CTA, the M tail in a warpgroup-1 tile, owned-n-tile walks, ...) holds on any
H100 variant.  Besides dense convolutions the sweep runs grouped ones the way the engine does (block-diagonal
"window" mode -- 64-channel windows for fprop / dgrad, 128 for wgrad -- or the dense block-diagonal expansion, with
operands from b200_group_weight_pack and the gradient kept by b200_group_wgrad_unpack; references use groups=) and the
ImageNet stem's descriptors, including the wide-pixel one whose x strides make pixels overlap (reference input: the
torch.as_strided view of the same buffer).  Every case runs in two tiers:

* tier 1 -- exact arithmetic: sparse integer operands in [-2, 2] (integer bias, residual and initial dw), so every
  product and partial sum is an integer far below 2^13 and representable in fp32, and |y| <= 256 is exact in bf16.  The
  kernel must equal the fp64 reference rounded once, bit for bit, and so must the fused BN statistics.
* tier 2 -- rounding-realistic: normal bf16 operands; every element must satisfy
  |y - ref| <= rt * |ref| + c * absref, where absref is the same convolution of |x| and |w| (plus |bias| and
  |residual|), rt = 2^-8 (one bf16 output rounding) for bf16 outputs and 0 for fp32 outputs.  The relative-L2 limits
  of test_gpu_ops.py are checked as well.

In both tiers outputs are written through out= into a NaN-filled view of a larger buffer whose guard regions must stay
intact, and each call is repeated on the same inputs and must give bitwise-identical results.  test_sweep_coverage
runs the sweep with the host's per-launch debug lines enabled and fails, naming the entry, when a configuration the
sweep is meant to reach is no longer reached.
"""
import math
import re
import zlib

import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

# tier-2 accumulation-error coefficients (|y - ref| beyond the output rounding, in units of absref).  Calibrated on an
# NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit): the worst ratios over the sweep were 8.5e-8 for bf16 outputs
# (halo dgrad, K = 256) and 1.4e-7 for fp32 outputs (fprop of a 64 -> 1000 fully connected layer), 5.6x and 6.9x
# below these bounds; test_tier2_calibration_report prints them again.  With the grouped and stem cases added (NVIDIA
# H100 80GB HBM3, 132 SMs, 700 W power limit) the bf16 worst is unchanged and the fp32 worst is 1.45e-7 (the window-128
# weight gradient of the K = 512 grouped case), 6.6x below.
C_BF16 = 2.0 ** -21
C_FP32 = 2.0 ** -20
GUARD = 256               # elements before and after every output view (keeps TMA's 16-byte alignment)
SENTINEL = -1536.0        # exact in bf16 and fp32


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ the sweep
def _case(N, H, W, C, K, R=1, S=1, stride=1, pad=(0, 0), ops='fdw', bias=False, res=False, act=0, fp32=False,
          stats=False, groups=1, window=0, x_strides=None, res_f=None, res_d=None, P=None, Q=None):
    """groups > 1: a grouped convolution, run with desc.window = window (64; wgrad 128) or, window = 0, on the dense
    block-diagonal expansion.  x_strides: (pixel, row, image) strides of x in elements (None: dense NHWC).
    res_f / res_d: a residual in the fprop / dgrad epilogue (default: res, and for dgrad only where R == 3 so that the
    stride-2 residue classes are all non-empty).  P, Q: the output size (default: that of the padded convolution)."""
    pad = (pad, pad) if isinstance(pad, int) else tuple(pad)
    assert window in (0, 64) and (not window or (groups > 1 and C == K and C % 128 == 0 and 64 % (C // groups) == 0)), \
        'window mode as the engine runs it: C == K, C % 128 == 0 (128-wide wgrad windows), groups of <= 64 channels'
    res_f = res if res_f is None else res_f
    res_d = (res and R == 3) if res_d is None else res_d
    return dict(N=N, H=H, W=W, C=C, K=K, R=R, S=S, stride=stride, pad=pad, ops=ops, bias=bias, res_f=res_f,
                res_d=res_d, act=act, fp32=fp32, stats=stats, groups=groups, window=window, x_strides=x_strides, P=P,
                Q=Q)


def sweep(sm):
    """name -> case.  Most implicit-GEMM cases use 8x8 output maps (64 pixels per image), so N = 2T - 1 images give T
    m-tiles with a 64-row M tail.  T = S + S/2 gives two tiles to the busiest CTA with the tail in warpgroup 1's tile,
    2S + S/2 three tiles, 4S + S/2 five."""
    h = sm // 2
    t2, t3, t5 = sm + h, 2 * sm + h, 4 * sm + h
    n_rr = next(n for n in (5, 7, 9, 11, 3) if (2 * sm) % n)   # n-tiles that do not divide twice the grid
    m_rr = -(-t3 // n_rr)
    own_ctas = sm // 2
    m_own = 4 * own_ctas + own_ctas // 2
    per_win = sm // 8           # CTAs per 64-channel window of the K = 512 halo window launch (8 windows)
    m_win_rr = -(-t3 // (2 * n_rr))   # 2 n_rr windows of 64 channels do not divide twice the grid either
    return {
        # igemm widths 16..128 with warpgroup 1 computing tiles; A-side ck 16 / 32 / 64; schedules
        'w16_c8_deep': _case(2 * t5 - 1, 8, 8, 8, 16),                                  # >= 5 tiles per CTA
        'w32_c24_3x3s2': _case(2 * t3 - 1, 16, 16, 24, 32, 3, 3, 2, 1),                 # 3 per CTA, 9 k-iters
        'w48_c64_tail_wg1': _case(2 * t2 - 1, 8, 8, 64, 48),
        'w80_c16_3x3': _case(2 * t2, 8, 8, 16, 80, 3, 3, 1, 1),
        'w96_c32_1x3': _case(2 * t2 - 1, 8, 8, 32, 96, 1, 3, 1, (0, 1)),
        'w112_c16_1x7': _case(2 * t2 - 1, 8, 8, 16, 112, 1, 7, 1, (0, 3)),
        'bias_relu6_w128': _case(2 * t2 - 1, 8, 8, 64, 128, bias=True, act=2),         # bias on the TMA-store path
        'res_relu_w64_3x3s2': _case(2 * t3 - 1, 16, 16, 64, 64, 3, 3, 2, 1, res=True, act=1),
        'fc_fp32_bias_1000': _case(-(-t3 // 8) * 128 - 37, 1, 1, 64, 1000, bias=True, fp32=True),
        'fc_64_16': _case(64, 1, 1, 64, 16, bias=True, fp32=True),                      # one tile; unsplit wgrad
        # fused BN statistics: round-robin walks whose warpgroups change n-tile between tiles, and an owned-n-tile walk
        'stats_w64_rr': _case(2 * m_rr - 1, 8, 8, 64, 64 * n_rr, stats=True),
        'stats_w128_rr': _case(2 * m_rr - 1, 8, 8, 64, 128 * n_rr, stats=True),
        'stats_own_w128': _case(2 * m_own - 1, 8, 8, 64, 256, stats=True),
        # dgrad with empty residue classes; orphaned diagnostic shapes with 16 channels on the dy side
        'p1s2_64_128': _case(8, 16, 16, 64, 128, 1, 1, 2, 0),
        'c3_16_16': _case(4, 32, 32, 16, 16, 3, 3, 1, 1),
        'c3s2_16_32': _case(4, 32, 32, 16, 32, 3, 3, 2, 1),
        'p1s2_16_32': _case(4, 32, 32, 16, 32, 1, 1, 2, 0),
        # weight-gradient tile widths (NC = boxes per CTA x channels per box) with ragged K
        'nc32_p1': _case(4, 8, 8, 32, 32),
        'nc48_k24_1x3': _case(4, 8, 8, 16, 24, 1, 3, 1, (0, 1)),
        'nc80_k40_1x5': _case(4, 8, 8, 16, 40, 1, 5, 1, (0, 2)),
        'nc160_1x5': _case(8, 8, 8, 32, 64, 1, 5, 1, (0, 2)),
        'nc192_p1': _case(8, 8, 8, 192, 64),
        'nc224_k48_1x7': _case(4, 8, 8, 32, 48, 1, 7, 1, (0, 3)),
        # halo shift-GEMM kernels
        'halo3_w64_stats': _case(8, 28, 28, 64, 64, 3, 3, 1, 1, stats=True),
        'halo3_w128_res': _case(4, 28, 28, 64, 128, 3, 3, 1, 1, res=True, act=1),
        'halo3_w256_bias': _case(8, 14, 14, 64, 256, 3, 3, 1, 1, bias=True),
        'halo3_one_split': _case(1, 10, 10, 64, 64, 3, 3, 1, 1),
        'halo4_w64': _case(4, 32, 32, 16, 64, 4, 4, 1, 0, ops='fw'),
        'halo4_w128_stats': _case(3, 32, 32, 16, 128, 4, 4, 1, 0, ops='fw', stats=True),
        # grouped convolutions in window mode (ResNeXt, C == K, 64 % (C/g) == 0): halo kernels with diag = 1 and the
        # halo wgrad with window 128
        'grp128_g32_28_stats': _case(8, 28, 28, 128, 128, 3, 3, 1, 1, stats=True, groups=32, window=64),
        # diag epilogues; every window's CTAs take 2 or 3 tiles
        'grp512_g32_14_res': _case(per_win + per_win // 4, 14, 14, 512, 512, 3, 3, 1, 1, res=True, act=1, groups=32,
                                   window=64),
        'grp512_g32_14_bias': _case(per_win + per_win // 4, 14, 14, 512, 512, 3, 3, 1, 1, bias=True, groups=32,
                                    window=64),
        # implicit GEMM: stride 2 (four dgrad residue classes, im2col wgrad at stride 2), 7x7 maps (halo ineligible,
        # M tail, split wgrad), a 64-pixel map (one wgrad split) and a round-robin walk whose warpgroups change window
        'grp256_g32_3x3s2_stats': _case(8, 28, 28, 256, 256, 3, 3, 2, 1, stats=True, groups=32, window=64),
        'grp1024_g32_7_tail': _case(43, 7, 7, 1024, 1024, 3, 3, 1, 1, groups=32, window=64),
        'grp256_g32_8_one_split': _case(1, 8, 8, 256, 256, 3, 3, 1, 1, groups=32, window=64),
        'grp_rr_3x3s2_stats': _case(2 * m_win_rr - 1, 16, 16, 128 * n_rr, 128 * n_rr, 3, 3, 2, 1, stats=True,
                                    groups=16 * n_rr, window=64),
        # dense block-diagonal expansion (window == C): CIFAR ResNeXt's layer1 conv2 and its C != K stage entries
        'grp64_g4_32_dense': _case(8, 32, 32, 64, 64, 3, 3, 1, 1, groups=4),
        'grp16_64_g4_32_stats': _case(8, 32, 32, 16, 64, 3, 3, 1, 1, stats=True, groups=4),
        'grp64_128_g8_s2_stats': _case(8, 32, 32, 64, 128, 3, 3, 2, 1, stats=True, groups=8),
        'grp128_256_g16_s2_stats': _case(8, 16, 16, 128, 256, 3, 3, 2, 1, stats=True, groups=16),
        # the engine's ImageNet stem descriptors: 224 px on the 4x4 halo kernel (bordered 115 x 115 x 16 tensor), and
        # 256 / 288 px as 4x1 convolutions over overlapping 64-channel "wide pixels" of the bordered tensor
        'stem224_halo4_stats': _case(2, 115, 115, 16, 64, 4, 4, 1, 0, ops='fw', stats=True),
        'stem256_wide_stats': _case(2, 131, 128, 64, 64, 4, 1, 1, 0, ops='fw', stats=True,
                                    x_strides=(16, 131 * 16, 131 * 131 * 16)),
        'stem288_wide_stats_odd': _case(3, 147, 144, 64, 64, 4, 1, 1, 0, ops='fw', stats=True,
                                        x_strides=(16, 147 * 16, 147 * 147 * 16)),
    }


_NAMES = list(sweep(132))


def _get(name):
    return sweep(_sm_count())[name]


def _wgrad_window(cs):
    return 128 if cs['window'] else 0


def _desc(cs, wgrad=False):
    return _ops().make_desc(cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'], cs['S'], cs['stride'], cs['pad'],
                            P=cs['P'], Q=cs['Q'], x_strides=cs['x_strides'] or (0, 0, 0),
                            window=_wgrad_window(cs) if wgrad else cs['window'])


def _cg(cs):
    return cs['C'] // cs['groups']


def _x_shape(cs):
    """the tensor the kernels read x from: NHWC, or the flat buffer that strided-x descriptors address"""
    if cs['x_strides'] is None:
        return (cs['N'], cs['H'], cs['W'], cs['C'])
    return (cs['N'] * cs['x_strides'][2],)


def _wgrad_shape(cs):
    """the weight gradient b200_conv_wgrad writes: [K, R*S, C], or [K, R*S, 128] in window mode"""
    return (cs['K'], cs['R'] * cs['S'], _wgrad_window(cs) or cs['C'])


def _gen(name, tier, device='cpu'):
    """the operand generator of a case; on 'cuda' the draws of large cases cost no host time (other values)"""
    return torch.Generator(device=device).manual_seed(zlib.crc32(('%s/%d' % (name, tier)).encode()))


# ------------------------------------------------------------------------------------------------ fp64 references
def _nchw(t):
    return t.double().permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _xview(x, cs):
    """[N, H, W, C] view of what the kernels read as x: for strided-x descriptors neighbouring pixels overlap"""
    if cs['x_strides'] is None:
        return x
    ps, rs, ims = cs['x_strides']
    assert (cs['H'] - 1) * rs + (cs['W'] - 1) * ps + cs['C'] <= ims, 'x strides address past the image'
    return torch.as_strided(x, (cs['N'], cs['H'], cs['W'], cs['C']), (ims, rs, ps, 1))


def _w_kcrs(w, cs):
    return w.double().view(cs['K'], cs['R'], cs['S'], _cg(cs)).permute(0, 3, 1, 2)


def ref_fprop(x, w, cs):
    """w: the fp32 master [K, R*S, C/g]"""
    return _nhwc(F.conv2d(_nchw(_xview(x, cs)), _w_kcrs(w, cs), stride=cs['stride'], padding=cs['pad'],
                          groups=cs['groups']))


def ref_dgrad(dy, w, cs):
    size = (cs['N'], cs['C'], cs['H'], cs['W'])
    return _nhwc(conv2d_input(size, _w_kcrs(w, cs), _nchw(dy), stride=cs['stride'], padding=cs['pad'],
                              groups=cs['groups']))


def ref_wgrad(x, dy, cs):
    """the dense weight gradient [K, R*S, C] (grouped cases: including the entries between groups)"""
    g = conv2d_weight(_nchw(_xview(x, cs)), (cs['K'], cs['C'], cs['R'], cs['S']), _nchw(dy), stride=cs['stride'],
                      padding=cs['pad'])
    return g.permute(0, 2, 3, 1).reshape(cs['K'], cs['R'] * cs['S'], cs['C'])


def _group_cols(K, C, groups, width, device):
    """[K, C/g]: where input channel i of output channel k's group sits in a row of `width` channels -- the row of the
    window that holds k (window mode, C == K), or the whole row (width == C: the dense expansion)"""
    assert width == C or (C == K and C % width == 0)
    cg, kg = C // groups, K // groups
    k = torch.arange(K, device=device).view(K, 1)
    c = (k // kg) * cg + torch.arange(cg, device=device).view(1, cg)
    return c if width == C else c - (k // width) * width


def _take_cols(t, cols):
    """t [rows, T, width], cols [rows, n] -> [rows, T, n] with out[r, t, i] = t[r, t, cols[r, i]]"""
    return t.gather(2, cols.unsqueeze(1).expand(t.shape[0], t.shape[1], cols.shape[1]))


def pack_ref(w32, K, T, C, groups, window, transpose):
    """the b200_group_weight_pack contract, restated: the dense block-diagonal weight [K, T, C], cut into the rows of
    each output channel's window ([K, T, window]); transposed, the same from each input channel's side ([C, T, window]).
    window == C is the dense expansion for any C and K: [K, T, C], transposed [C, T, K]."""
    assert window == C or (C == K and C % window == 0)
    cg, kg = C // groups, K // groups
    dense = torch.zeros(K, T, C, dtype=w32.dtype, device=w32.device)
    for g in range(groups):
        dense[g * kg:(g + 1) * kg, :, g * cg:(g + 1) * cg] = w32[g * kg:(g + 1) * kg]
    if transpose:
        dense = dense.permute(2, 1, 0)
    if window == C:
        return dense.contiguous()
    rows = dense.shape[0]
    cols = (torch.arange(rows, device=w32.device) // window * window).view(rows, 1) + \
        torch.arange(window, device=w32.device).view(1, window)
    return _take_cols(dense, cols)


def ref_wgrad_kernel_layout(dense, cs):
    """the dense gradient as b200_conv_wgrad writes it: unchanged, or in window mode each output channel's window"""
    W = _wgrad_window(cs)
    if not W:
        return dense
    K = cs['K']
    assert K == cs['C'] and K % W == 0
    cols = (torch.arange(K, device=dense.device) // W * W).view(K, 1) + torch.arange(W, device=dense.device).view(1, W)
    return _take_cols(dense, cols)


def ref_wgrad_grouped(dense, cs):
    """[K, R*S, C/g]: the gradient of the grouped master weight"""
    return _take_cols(dense, _group_cols(cs['K'], cs['C'], cs['groups'], cs['C'], dense.device))


def _act(v, act):
    return v.relu() if act == 1 else (v.clamp(0, 6) if act == 2 else v)


# ------------------------------------------------------------------------------------------------ kernel calls
def _guarded(shape, dtype, fill):
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=dtype, device='cuda')
    view = buf[GUARD:GUARD + n].view(shape)
    view.fill_(fill)
    return buf, view


def _check_written(buf, view, what):
    n = view.numel()
    assert bool((buf[:GUARD] == SENTINEL).all()), '%s: wrote before its output' % what
    assert bool((buf[GUARD + n:] == SENTINEL).all()), '%s: wrote past its output' % what
    assert not bool(view.isnan().any()), '%s: %d output elements never written' % (what, int(view.isnan().sum()))


def _outshape(cs):
    d = _desc(cs)
    return d.P, d.Q


def call_fprop(cs, x, w, bias, res):
    """-> (y, per-channel [sum, sum of squares] from the fused statistics or None)"""
    ops = _ops()
    P, Q = _outshape(cs)
    buf, y = _guarded((cs['N'], P, Q, cs['K']), torch.float32 if cs['fp32'] else bf16, float('nan'))
    ws = torch.zeros(ops.bn_workspace_floats(cs['K']), device='cuda') if cs['stats'] else None
    ops.conv_fprop(x, w, _desc(cs), out=y, bias=bias, residual=res, act=cs['act'], out_fp32=cs['fp32'],
                   bn_stats_ws=ws)
    torch.cuda.synchronize()
    _check_written(buf, y, 'fprop')
    sums = None
    if ws is not None:
        K = cs['K']
        sums = ws[:16 * 2 * K * 2].view(torch.float64).view(16, 2, K).sum(0)   # kStatReplicas x {sum, sum^2} x K
    return y, sums


def call_dgrad(cs, dy, wt, res):
    """wt: the dgrad operand (_operands)"""
    ops = _ops()
    buf, dx = _guarded((cs['N'], cs['H'], cs['W'], cs['C']), bf16, float('nan'))
    ops.conv_dgrad(dy, wt, _desc(cs), out=dx, residual=res)
    torch.cuda.synchronize()
    _check_written(buf, dx, 'dgrad')
    return dx


def call_wgrad(cs, x, dy, dw0):
    buf, dw = _guarded(tuple(dw0.shape), torch.float32, 0.0)
    dw.copy_(dw0)
    _ops().conv_wgrad(x, dy, _desc(cs, wgrad=True), dw)
    torch.cuda.synchronize()
    _check_written(buf, dw, 'wgrad')
    return dw


def call_pack(w32, K, T, C, groups, window, transpose):
    """b200_group_weight_pack into a guarded NaN-filled buffer, checked bit for bit against pack_ref"""
    want = pack_ref(w32, K, T, C, groups, window, transpose)
    buf, out = _guarded(tuple(want.shape), bf16, float('nan'))
    _ops().group_weight_pack(w32, K, T, C, groups, window, transpose=transpose, out=out)
    torch.cuda.synchronize()
    _check_written(buf, out, 'group_weight_pack')
    bad = out.float() != want
    assert not bool(bad.any()), 'group_weight_pack(C=%d K=%d groups=%d window=%d transpose=%d): %d of %d elements ' \
        'differ, first at %s' % (C, K, groups, window, transpose, int(bad.sum()), bad.numel(),
                                 tuple(bad.nonzero()[0].tolist()))
    return out


def call_unpack(dw_win, K, T, C, groups, window, dwg0):
    """b200_group_wgrad_unpack (dw_g += ...) onto a guarded copy of dwg0, checked bit for bit"""
    buf, dwg = _guarded(tuple(dwg0.shape), torch.float32, 0.0)
    dwg.copy_(dwg0)
    _ops().group_wgrad_unpack(dw_win, K, T, C, groups, window, dwg)
    torch.cuda.synchronize()
    _check_written(buf, dwg, 'group_wgrad_unpack')
    want = dwg0 + _take_cols(dw_win, _group_cols(K, C, groups, window, dw_win.device))
    bad = dwg != want
    assert not bool(bad.any()), 'group_wgrad_unpack(C=%d K=%d groups=%d window=%d): %d of %d elements differ, first ' \
        'at %s' % (C, K, groups, window, int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
    return dwg


def _operands(cs, w32):
    """(fprop, dgrad) bf16 weight operands from the fp32 master w32 [K, R*S, C/g] (values exact in bf16): the cast and
    its transpose, or for grouped cases the packings of b200_group_weight_pack (window 64, or C: the dense expansion)"""
    if cs['groups'] == 1:
        w = w32.to(bf16)
        return w, _ops().weight_transpose(w)
    K, T, C, g = cs['K'], cs['R'] * cs['S'], cs['C'], cs['groups']
    win = cs['window'] or C
    return call_pack(w32, K, T, C, g, win, False), call_pack(w32, K, T, C, g, win, True)


def _res_fprop(cs):
    return cs['res_f']


def _res_dgrad(cs):
    return cs['res_d']


# ------------------------------------------------------------------------------------------------ tier 1
def _ints(shape, density, g, lo=-2, hi=2):
    v = torch.randint(lo, hi, shape, generator=g, device=g.device).float()
    v = torch.where(v >= 0, v + 1, v)                       # {lo..hi} without 0
    return torch.where(torch.rand(shape, generator=g, device=g.device) < density, v, v.new_zeros(()))


def _density(n, target):
    """density of two sparse operands whose n-term products have a mean absolute sum near target"""
    return min(1.0, math.sqrt(target / (2.25 * n)))


def _exact_preconditions(absref, what, bf16_out):
    amax = float(absref.max())
    assert amax <= 2 ** 11, '%s: partial sums up to %g are not far below 2^13' % (what, amax)
    if bf16_out:
        assert amax <= 256, '%s: |y| up to %g is not exact in bf16' % (what, amax)


def check_exact(cs, tag, rng='cpu'):
    """tier 1 of case cs (the directions in cs['ops']); tag seeds the operands (drawn on device rng) and names the
    case"""
    g = _gen(tag, 1, rng)
    N, H, W, C, K, RS = cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'] * cs['S']
    cg, kg = _cg(cs), K // cs['groups']
    P, Q = _outshape(cs)
    dev = 'cuda'
    if 'f' in cs['ops']:
        # fused statistics: the per-channel sum of y^2 over all M = N P Q output pixels must stay exact in fp32
        d = _density(cg * RS, min(8, 2 ** 20 / (N * P * Q)) if cs['stats'] else 16)
        x, w = _ints(_x_shape(cs), d, g), _ints((K, RS, cg), d, g)
        bias = torch.randint(-4, 5, (K,), generator=g, device=rng).float().to(dev) if cs['bias'] else None
        res = _ints((N, P, Q, K), 0.5, g).to(dev).to(bf16) if _res_fprop(cs) else None
        x, w = x.to(dev).to(bf16), w.to(dev)
        wf, _ = _operands(cs, w)
        pre = ref_fprop(x, w, cs)
        absref = ref_fprop(x.abs(), w.abs(), cs)
        if bias is not None:
            pre, absref = pre + bias.double(), absref + bias.double().abs()
        if res is not None:
            pre, absref = pre + res.double(), absref + res.double().abs()
        _exact_preconditions(absref, 'fprop', not cs['fp32'])
        ref = _act(pre, cs['act'])
        y, sums = call_fprop(cs, x, wf, bias, res)
        y2, sums2 = call_fprop(cs, x, wf, bias, res)
        assert torch.equal(y, y2), 'fprop is not deterministic'
        want = ref.to(y.dtype)
        bad = (y != want)
        assert not bool(bad.any()), 'fprop: %d of %d elements differ, first at %s' % (
            int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
        if sums is not None:
            flat = ref.reshape(-1, K)
            assert float((flat * flat).sum(0).max()) < 2 ** 24, 'statistics partials would not be exact in fp32'
            assert torch.equal(sums, sums2), 'fused statistics are not deterministic'
            assert torch.equal(sums[0], flat.sum(0)), 'fused statistics: per-channel sum differs'
            assert torch.equal(sums[1], (flat * flat).sum(0)), 'fused statistics: per-channel sum of squares differs'
    if 'd' in cs['ops']:
        d = _density(kg * RS, 16)
        dy, w = _ints((N, P, Q, K), d, g).to(dev).to(bf16), _ints((K, RS, cg), d, g).to(dev)
        res = _ints((N, H, W, C), 0.5, g).to(dev).to(bf16) if _res_dgrad(cs) else None
        _, wt = _operands(cs, w)
        ref = ref_dgrad(dy, w, cs)
        absref = ref_dgrad(dy.abs(), w.abs(), cs)
        if res is not None:
            ref, absref = ref + res.double(), absref + res.double().abs()
        _exact_preconditions(absref, 'dgrad', True)
        dx = call_dgrad(cs, dy, wt, res)
        assert torch.equal(dx, call_dgrad(cs, dy, wt, res)), 'dgrad is not deterministic'
        bad = dx != ref.to(bf16)
        assert not bool(bad.any()), 'dgrad: %d of %d elements differ, first at %s' % (
            int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
    if 'w' in cs['ops']:
        d = _density(N * P * Q, 256)
        x, dy = _ints(_x_shape(cs), d, g).to(dev).to(bf16), _ints((N, P, Q, K), d, g).to(dev).to(bf16)
        dw0 = torch.randint(-8, 9, _wgrad_shape(cs), generator=g, device=rng).float().to(dev)
        dense = ref_wgrad(x, dy, cs)
        ref = ref_wgrad_kernel_layout(dense, cs)
        _exact_preconditions(ref_wgrad(x.abs(), dy.abs(), cs) + 8, 'wgrad', False)
        zero = torch.zeros_like(dw0)
        dwz = call_wgrad(cs, x, dy, zero)
        assert torch.equal(dwz, call_wgrad(cs, x, dy, zero)), 'wgrad is not deterministic'
        dw = call_wgrad(cs, x, dy, dw0)
        bad = dw.double() != ref + dw0.double()
        assert not bool(bad.any()), 'wgrad (dw += ...): %d of %d elements differ, first at %s' % (
            int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))
        if cs['groups'] > 1:
            # keep each output channel's group (unpack, dw_g += ...): the gradient of the grouped master weight
            dwg0 = torch.randint(-8, 9, (K, RS, cg), generator=g, device=rng).float().to(dev)
            dwg = call_unpack(dwz, K, RS, C, cs['groups'], _wgrad_window(cs) or C, dwg0)
            bad = dwg.double() != ref_wgrad_grouped(dense, cs) + dwg0.double()
            assert not bool(bad.any()), 'grouped wgrad: %d of %d elements differ, first at %s' % (
                int(bad.sum()), bad.numel(), tuple(bad.nonzero()[0].tolist()))


@pytest.mark.parametrize('name', _NAMES)
def test_tier1_exact(name):
    check_exact(_get(name), name)


# ------------------------------------------------------------------------------------------------ tier 2
WORST = {}   # output type -> (worst (|y - ref| - rt |ref|) / absref, where)


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _check_bound(y, ref, absref, what, worst=WORST, coef=(C_BF16, C_FP32, 4e-3, 2e-5)):
    """coef: (c for bf16 outputs, c for fp32 outputs, rel-L2 limit for bf16 outputs, rel-L2 limit for fp32 outputs)"""
    is_bf16 = y.dtype == bf16
    rt, c = (2.0 ** -8, coef[0]) if is_bf16 else (0.0, coef[1])
    err = (y.double() - ref).abs()
    excess = err - rt * ref.abs()
    ratio = float((excess / absref.clamp_min(1e-300)).max())
    key = 'bf16' if is_bf16 else 'fp32'
    if ratio > worst.get(key, (-math.inf, ''))[0]:
        worst[key] = (ratio, what)
    bad = excess > c * absref
    assert not bool(bad.any()), '%s: %d elements outside |y-ref| <= %g |ref| + %g absref (worst ratio %.3g)' % (
        what, int(bad.sum()), rt, c, ratio)
    assert _rel_l2(y, ref) < (coef[2] if is_bf16 else coef[3]), what


def check_rounding(cs, tag, worst=WORST, rng='cpu', coef=(C_BF16, C_FP32, 4e-3, 2e-5)):
    """tier 2 of case cs (operands drawn on device rng) with the bounds coef of _check_bound; the worst excess ratios
    go into `worst`"""
    name = tag
    g = _gen(tag, 2, rng)
    N, H, W, C, K, RS = cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'] * cs['S']
    cg = _cg(cs)
    P, Q = _outshape(cs)
    dev = 'cuda'
    x = torch.randn(*_x_shape(cs), generator=g, device=rng).to(dev).to(bf16)
    w = (torch.randn(K, RS, cg, generator=g, device=rng) / math.sqrt(RS * cg)).to(dev).to(bf16).float()
    dy = torch.randn(N, P, Q, K, generator=g, device=rng).to(dev).to(bf16)
    wf, wt = _operands(cs, w)
    if 'f' in cs['ops']:
        bias = torch.randn(K, generator=g, device=rng).to(dev) if cs['bias'] else None
        res = torch.randn(N, P, Q, K, generator=g, device=rng).to(dev).to(bf16) if _res_fprop(cs) else None
        pre, absref = ref_fprop(x, w, cs), ref_fprop(x.abs(), w.abs(), cs)
        if bias is not None:
            pre, absref = pre + bias.double(), absref + bias.double().abs()
        if res is not None:
            pre, absref = pre + res.double(), absref + res.double().abs()
        y, _ = call_fprop(cs, x, wf, bias, res)
        assert torch.equal(y, call_fprop(cs, x, wf, bias, res)[0]), 'fprop is not deterministic'
        _check_bound(y, _act(pre, cs['act']), absref, '%s fprop' % name, worst, coef)
    if 'd' in cs['ops']:
        res = torch.randn(N, H, W, C, generator=g, device=rng).to(dev).to(bf16) if _res_dgrad(cs) else None
        ref, absref = ref_dgrad(dy, w, cs), ref_dgrad(dy.abs(), w.abs(), cs)
        if res is not None:
            ref, absref = ref + res.double(), absref + res.double().abs()
        dx = call_dgrad(cs, dy, wt, res)
        assert torch.equal(dx, call_dgrad(cs, dy, wt, res)), 'dgrad is not deterministic'
        _check_bound(dx, ref, absref, '%s dgrad' % name, worst, coef)
    if 'w' in cs['ops']:
        zero = torch.zeros(_wgrad_shape(cs), device=dev)
        dw = call_wgrad(cs, x, dy, zero)
        assert torch.equal(dw, call_wgrad(cs, x, dy, zero)), 'wgrad is not deterministic'
        _check_bound(dw, ref_wgrad_kernel_layout(ref_wgrad(x, dy, cs), cs),
                     ref_wgrad_kernel_layout(ref_wgrad(x.abs(), dy.abs(), cs), cs), '%s wgrad' % name, worst, coef)


@pytest.mark.parametrize('name', _NAMES)
def test_tier2_rounding(name):
    check_rounding(_get(name), name)


def test_tier2_calibration_report():
    """Prints the worst observed excess ratio next to each tier-2 coefficient (run after the tier-2 cases, e.g. with
    -s); the coefficients should stay within 8x of what the H100 shows."""
    if not WORST:
        pytest.skip('no tier-2 case ran in this session')
    for key, c in (('bf16', C_BF16), ('fp32', C_FP32)):
        if key in WORST:
            ratio, where = WORST[key]
            print('tier-2 %s outputs: worst (|y-ref| - rt|ref|)/absref = %.3e (%s), bound c = %.3e (%.1fx)' % (
                key, ratio, where, c, c / ratio if ratio > 0 else math.inf))


# ------------------------------------------------------------------------------------------------ coverage
_LINE = re.compile(r'^\[(igemm|wgrad|halo|halo_wgrad)\] (.*)$')


def _parse(text, case, op, cs):
    recs = []
    for line in text.splitlines():
        m = _LINE.match(line.strip())
        if m:
            r = {k: int(v) for k, v in (kv.split('=') for kv in m.group(2).split())}
            r.update(kind=m.group(1), case=case, op=op, filt=(cs['R'], cs['S']), conv_stride=cs['stride'])
            recs.append(r)
    return recs


def _tail_in_wg1(r):
    """an igemm launch whose last (partial) m-tile is computed by warpgroup 1 of its CTA"""
    if r['M'] % 128 == 0:
        return False
    last = r['m_tiles'] - 1
    if r['own']:
        return (last // (r['grid'] // r['n_tiles'])) & 1 == 1
    return any(((last * r['n_tiles'] + n) // r['grid']) & 1 for n in range(r['n_tiles']))


def _requirements():
    ig = lambda r: r['kind'] == 'igemm'
    igf = lambda r: ig(r) and r['op'] == 'fprop'
    igd = lambda r: ig(r) and r['op'] == 'dgrad'
    wg = lambda r: r['kind'] == 'wgrad'
    ha = lambda r: r['kind'] == 'halo'
    hw = lambda r: r['kind'] == 'halo_wgrad'
    req = {}
    for bn in range(16, 129, 16):
        req['igemm fprop width %d, warpgroup 1 computing' % bn] = \
            lambda r, bn=bn: igf(r) and r['block_n'] == bn and r['max_tiles'] >= 2
    req.update({
        'igemm 1 tile per CTA': lambda r: ig(r) and r['max_tiles'] == 1,
        'igemm odd tile count per CTA': lambda r: ig(r) and r['max_tiles'] >= 3 and r['max_tiles'] % 2 == 1,
        'igemm >= 5 tiles per CTA': lambda r: ig(r) and r['max_tiles'] >= 5,
        'igemm ring wraps mid-tile': lambda r: ig(r) and r['max_tiles'] >= 2 and r['k_iters'] % r['stages'] != 0,
        'igemm M tail in a warpgroup-1 tile': lambda r: ig(r) and _tail_in_wg1(r),
        'igemm tma_store on': lambda r: ig(r) and r['tma_store'] == 1,
        'igemm tma_store off': lambda r: ig(r) and r['tma_store'] == 0,
        'igemm plain_a on': lambda r: ig(r) and r['plain_a'] == 1,
        'igemm plain_a off': lambda r: ig(r) and r['plain_a'] == 0,
        'igemm b_stationary': lambda r: ig(r) and r['bstat'] == 1,
        'igemm own_ntile': lambda r: ig(r) and r['own'] == 1,
        'igemm fprop ck 16 (C = 8)': lambda r: igf(r) and r['ck'] == 16 and r['C'] == 8,
        'igemm fprop ck 32 (C = 24)': lambda r: igf(r) and r['ck'] == 32 and r['C'] == 24,
        'igemm fprop ck 64': lambda r: igf(r) and r['ck'] == 64,
        'igemm bias, bf16 TMA-store output': lambda r: igf(r) and r['bias'] and r['tma_store'] and not r['out_fp32'],
        'igemm bias, fp32 output': lambda r: igf(r) and r['bias'] and r['out_fp32'],
        'igemm fprop residual': lambda r: igf(r) and r['res'],
        'igemm act 1': lambda r: igf(r) and r['act'] == 1,
        'igemm act 2': lambda r: igf(r) and r['act'] == 2,
        'igemm statistics, width 64': lambda r: ig(r) and r['stats'] and r['block_n'] == 64,
        'igemm statistics, width 128': lambda r: ig(r) and r['stats'] and r['block_n'] == 128,
        'igemm statistics, warpgroup changes n-tile, M tail':
            lambda r: ig(r) and r['stats'] and not r['own'] and (2 * r['grid']) % r['n_tiles'] != 0
            and r['max_tiles'] >= 3 and r['M'] % 128 != 0,
        'dgrad stride 1': lambda r: igd(r) and r['os'] == 1,
        'dgrad stride 2': lambda r: igd(r) and r['os'] == 2,
        'dgrad 1x1 stride 2 (empty residue classes)': lambda r: igd(r) and r['os'] == 2 and r['filt'] == (1, 1),
        'dgrad 3x3 stride 2': lambda r: igd(r) and r['os'] == 2 and r['filt'] == (3, 3),
        'dgrad residual': lambda r: igd(r) and r['res'],
        'dgrad dy-side ck 16': lambda r: igd(r) and r['ck'] == 16,
        'dgrad dy-side ck 32': lambda r: igd(r) and r['ck'] == 32,
        'dgrad dy-side ck 64': lambda r: igd(r) and r['ck'] == 64,
    })
    for nc in (16, 32, 48, 64, 80, 96, 112, 128, 160, 192, 224, 256):
        req['wgrad NC %d' % nc] = lambda r, nc=nc: wg(r) and r['nc'] == nc
    req.update({
        'wgrad split (partial tiles + reduce)': lambda r: wg(r) and r['partial'] == 1,
        'wgrad unsplit (direct red.add)': lambda r: wg(r) and r['partial'] == 0,
        'wgrad partial last column group': lambda r: wg(r) and r['nboxes_last'] < r['bpc'],
        'wgrad K % 128 <= 64': lambda r: wg(r) and r['K'] % 128 <= 64,
        'wgrad K % 128 > 64': lambda r: wg(r) and r['K'] % 128 > 64,
        'wgrad ckA 16': lambda r: wg(r) and r['ckA'] == 16,
        'wgrad ckA 32': lambda r: wg(r) and r['ckA'] == 32,
        'wgrad plain_x on': lambda r: wg(r) and r['plain_x'] == 1,
        'wgrad plain_x off': lambda r: wg(r) and r['plain_x'] == 0,
        'wgrad stride 2': lambda r: wg(r) and r['stride'] == 2,
    })
    for bn in (64, 128, 256):
        req['halo 3x3 block_n %d' % bn] = lambda r, bn=bn: ha(r) and r['taps'] == 9 and r['block_n'] == bn
    for bn in (64, 128):
        req['halo 4x4 stem block_n %d' % bn] = lambda r, bn=bn: ha(r) and r['taps'] == 16 and r['block_n'] == bn
    req.update({
        'halo 3x3 stationary weights': lambda r: ha(r) and r['taps'] == 9 and r['bstat'] == 1,
        'halo 3x3 streamed weights': lambda r: ha(r) and r['taps'] == 9 and r['bstat'] == 0,
        'halo dgrad': lambda r: ha(r) and r['dir'] == 1,
        'halo residual + ReLU': lambda r: ha(r) and r['res'] and r['act'] == 1,
        'halo bias': lambda r: ha(r) and r['bias'],
        'halo fused statistics': lambda r: ha(r) and r['stats'],
        'halo wgrad 3x3': lambda r: hw(r) and r['taps'] == 9,
        'halo wgrad 4x4': lambda r: hw(r) and r['taps'] == 16,
        'halo wgrad K % 128 == 64': lambda r: hw(r) and r['K'] % 128 == 64,
        'halo wgrad one split': lambda r: hw(r) and r['splits'] == 1,
        'halo wgrad many splits': lambda r: hw(r) and r['splits'] > 1,
    })
    # grouped convolutions in window mode, and the ImageNet stem's descriptors
    req.update({
        'igemm window fprop stride 1': lambda r: igf(r) and r['window'] == 64 and r['conv_stride'] == 1,
        'igemm window fprop stride 2': lambda r: igf(r) and r['window'] == 64 and r['conv_stride'] == 2,
        'igemm window dgrad stride 1': lambda r: igd(r) and r['window'] == 64 and r['os'] == 1,
        'igemm window dgrad stride 2': lambda r: igd(r) and r['window'] == 64 and r['os'] == 2,
        'igemm window + statistics': lambda r: ig(r) and r['window'] == 64 and r['stats'],
        'igemm window, M tail': lambda r: ig(r) and r['window'] == 64 and r['M'] % 128 != 0,
        'igemm window, warpgroup changes window':
            lambda r: ig(r) and r['window'] == 64 and not r['own'] and (2 * r['grid']) % r['n_tiles'] != 0
            and r['max_tiles'] >= 3,
        'halo diag fprop': lambda r: ha(r) and r['diag'] and r['dir'] == 0,
        'halo diag dgrad': lambda r: ha(r) and r['diag'] and r['dir'] == 1,
        'halo diag statistics': lambda r: ha(r) and r['diag'] and r['stats'],
        'halo diag residual + ReLU': lambda r: ha(r) and r['diag'] and r['res'] and r['act'] == 1,
        'halo diag bias': lambda r: ha(r) and r['diag'] and r['bias'],
        'wgrad window 128, split': lambda r: wg(r) and r['window'] == 128 and r['partial'] == 1,
        'wgrad window 128, one split': lambda r: wg(r) and r['window'] == 128 and r['partial'] == 0,
        'wgrad window 128, stride 2': lambda r: wg(r) and r['window'] == 128 and r['stride'] == 2,
        'halo wgrad window 128': lambda r: hw(r) and r['window'] == 128,
        'igemm x pixel stride + statistics': lambda r: igf(r) and r['xs'] > 0 and r['stats'],
        'wgrad x pixel stride': lambda r: wg(r) and r['xs'] > 0,
        'halo 4x4 stem K = 64 + statistics': lambda r: ha(r) and r['taps'] == 16 and r['K'] == 64 and r['stats'],
    })
    return req


def coverage_records(cases, capfd):
    """launch every case of `cases` (name -> case) once on zeros and parse the per-launch debug lines (the caller
    enables them) into records tagged with the case name and direction"""
    recs = []
    capfd.readouterr()
    for name, cs in cases.items():
        N, H, W, C, K, RS = cs['N'], cs['H'], cs['W'], cs['C'], cs['K'], cs['R'] * cs['S']
        P, Q = _outshape(cs)
        x = torch.zeros(_x_shape(cs), device='cuda', dtype=bf16)
        wf, wt = _operands(cs, torch.zeros(K, RS, _cg(cs), device='cuda'))
        dy = torch.zeros(N, P, Q, K, device='cuda', dtype=bf16)
        capfd.readouterr()
        if 'f' in cs['ops']:
            call_fprop(cs, x, wf, torch.zeros(K, device='cuda') if cs['bias'] else None,
                       torch.zeros(N, P, Q, K, device='cuda', dtype=bf16) if _res_fprop(cs) else None)
            recs += _parse(capfd.readouterr().err, name, 'fprop', cs)
        if 'd' in cs['ops']:
            call_dgrad(cs, dy, wt, torch.zeros(N, H, W, C, device='cuda', dtype=bf16) if _res_dgrad(cs) else None)
            recs += _parse(capfd.readouterr().err, name, 'dgrad', cs)
        if 'w' in cs['ops']:
            call_wgrad(cs, x, dy, torch.zeros(_wgrad_shape(cs), device='cuda'))
            recs += _parse(capfd.readouterr().err, name, 'wgrad', cs)
    return recs


def enable_debug_lines(monkeypatch):
    for var in ('B200_IGEMM_DEBUG', 'B200_WGRAD_DEBUG', 'B200_HALO_DEBUG'):
        monkeypatch.setenv(var, '1')


def test_sweep_coverage(monkeypatch, capfd):
    """Every configuration of the table in _requirements() is reached by some launch of the sweep."""
    enable_debug_lines(monkeypatch)
    recs = coverage_records(sweep(_sm_count()), capfd)
    missing = []
    lines = []
    for label, pred in _requirements().items():
        hit = next((r for r in recs if pred(r)), None)
        if hit is None:
            missing.append(label)
        else:
            lines.append('covered: %-55s by %s %s' % (label, hit['case'], hit['op']))
    with capfd.disabled():
        print('\n' + '\n'.join(lines))
    assert not missing, 'configurations no longer reached by the sweep (SMs=%d): %s' % (_sm_count(), missing)


# ------------------------------------------------------------------------------------------------ relayout kernels
# (C, K, groups, window): C/g in {4, 8, 16, 32, 64}; windows 64, 128 and C; C == K, C < K (CIFAR ResNeXt's stage
# entries) and C > K
_PACK_CASES = [
    (128, 128, 32, 64), (128, 128, 32, 128),
    (256, 256, 32, 64), (256, 256, 32, 128), (256, 256, 32, 256),
    (512, 512, 32, 64), (512, 512, 32, 128), (512, 512, 32, 512),
    (1024, 1024, 32, 64), (1024, 1024, 32, 128), (1024, 1024, 32, 1024),
    (256, 256, 4, 64), (256, 256, 4, 128), (256, 256, 4, 256),
    (64, 64, 4, 64),
    (16, 64, 4, 16), (64, 128, 8, 64), (128, 256, 16, 128), (64, 32, 2, 64), (128, 64, 2, 128),
]


@pytest.mark.parametrize('C,K,groups,window', _PACK_CASES)
def test_group_weight_pack_and_unpack(C, K, groups, window):
    """b200_group_weight_pack (both orientations) and b200_group_wgrad_unpack (dw_g += ...) bit for bit against the
    index restatement of their contract, written into guarded buffers."""
    g = torch.Generator().manual_seed(zlib.crc32(('pack/%d/%d/%d/%d' % (C, K, groups, window)).encode()))
    T, cg = 9, C // groups
    w32 = torch.randint(-256, 257, (K, T, cg), generator=g).float().cuda()      # exact in bf16
    for transpose in (False, True):
        call_pack(w32, K, T, C, groups, window, transpose)
    dw_win = torch.randint(-1000, 1001, (K, T, window), generator=g).float().cuda()
    dwg0 = torch.randint(-1000, 1001, (K, T, cg), generator=g).float().cuda()
    call_unpack(dw_win, K, T, C, groups, window, dwg0)


def test_group_pack_refuses_windows_outside_the_contract():
    from convnet.pytorch_b200.lib import B200Error
    ops = _ops()
    for C, K, groups, window in ((16, 64, 4, 64), (256, 256, 64, 96), (256, 256, 32, 48)):
        w32 = torch.zeros(K, 9, C // groups, device='cuda')
        with pytest.raises(B200Error):
            ops.group_weight_pack(w32, K, 9, C, groups, window, out=torch.zeros(K, 9, window, device='cuda',
                                                                               dtype=bf16))
        with pytest.raises(B200Error):
            ops.group_wgrad_unpack(torch.zeros(K, 9, window, device='cuda'), K, 9, C, groups, window,
                                   torch.zeros(K, 9, C // groups, device='cuda'))


@pytest.mark.parametrize('window', [128, 256])
def test_conv_window_other_than_64_refused(window):
    """fprop / dgrad run block-diagonal windows of 64 channels only, wgrad of 128 only: other windows are refused
    before anything is launched."""
    from convnet.pytorch_b200.lib import B200Error
    ops = _ops()
    C = K = 512
    x = torch.zeros(2, 8, 8, C, device='cuda', dtype=bf16)
    w = torch.zeros(K, 9, window, device='cuda', dtype=bf16)
    d = ops.make_desc(2, 8, 8, C, K, 3, 3, 1, 1, window=window)
    with pytest.raises(B200Error):
        ops.conv_fprop(x, w, d)
    with pytest.raises(B200Error):
        ops.conv_dgrad(x, w, d)
    for ww in (64, 2 * window):
        with pytest.raises(B200Error):
            ops.conv_wgrad(x, x, ops.make_desc(2, 8, 8, C, K, 3, 3, 1, 1, window=ww),
                           torch.zeros(K, 9, ww, device='cuda'))


def _stem_taps(C):
    """(s2d tap, channel block, r, s) of the 7x7/s2/p3 stem as a 4x4 convolution over the 2x2 space-to-depth input
    with a 2-pixel low border: s2d tap (ah, aw), sub-pixel (bh, bw) at channels (2 bh + bw) C .. + C reads filter
    tap r = 2 ah + bh - 1, s = 2 aw + bw - 1 when that lies inside the 7x7 filter"""
    out = []
    for ah in range(4):
        for aw in range(4):
            for bh in range(2):
                for bw in range(2):
                    r, s = 2 * ah + bh - 1, 2 * aw + bw - 1
                    if 0 <= r < 7 and 0 <= s < 7:
                        out.append((ah * 4 + aw, (bh * 2 + bw) * C, r, s))
    return out


@pytest.mark.parametrize('K,C,cpad', [(64, 3, 16), (24, 4, 16), (8, 1, 6)])
def test_stem_weight_relayout(K, C, cpad):
    """stem_weight_to_s2d (zeros in the slots no filter tap maps to and in the padding channels) and
    stem_wgrad_from_s2d (dw += ... onto a non-zero dw) bit for bit against the index restatement"""
    ops = _ops()
    g = torch.Generator().manual_seed(K * 100 + C)
    w = torch.randint(-256, 257, (K, 7, 7, C), generator=g).float().cuda()
    want = torch.zeros(K, 16, cpad, device='cuda')
    for tap, c0, r, s in _stem_taps(C):
        want[:, tap, c0:c0 + C] = w[:, r, s]
    buf, ws = _guarded((K, 16, cpad), bf16, float('nan'))
    ops.stem_weight_to_s2d(w, K, C, cpad, ws)
    torch.cuda.synchronize()
    _check_written(buf, ws, 'stem_weight_to_s2d')
    assert torch.equal(ws.float(), want)
    dws = torch.randint(-1000, 1001, (K, 16, cpad), generator=g).float().cuda()
    dw0 = torch.randint(-1000, 1001, (K, 7, 7, C), generator=g).float().cuda()
    want = dw0.clone()
    for tap, c0, r, s in _stem_taps(C):
        want[:, r, s] += dws[:, tap, c0:c0 + C]
    buf, dw = _guarded((K, 7, 7, C), torch.float32, 0.0)
    dw.copy_(dw0)
    ops.stem_wgrad_from_s2d(dws, K, C, cpad, dw)
    torch.cuda.synchronize()
    _check_written(buf, dw, 'stem_wgrad_from_s2d')
    assert torch.equal(dw, want)


@pytest.mark.parametrize('px,N', [(224, 2), (256, 1)])
def test_stem_end_to_end_exact(px, N):
    """The ImageNet stem as the engine runs it, in integers: input_prep (space-to-depth with the zero border), the
    engine's descriptor for the width (4x4 halo convolution while Ws + 3 <= 128, else 4x1 over overlapping wide
    pixels), stem_weight_to_s2d, and for the weight gradient conv_wgrad + stem_wgrad_from_s2d -- equal to the fp64
    7x7 / stride 2 / pad 3 convolution and its weight gradient bit for bit."""
    ops = _ops()
    g = torch.Generator().manual_seed(px)
    K, Cin, Hs = 64, 3, px // 2
    d = _density(49 * Cin, 16)
    x = _ints((N, Cin, px, px), d, g).cuda()
    w = _ints((K, 7, 7, Cin), d, g).cuda()
    xs = ops.input_prep(x, 16, s2d=True, border=True)
    ws = torch.empty(K, 16, 16, device='cuda', dtype=bf16)
    ops.stem_weight_to_s2d(w, K, Cin, 16, ws)
    if Hs + 3 <= 128:
        desc = ops.make_desc(N, Hs + 3, Hs + 3, 16, K, 4, 4, 1, 0, P=Hs, Q=Hs)
    else:
        desc = ops.make_desc(N, Hs + 3, Hs, 64, K, 4, 1, 1, 0, P=Hs, Q=Hs,
                             x_strides=(16, (Hs + 3) * 16, (Hs + 3) * (Hs + 3) * 16))
    y = ops.conv_fprop(xs, ws, desc)
    ref = F.conv2d(x.double(), w.double().permute(0, 3, 1, 2), stride=2, padding=3)
    _exact_preconditions(F.conv2d(x.double().abs(), w.double().abs().permute(0, 3, 1, 2), stride=2, padding=3),
                         'stem fprop', True)
    assert torch.equal(y.permute(0, 3, 1, 2).double(), ref), 'stem fprop differs'
    dd = _density(N * Hs * Hs, 256)
    x = _ints((N, Cin, px, px), dd, g).cuda()
    dy = _ints((N, Hs, Hs, K), dd, g).cuda()
    xs = ops.input_prep(x, 16, s2d=True, border=True)
    dws = torch.zeros(K, 16, 16, device='cuda')
    ops.conv_wgrad(xs, dy.to(bf16), desc, dws)
    dw0 = torch.randint(-8, 9, (K, 7, 7, Cin), generator=g).float().cuda()
    dw = ops.stem_wgrad_from_s2d(dws, K, Cin, 16, dw0.clone())
    gref = conv2d_weight(x.double(), (K, Cin, 7, 7), dy.double().permute(0, 3, 1, 2), stride=2, padding=3)
    _exact_preconditions(conv2d_weight(x.double().abs(), (K, Cin, 7, 7), dy.double().abs().permute(0, 3, 1, 2),
                                       stride=2, padding=3) + 8, 'stem wgrad', False)
    bad = dw.double() != gref.permute(0, 2, 3, 1) + dw0.double()
    assert not bool(bad.any()), 'stem wgrad: %d of %d elements differ' % (int(bad.sum()), bad.numel())
