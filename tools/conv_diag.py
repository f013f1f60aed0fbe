"""GPU diagnostic for the wgmma convolution kernels: runs ONE case (argv[1]) or lists cases.

Each case compares fprop / dgrad / wgrad of libb200conv.so with an fp64 torch reference computed on
bf16-rounded operands.  Driven case-by-case from tools/run_gpu_diag.sh so that a trapped kernel (sticky
CUDA error) only takes down its own process.
"""
import sys
import os
import json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

# name: (N,H,W,C,K,R,S,stride,pad, extras)
CASES = {
    "p1_64_64_m128": (2, 8, 8, 64, 64, 1, 1, 1, 0, {}),
    "p1_128_256": (2, 8, 8, 128, 256, 1, 1, 1, 0, {}),
    "p1_256_64_odd": (3, 7, 7, 256, 64, 1, 1, 1, 0, {}),
    "c3_64_64": (2, 8, 8, 64, 64, 3, 3, 1, 1, {}),
    "c3s2_64_128": (2, 16, 16, 64, 128, 3, 3, 2, 1, {}),
    "c3_16_16": (4, 32, 32, 16, 16, 3, 3, 1, 1, {}),
    "c3s2_16_32": (4, 32, 32, 16, 32, 3, 3, 2, 1, {}),
    "c3_32_32": (4, 16, 16, 32, 32, 3, 3, 1, 1, {}),
    "p1s2_16_32": (4, 32, 32, 16, 32, 1, 1, 2, 0, {}),
    "p1s2_256_512": (4, 28, 28, 256, 512, 1, 1, 2, 0, {}),
    "c3_64_64_56": (8, 56, 56, 64, 64, 3, 3, 1, 1, {}),
    "p1_64_256_56": (8, 56, 56, 64, 256, 1, 1, 1, 0, {}),
    "p1_1024_256_14": (8, 14, 14, 1024, 256, 1, 1, 1, 0, {}),
    "p1_512_2048_7": (8, 7, 7, 512, 2048, 1, 1, 1, 0, {}),
    "c3_512_512_7": (8, 7, 7, 512, 512, 3, 3, 1, 1, {}),
    "c3s2_128_128_56": (4, 56, 56, 128, 128, 3, 3, 2, 1, {}),
    "fc_2048_1000": (64, 1, 1, 2048, 1000, 1, 1, 1, 0, {"bias": True, "out_fp32": True}),
    "fc_64_16": (64, 1, 1, 64, 16, 1, 1, 1, 0, {"bias": True, "out_fp32": True}),
    "stem_s2d": (2, 112, 112, 16, 64, 4, 4, 1, 2, {"P": 112, "Q": 112, "no_dgrad": True}),
    "mb_24_144": (2, 56, 56, 24, 144, 1, 1, 1, 0, {}),
    "mb_144_24": (2, 56, 56, 144, 24, 1, 1, 1, 0, {}),
    "res_relu": (2, 8, 8, 64, 64, 3, 3, 1, 1, {"residual": True, "act": 1}),
    "halo_28_128": (4, 28, 28, 128, 128, 3, 3, 1, 1, {}),
    "halo_14_256": (4, 14, 14, 256, 256, 3, 3, 1, 1, {}),
    "halo_56_res": (2, 56, 56, 64, 64, 3, 3, 1, 1, {"residual": True, "act": 1}),
    "halo_36_odd": (3, 36, 36, 64, 128, 3, 3, 1, 1, {}),
    "halo_18_512": (2, 18, 18, 128, 512, 3, 3, 1, 1, {}),
    "halo_20x12": (3, 20, 12, 64, 64, 3, 3, 1, 1, {}),
    "halo_stem": (2, 115, 115, 16, 64, 4, 4, 1, 0, {"no_dgrad": True}),
    "halo_stem_67": (3, 67, 67, 16, 64, 4, 4, 1, 0, {"no_dgrad": True}),
    "halo_56_128": (2, 56, 56, 128, 64, 3, 3, 1, 1, {}),
    "halo_8_256": (5, 8, 8, 256, 128, 3, 3, 1, 1, {}),
    # wide 1x1 layers: ragged M, residual + ReLU
    "p1_256_128_ragged": (3, 13, 13, 256, 128, 1, 1, 1, 0, {}),
    "p1_512_512_res": (2, 14, 14, 512, 512, 1, 1, 1, 0, {"residual": True, "act": 1}),
    "p1_256_1024_14": (4, 14, 14, 256, 1024, 1, 1, 1, 0, {}),
    # enough m-tiles for the owned-n-tile (weight-stationary) walk of the igemm kernel: fprop with 4 n-tiles (ragged M),
    # dgrad with 4 n-tiles, 2 n-tiles with residual + ReLU epilogue
    "own_256_1024": (97, 14, 14, 256, 1024, 1, 1, 1, 0, {}),
    "own_1024_256": (97, 14, 14, 1024, 256, 1, 1, 1, 0, {}),
    "own_128_512_res": (50, 28, 28, 128, 512, 1, 1, 1, 0, {"residual": True, "act": 1}),
}


# grouped 3x3 convolutions (ResNeXt 32 groups) through the block-diagonal "window" mode: (N,H,W,C=K,stride,groups)
GROUPED = {
    "g32_128_56": (2, 56, 56, 128, 1, 32),      # C/g = 4, halo kernels (fprop/dgrad window 64, wgrad window 128)
    "g32_256_28s2": (2, 28, 28, 256, 2, 32),    # stride 2: im2col igemm + im2col wgrad, 4 dgrad residue classes
    "g32_512_14": (3, 14, 14, 512, 1, 32),      # C/g = 16
    "g32_1024_7": (4, 7, 7, 1024, 1, 32),       # 7x7 maps: im2col path, C/g = 32
    "g8_256_20x12": (2, 20, 12, 256, 1, 8),     # C/g = 32, non-square map
}


def run_grouped(name):
    from convnet.pytorch_b200 import ops
    N, H, W, C, stride, groups = GROUPED[name]
    K, cg, T = C, C // groups, 9
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(4321)
    x = torch.randn(N, H, W, C, generator=g).to(dev).to(torch.bfloat16)
    wg = (torch.randn(K, T, cg, generator=g) / (T * cg) ** 0.5).to(dev)
    wg = wg.to(torch.bfloat16).float()                                   # fp32 master with bf16-exact values
    d64 = ops.make_desc(N, H, W, C, K, 3, 3, stride, 1, window=64)
    d128 = ops.make_desc(N, H, W, C, K, 3, 3, stride, 1, window=128)
    P, Q = d64.P, d64.Q
    xd = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    wd = wg.double().view(K, 3, 3, cg).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yref = F.conv2d(xd, wd, None, stride=stride, padding=1, groups=groups)
    out = {"case": name}
    w64 = ops.group_weight_pack(wg, K, T, C, groups, 64)
    y = ops.conv_fprop(x, w64, d64)
    torch.cuda.synchronize()
    out["fprop"] = rel_err(y.permute(0, 3, 1, 2), yref.detach())
    dy = torch.randn(N, P, Q, K, generator=g).to(dev).to(torch.bfloat16)
    gx, gw = torch.autograd.grad(yref, [xd, wd], dy.double().permute(0, 3, 1, 2))
    wt64 = ops.group_weight_pack(wg, K, T, C, groups, 64, transpose=True)
    dx = ops.conv_dgrad(dy, wt64, d64)
    torch.cuda.synchronize()
    out["dgrad"] = rel_err(dx.permute(0, 3, 1, 2), gx)
    scratch = torch.zeros(K, T, 128, device=dev, dtype=torch.float32)
    ops.conv_wgrad(x, dy, d128, scratch)
    dwg = torch.zeros(K, T, cg, device=dev, dtype=torch.float32)
    ops.group_wgrad_unpack(scratch, K, T, C, groups, 128, dwg)
    torch.cuda.synchronize()
    out["wgrad"] = rel_err(dwg, gw.permute(0, 2, 3, 1).reshape(K, T, cg))
    # the dense expansion (window == C) must agree with the windowed result
    wfull = ops.group_weight_pack(wg, K, T, C, groups, C)
    y2 = ops.conv_fprop(x, wfull, ops.make_desc(N, H, W, C, K, 3, 3, stride, 1))
    torch.cuda.synchronize()
    out["dense_vs_window"] = rel_err(y2, y)
    return out


def rel_err(a, b):
    a = a.double(); b = b.double()
    return float((a - b).norm() / (b.norm() + 1e-30)), float((a - b).abs().max()), float(b.abs().max())


def run(name):
    from convnet.pytorch_b200 import ops
    N, H, W, C, K, R, S, stride, pad, ex = CASES[name]
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(1234)
    x = torch.randn(N, H, W, C, generator=g).to(dev).to(torch.bfloat16)
    w = (torch.randn(K, R * S, C, generator=g) / (R * S * C) ** 0.5).to(dev).to(torch.bfloat16)
    P = ex.get("P"); Q = ex.get("Q")
    desc = ops.make_desc(N, H, W, C, K, R, S, stride, pad, P, Q)
    P, Q = desc.P, desc.Q
    pad_hi_h = (P - 1) * stride + R - H - pad
    pad_hi_w = (Q - 1) * stride + S - W - pad
    # references in fp64, NCHW
    xd = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    wd = w.double().view(K, R, S, C).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    xp = F.pad(xd, (pad, pad_hi_w, pad, pad_hi_h))
    bias = torch.randn(K, generator=g).to(dev) if ex.get("bias") else None
    yref = F.conv2d(xp, wd, bias.double() if bias is not None else None, stride=stride)
    res = None
    if ex.get("residual"):
        res = torch.randn(N, P, Q, K, generator=g).to(dev).to(torch.bfloat16)
        yref = yref + res.double().permute(0, 3, 1, 2)
    if ex.get("act") == 1:
        yref = yref.relu()
    out = {"case": name}
    y = ops.conv_fprop(x, w, desc, bias=bias, residual=res, act=ex.get("act", 0), out_fp32=ex.get("out_fp32", False))
    torch.cuda.synchronize()
    out["fprop"] = rel_err(y.permute(0, 3, 1, 2), yref.detach())
    # backward
    dy = torch.randn(N, P, Q, K, generator=g).to(dev).to(torch.bfloat16)
    yplain = F.conv2d(xp, wd, None, stride=stride)
    gx, gw = torch.autograd.grad(yplain, [xd, wd], dy.double().permute(0, 3, 1, 2))
    if not ex.get("no_dgrad"):
        wt = ops.weight_transpose(w)
        torch.cuda.synchronize()
        wt_ref = w.permute(2, 1, 0).contiguous()
        out["transpose_ok"] = bool(torch.equal(wt, wt_ref))
        dx = ops.conv_dgrad(dy, wt, desc)
        torch.cuda.synchronize()
        out["dgrad"] = rel_err(dx.permute(0, 3, 1, 2), gx)
    dw = torch.zeros(K, R * S, C, device=dev, dtype=torch.float32)
    ops.conv_wgrad(x, dy, desc, dw)
    torch.cuda.synchronize()
    gw_krsc = gw.permute(0, 2, 3, 1).reshape(K, R * S, C)
    out["wgrad"] = rel_err(dw, gw_krsc)
    if os.environ.get("B200_DIAG_TAPS"):
        # which tap slot holds which tap's gradient?  best-matching reference tap for every computed tap
        best = []
        for t in range(R * S):
            errs = [rel_err(dw[:, t, :], gw_krsc[:, u, :])[0] for u in range(R * S)]
            u = min(range(R * S), key=lambda i: errs[i])
            best.append((t, u, round(errs[u], 4)))
        out["tap_match"] = best
    # accumulate semantics
    ops.conv_wgrad(x, dy, desc, dw)
    torch.cuda.synchronize()
    out["wgrad_acc"] = rel_err(dw, 2 * gw_krsc)
    return out


if __name__ == "__main__":
    if len(sys.argv) < 2:
        print("\n".join(CASES))
    else:
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            r = run_grouped(sys.argv[1]) if sys.argv[1] in GROUPED else run(sys.argv[1])
            ok = all(v[0] < 1e-2 for k, v in r.items() if isinstance(v, tuple))
            r["ok"] = ok
            print("DIAG " + json.dumps(r))
        except Exception as e:  # noqa
            print("DIAG " + json.dumps({"case": sys.argv[1], "ok": False, "error": repr(e)[:500]}))
