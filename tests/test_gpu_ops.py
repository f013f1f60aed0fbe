"""Op-level parity of the HBM-bound kernels (BN, pooling, layout transforms, loss, optimizer, depthwise
conv) against fp64/fp32 torch references on bf16-rounded operands.  Tolerances: SURVEY.md section 8c
(bf16 outputs: <= 2^-7 of the tensor max; fp32 outputs: rel-L2 <= 1e-5 * sqrt(reduction/1e4))."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _ops():
    from convnet.pytorch_b200 import ops
    return ops


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def close_bf16(a, ref, tol=2 ** -7):
    a, ref = a.double(), ref.double()
    return float((a - ref).abs().max()) <= tol * float(ref.abs().max()) + 1e-6


@pytest.mark.parametrize("M,C", [(128, 64), (1000, 16), (6272, 256), (333, 24), (50, 2048), (25088, 64)])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_bn_forward_backward(M, C, act):
    ops = _ops()
    g = torch.Generator().manual_seed(M * 7 + C + act)
    z = (torch.randn(M, C, generator=g) * 1.5 + 0.3).cuda().to(bf16)
    gamma = (torch.rand(C, generator=g) + 0.5).cuda()
    beta = (torch.randn(C, generator=g) * 0.2).cuda()
    rm, rv = torch.zeros(C).cuda(), torch.ones(C).cuda()
    nbt = torch.zeros((), dtype=torch.int64).cuda()
    mean, invstd, scale, shift = [torch.empty(C).cuda() for _ in range(4)]
    ws = torch.zeros(ops.bn_workspace_floats(C)).cuda()
    res = torch.randn(M, C, generator=g).cuda().to(bf16)
    ops.bn_stats(z, gamma, beta, 1e-5, 0.1, rm, rv, nbt, mean, invstd, scale, shift, ws)
    y = ops.bn_apply(z, scale, shift, act, residual=res)
    torch.cuda.synchronize()
    # reference
    zd = z.double().requires_grad_(True)
    mu = zd.mean(0)
    var = zd.var(0, unbiased=False)
    xhat = (zd - mu) / torch.sqrt(var + 1e-5)
    pre = xhat * gamma.double() + beta.double() + res.double()
    yref = pre.relu() if act == 1 else (pre.clamp(0, 6) if act == 2 else pre)
    assert rel(mean, mu.detach()) < 1e-5 and rel(invstd, 1 / torch.sqrt(var.detach() + 1e-5)) < 1e-5
    assert rel(rm, 0.1 * mu.detach()) < 1e-5
    assert rel(rv, 0.9 + 0.1 * zd.detach().var(0, unbiased=True)) < 1e-5
    assert int(nbt) == 1
    assert close_bf16(y, yref.detach())
    # backward: use the kernel's own (bf16) y for the activation mask, as the engine does
    dy = torch.randn(M, C, generator=g).cuda().to(bf16)
    yk = y.double()
    mask = torch.ones_like(yk) if act == 0 else ((yk > 0).double() if act == 1 else ((yk > 0) & (yk < 6)).double())
    gd = dy.double() * mask
    sums = torch.empty(2 * C).cuda()
    dgam, dbet = torch.zeros(C).cuda(), torch.zeros(C).cuda()
    ops.bn_bwd_reduce(dy, y, z, act, mean, invstd, gamma, beta, sums, dgam, dbet, ws)
    gout = torch.empty_like(dy)
    dz = ops.bn_bwd_dx(dy, y, z, act, mean, invstd, gamma, beta, sums, g_out=gout)
    torch.cuda.synchronize()
    (pre_lin := xhat * gamma.double() + beta.double())
    dzd, dgam_ref, dbet_ref = torch.autograd.grad(pre_lin, [zd, ], gd, retain_graph=True)[0], \
        (gd * xhat.detach()).sum(0), gd.sum(0)
    tol = 1e-5 * math.sqrt(max(M, 1e4) / 1e4) * 10
    assert rel(dgam, dgam_ref) < tol and rel(dbet, dbet_ref) < tol
    assert rel(sums[:C], dgam_ref) < tol
    assert close_bf16(dz, dzd)
    assert close_bf16(gout, gd)
    # accumulate semantics of dgamma/dbeta
    ops.bn_bwd_reduce(dy, y, z, act, mean, invstd, gamma, beta, sums, dgam, dbet, ws)
    torch.cuda.synchronize()
    assert rel(dgam, 2 * dgam_ref) < tol
    # 1-bit activation masks written by bn_apply replace y in both backward kernels.  The bits test the fp32
    # PRE-activation value (like torch's relu/hardtanh backward); they may differ from the mask derived from the
    # bf16-rounded output only where the output rounds onto a clamp boundary.
    bits = torch.zeros(ops.bn_act_mask_bytes(M, C), dtype=torch.uint8).cuda()
    y2 = ops.bn_apply(z, scale, shift, act, residual=res, act_mask=bits)
    assert torch.equal(y2, y)
    shifts = torch.arange(8, device='cuda', dtype=torch.int32)
    # "row quad" layout: byte (row % 4) of word (row // 4) * (C / 8) + v8
    by_row = bits.view(-1, C // 8, 4).permute(0, 2, 1).reshape(-1, C // 8)[:M]
    mask2 = ((by_row.reshape(M, C // 8, 1).to(torch.int32) >> shifts) & 1).view(M, C).double()
    assert float((mask2 != mask).double().mean()) < 2e-3
    if act != 2:
        assert torch.equal(mask2, mask)
    gd2 = dy.double() * mask2
    sums2, dg2, db2 = torch.empty(2 * C).cuda(), torch.zeros(C).cuda(), torch.zeros(C).cuda()
    ops.bn_bwd_reduce(dy, None, z, act, mean, invstd, gamma, beta, sums2, dg2, db2, ws, act_mask=bits)
    gout2 = torch.empty_like(dy)
    dz2 = ops.bn_bwd_dx(dy, None, z, act, mean, invstd, gamma, beta, sums2, g_out=gout2, act_mask=bits)
    torch.cuda.synchronize()
    dzd2 = torch.autograd.grad(pre_lin, [zd], gd2)[0]
    assert rel(dg2, (gd2 * xhat.detach()).sum(0)) < tol and rel(db2, gd2.sum(0)) < tol
    assert close_bf16(dz2, dzd2) and close_bf16(gout2, gd2)


def test_bn_dual_apply_and_eval():
    ops = _ops()
    M, C = 777, 128
    g = torch.Generator().manual_seed(3)
    z = torch.randn(M, C, generator=g).cuda().to(bf16)
    z2 = torch.randn(M, C, generator=g).cuda().to(bf16)
    s1, b1, s2, b2 = [torch.randn(C, generator=g).cuda() for _ in range(4)]
    y = ops.bn_apply(z, s1, b1, 1, z2=z2, scale2=s2, shift2=b2)
    ref = (z.double() * s1.double() + b1.double() + z2.double() * s2.double() + b2.double()).relu()
    assert close_bf16(y, ref)
    gamma, beta = torch.rand(C).cuda() + 0.5, torch.randn(C).cuda()
    rm, rv = torch.randn(C).cuda(), torch.rand(C).cuda() + 0.5
    sc, sh = torch.empty(C).cuda(), torch.empty(C).cuda()
    ops.bn_eval_coeffs(gamma, beta, rm, rv, 1e-5, sc, sh)
    y = ops.bn_apply(z, sc, sh, 0)
    ref = F.batch_norm(z.double(), rm.double(), rv.double(), gamma.double(), beta.double(), False, 0.1, 1e-5)
    assert close_bf16(y, ref)


def test_bn_cumulative_momentum():
    ops = _ops()
    C = 32
    rm, rv = torch.zeros(C).cuda(), torch.ones(C).cuda()
    nbt = torch.zeros((), dtype=torch.int64).cuda()
    ws = torch.zeros(ops.bn_workspace_floats(C)).cuda()
    bn = torch.nn.BatchNorm2d(C, momentum=None).double()
    bufs = [torch.empty(C).cuda() for _ in range(4)]
    for i in range(3):
        z = torch.randn(4, 5, 5, C).cuda().to(bf16)
        ops.bn_stats(z, None, None, 1e-5, None, rm, rv, nbt, *bufs, ws)
        bn(z.double().cpu().permute(0, 3, 1, 2))
    assert int(nbt) == 3
    assert rel(rm.cpu(), bn.running_mean) < 1e-5 and rel(rv.cpu(), bn.running_var) < 1e-5


@pytest.mark.parametrize("N,H,W,C", [(2, 112, 112, 64), (3, 17, 23, 16), (1, 8, 8, 8), (5, 30, 31, 24), (70, 59, 8, 64)])
def test_maxpool(N, H, W, C):
    ops = _ops()
    x = torch.randn(N, H, W, C).cuda().to(bf16)
    y, am = ops.maxpool_fwd(x)
    xr = x.float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.max_pool2d(xr, 3, 2, 1)
    assert torch.equal(y.permute(0, 3, 1, 2).float(), yr)
    dy = torch.randn_like(y)
    dx = ops.maxpool_bwd(dy, am, (N, H, W, C))
    dxr, = torch.autograd.grad(yr, xr, dy.float().permute(0, 3, 1, 2))
    assert close_bf16(dx.permute(0, 3, 1, 2), dxr, 2 ** -7)


@pytest.mark.parametrize("N,H,W,C", [(4, 112, 112, 64), (3, 17, 23, 16), (2, 9, 8, 128)])
def test_stem_bn_relu_maxpool_chain(N, H, W, C):
    """ImageNet stem tail (models/resnet.py:226-230 of the reference: bn1 -> relu -> maxpool): the fused forward is
    bit-identical to bn_apply + maxpool_fwd; the backward chain the engine runs (maxpool_bwd -> bn_bwd_reduce ->
    bn_bwd_dx, ReLU mask recomputed from z) against fp64 autograd of the same function."""
    ops = _ops()
    g = torch.Generator().manual_seed(11)
    z = (torch.randn(N, H, W, C, generator=g) * 1.5 + 0.3).cuda().to(bf16)
    gamma, beta = (torch.rand(C, generator=g) + 0.5).cuda(), (torch.randn(C, generator=g) * 0.3).cuda()
    gamma[::5] *= -1.0                                    # negative scales: max(relu(s*z+b)) is not monotone in z
    ws = torch.zeros(ops.bn_workspace_floats(C)).cuda()
    mean, invstd, scale, shift = [torch.empty(C).cuda() for _ in range(4)]
    ops.bn_stats(z, gamma, beta, 1e-5, 0.1, None, None, None, mean, invstd, scale, shift, ws)
    a = ops.bn_apply(z, scale, shift, 1)
    p_ref, am_ref = ops.maxpool_fwd(a)
    p, am = ops.bn_apply_maxpool(z, scale, shift, 1)
    torch.cuda.synchronize()
    assert torch.equal(p, p_ref) and torch.equal(am, am_ref)

    dp = torch.randn(p.shape, generator=g).cuda().to(bf16)
    da = ops.maxpool_bwd(dp, am, (N, H, W, C))
    sums, dgam, dbet = torch.empty(2 * C).cuda(), torch.zeros(C).cuda(), torch.zeros(C).cuda()
    ops.bn_bwd_reduce(da, None, z, 1, mean, invstd, gamma, beta, sums, dgam, dbet, ws)
    dz = ops.bn_bwd_dx(da, None, z, 1, mean, invstd, gamma, beta, sums)
    torch.cuda.synchronize()
    # fp64 reference with the kernel's routing: gradient to the stored argmax element, rounded to bf16 once (the
    # materialised pre-pool gradient), ReLU mask on the fp32 argument
    zd = z.double().view(-1, C).requires_grad_(True)
    mu, var = zd.mean(0), zd.var(0, unbiased=False)
    xhat = (zd - mu) / torch.sqrt(var + 1e-5)
    pre = xhat * gamma.double() + beta.double()
    gd = torch.zeros(N, H, W, C, dtype=torch.float64, device='cuda')
    n_i, p_i, q_i, c_i = torch.meshgrid(torch.arange(N), torch.arange(p.shape[1]), torch.arange(p.shape[2]),
                                        torch.arange(C), indexing='ij')
    n_i, p_i, q_i, c_i = [t.cuda() for t in (n_i, p_i, q_i, c_i)]
    hh = 2 * p_i - 1 + am.long() // 3
    ww = 2 * q_i - 1 + am.long() % 3
    gd.index_put_((n_i, hh, ww, c_i), dp.double(), accumulate=True)
    gd = gd.to(bf16).double()
    mask = ((z.float() * scale + shift) > 0).double()
    gd = (gd * mask).view(-1, C)
    dz_ref, = torch.autograd.grad(pre, zd, gd)
    tol = 1e-5 * math.sqrt(max(N * H * W, 1e4) / 1e4) * 10
    assert rel(dgam, (gd * xhat.detach()).sum(0)) < tol and rel(dbet, gd.sum(0)) < tol
    assert close_bf16(dz.view(-1, C), dz_ref)


def test_avgpool():
    ops = _ops()
    x = torch.randn(5, 7, 7, 256).cuda().to(bf16)
    y = ops.avgpool_fwd(x)
    assert close_bf16(y.view(5, 256), x.double().mean((1, 2)))
    dy = torch.randn(5, 1, 1, 256).cuda().to(bf16)
    dx = ops.avgpool_bwd(dy, (5, 7, 7, 256))
    assert close_bf16(dx, (dy.double() / 49).expand(5, 7, 7, 256))


def test_input_prep_and_stem_weights():
    ops = _ops()
    x = torch.randn(3, 3, 32, 48).cuda()
    o = ops.input_prep(x, 16)
    ref = torch.zeros(3, 32, 48, 16, device='cuda')
    ref[..., :3] = x.permute(0, 2, 3, 1)
    assert torch.equal(o.float(), ref.to(bf16).float())
    o = ops.input_prep(x, 16, s2d=True)
    ref = torch.zeros(3, 16, 24, 16, device='cuda')
    for dy in range(2):
        for dx in range(2):
            ref[..., (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + 3] = x[:, :, dy::2, dx::2].permute(0, 2, 3, 1)
    assert torch.equal(o.float(), ref.to(bf16).float())
    # s2d stem == 7x7/s2/p3 conv
    w = torch.randn(8, 7, 7, 3).cuda()      # KRSC
    ws = torch.empty(8, 16, 16, device='cuda', dtype=bf16)
    ops.stem_weight_to_s2d(w, 8, 3, 16, ws)
    xs = ops.input_prep(x, 16, s2d=True)
    desc = ops.make_desc(3, 16, 24, 16, 8, 4, 4, 1, 2, P=16, Q=24)
    y = ops.conv_fprop(xs, ws, desc)
    yref = F.conv2d(x.to(bf16).double(), w.to(bf16).double().permute(0, 3, 1, 2), stride=2, padding=3)
    assert close_bf16(y.permute(0, 3, 1, 2), yref)
    # stem_weight_to_s2d / stem_wgrad_from_s2d bit for bit: test_gpu_conv_sweep.py::test_stem_weight_relayout


def test_weight_transpose_and_cast():
    ops = _ops()
    w = torch.randn(70, 9, 40).cuda().to(bf16)
    assert torch.equal(ops.weight_transpose(w), w.permute(2, 1, 0).contiguous())
    src = torch.randn(100003).cuda()
    dst = torch.empty(100003, device='cuda', dtype=bf16)
    ops.cast_bf16(src, dst)
    assert torch.equal(dst, src.to(bf16))
    # multi-tensor transpose: three weights of different shapes inside one flat arena, one launch
    shapes = [(70, 9, 40), (64, 1, 256), (33, 4, 16)]
    offs, n = [], 0
    for K, T, C in shapes:
        offs.append(n)
        n += (K * T * C + 63) // 64 * 64
    flat = torch.randn(n).cuda().to(bf16)
    out = torch.zeros_like(flat)
    jobs, tiles = ops.transpose_jobs([(o, o, K, T, C) for o, (K, T, C) in zip(offs, shapes)], 'cuda')
    ops.weight_transpose_batched(flat, out, jobs, tiles)
    for o, (K, T, C) in zip(offs, shapes):
        want = flat[o:o + K * T * C].view(K, T, C).permute(2, 1, 0).contiguous()
        assert torch.equal(out[o:o + K * T * C].view(C, T, K), want)


@pytest.mark.parametrize("B,K,ld,eps", [(64, 1000, 1000, 0.0), (37, 10, 16, 0.0), (64, 1000, 1000, 0.1)])
def test_softmax_ce(B, K, ld, eps):
    ops = _ops()
    from convnet.pytorch_b200.utils.cross_entropy import cross_entropy
    logits = torch.zeros(B, ld).cuda()
    logits[:, :K] = torch.randn(B, K).cuda() * 3
    target = torch.randint(0, K, (B,)).cuda()
    loss = torch.full((3,), 77.0).cuda()          # {loss, top-1 %, top-5 %}: overwritten, not accumulated
    rows = torch.empty(2 * B, device='cuda')
    dl = torch.empty(B, ld, device='cuda', dtype=bf16)
    up = torch.full((1,), 0.5).cuda()             # upstream gradient of the loss as a device scalar
    ops.softmax_ce(logits, target, K, eps, loss=loss, row_loss=rows, dlogits=dl, grad_scale=4.0, grad_scale_dev=up)
    lr = logits[:, :K].double().requires_grad_(True)
    ref = cross_entropy(lr, target, smooth_eps=eps if eps else None)
    gref, = torch.autograd.grad(ref, lr)
    assert abs(float(loss[0]) - float(ref)) < 1e-5 * max(1.0, abs(float(ref)))
    from convnet.pytorch_b200.utils.meters import accuracy
    p1, p5 = accuracy(logits[:, :K], target, topk=(1, 5))       # utils/meters.py:59-72 of the reference
    assert abs(float(loss[1]) - float(p1)) < 1e-3 and abs(float(loss[2]) - float(p5)) < 1e-3
    assert close_bf16(dl[:, :K], 2.0 * gref)
    assert float(dl[:, K:].float().abs().sum()) == 0.0


def test_colsum():
    ops = _ops()
    m = torch.randn(256, 1000).cuda().to(bf16)
    out = torch.ones(1000).cuda()
    ops.colsum_bf16(m, out)
    assert rel(out, 1 + m.double().sum(0)) < 1e-5


@pytest.mark.parametrize("n,wd_count", [(1000003, 700000), (4096, 4096), (17, 0)])
def test_fused_sgd_matches_reference_chain(n, wd_count):
    """unscale -> WeightDecay.pre_step -> torch.optim.SGD(momentum) -> bf16 copy, three steps."""
    ops = _ops()
    g = torch.Generator().manual_seed(n)
    p0 = torch.randn(n, generator=g).cuda()
    p = p0.clone()
    m = torch.zeros(n).cuda()
    p16 = torch.empty(n, device='cuda', dtype=bf16)
    pref = p0.clone().double().requires_grad_(True)
    opt = torch.optim.SGD([pref], lr=0.1, momentum=0.9)
    for step in range(3):
        grad = torch.randn(n, generator=g).cuda() * 128.0
        ops.fused_sgd(p, grad, m, p16, n, wd_count, 0.1, 0.9, 0.0, 1e-4, 1.0 / 128.0, None, step == 0)
        gr = grad.double() / 128.0
        gr[:wd_count] += 1e-4 * pref.detach()[:wd_count]
        pref.grad = gr
        opt.step()
    torch.cuda.synchronize()
    assert rel(p, pref.detach()) < 1e-6
    assert rel(m, opt.state[pref]['momentum_buffer']) < 1e-6
    assert torch.equal(p16, p.to(bf16))


def test_sumsq_and_grad_coef():
    ops = _ops()
    g = torch.randn(3000001).cuda() * 64
    out = torch.zeros(8).cuda()
    ws = torch.empty(1024).cuda()
    ops.sumsq(g, g.numel(), out[0:1], ws)
    assert rel(out[0], (g.double() ** 2).sum()) < 1e-6
    norm = float(g.double().norm()) / 64
    ops.grad_coef(out[0:1], 1 / 64., 0, 5.0, 0.0, None, out[1:2], out[2:3])
    assert abs(float(out[2]) - norm) / norm < 1e-5 and abs(float(out[1]) - min(1.0, 5.0 / (norm + 1e-6))) < 1e-6
    state = out[4:6]
    ops.grad_coef(out[0:1], 1 / 64., 1, 0.0, 0.9, state, out[1:2], out[2:3])
    assert float(out[1]) == 1.0 and abs(float(state[0]) - norm) / norm < 1e-5
    g2 = g * 2
    ops.sumsq(g2, g2.numel(), out[0:1], ws)
    ops.grad_coef(out[0:1], 1 / 64., 1, 0.0, 0.9, state, out[1:2], out[2:3])
    run = 0.9 * norm + 0.1 * 2 * norm
    assert abs(float(out[1]) - run / (2 * norm + 1e-6)) < 1e-5


@pytest.mark.parametrize("N,H,C,stride", [(2, 28, 96, 1), (2, 56, 144, 2), (1, 7, 960, 1), (3, 14, 24, 2), (5, 7, 576, 2),
                                          (4, 19, 32, 1), (2, 37, 16, 2), (33, 112, 32, 1), (9, 112, 96, 2), (40, 4, 1024, 1)])
def test_depthwise(N, H, C, stride):
    """depthwise 3x3 (sliding-window kernels for stride 1 / 2; odd map sizes exercise the row / column tails, maps taller
    than 16 rows the chunking, large N the grid-stride loops)"""
    ops = _ops()
    x = torch.randn(N, H, H, C).cuda().to(bf16)
    w = (torch.randn(9, C) / 3).cuda().to(bf16)
    desc = ops.make_desc(N, H, H, C, C, 3, 3, stride, 1)
    y = ops.dwconv_fprop(x, w, desc)
    xr = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wr = w.double().t().reshape(C, 1, 3, 3).requires_grad_(True)
    yr = F.conv2d(xr, wr, stride=stride, padding=1, groups=C)
    assert close_bf16(y.permute(0, 3, 1, 2), yr.detach())
    dy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(yr, [xr, wr], dy.double().permute(0, 3, 1, 2))
    dx = ops.dwconv_dgrad(dy, w, desc)
    assert close_bf16(dx.permute(0, 3, 1, 2), gx)
    dw = torch.zeros(9, C).cuda()
    ws = torch.empty(592 * 9 * C).cuda()
    ops.dwconv_wgrad(x, dy, desc, dw, ws)
    assert rel(dw, gw.reshape(C, 9).t()) < 1e-5


def test_wide_pixel_stem_matches_7x7_conv():
    """bordered space-to-depth input read as overlapping 64-channel 'wide pixels' (4x1 conv) == 7x7/s2/p3 conv,
    forward and weight gradient (the ImageNet stem path of engine.ResNetRuntime)."""
    ops = _ops()
    N, H, W, K = 3, 64, 96, 32
    g = torch.Generator().manual_seed(5)
    x = torch.randn(N, 3, H, W, generator=g).cuda()
    w = (torch.randn(K, 7, 7, 3, generator=g) / 12).cuda()      # KRSC master layout
    ws = torch.empty(K, 16, 16, device='cuda', dtype=bf16)
    ops.stem_weight_to_s2d(w, K, 3, 16, ws)
    Hs, Ws = H // 2, W // 2
    xs = ops.input_prep(x, 16, s2d=True, border=True)
    assert xs.shape == (N, Hs + 3, Ws + 3, 16)
    assert float(xs[:, :2].float().abs().sum()) == 0 and float(xs[:, :, -1].float().abs().sum()) == 0
    desc = ops.make_desc(N, Hs + 3, Ws, 64, K, 4, 1, 1, 0, P=Hs, Q=Ws,
                         x_strides=(16, (Ws + 3) * 16, (Hs + 3) * (Ws + 3) * 16))
    y = ops.conv_fprop(xs, ws, desc)
    xr = x.to(bf16).double().requires_grad_(False)
    wr = w.to(bf16).double().permute(0, 3, 1, 2).requires_grad_(True)
    yr = F.conv2d(xr, wr, stride=2, padding=3)
    assert close_bf16(y.permute(0, 3, 1, 2), yr.detach())
    dy = torch.randn(N, Hs, Ws, K, generator=g).cuda().to(bf16)
    gw, = torch.autograd.grad(yr, wr, dy.double().permute(0, 3, 1, 2))
    dws = torch.zeros(K, 16, 16, device='cuda')
    ops.conv_wgrad(xs, dy, desc, dws)
    dw = torch.zeros(K, 7, 7, 3, device='cuda')
    ops.stem_wgrad_from_s2d(dws, K, 3, 16, dw)
    assert rel(dw, gw.permute(0, 2, 3, 1)) < 1e-4


@pytest.mark.parametrize("N,H,C,K,R", [(4, 28, 64, 64, 3), (8, 14, 128, 256, 1), (3, 9, 64, 512, 1), (2, 56, 64, 128, 1),
                                       (97, 14, 256, 1024, 1), (50, 28, 128, 512, 1)])   # the last two: owned-n-tile walk
def test_fused_bn_statistics_in_conv_epilogue(N, H, C, K, R):
    """conv_fprop(bn_stats_ws=...) + bn_finalize == conv_fprop followed by bn_stats on its output."""
    ops = _ops()
    assert ops.can_fuse_bn_stats(K)
    g = torch.Generator().manual_seed(K + C)
    x = torch.randn(N, H, H, C, generator=g).cuda().to(bf16)
    w = (torch.randn(K, R * R, C, generator=g) / (R * R * C) ** 0.5).cuda().to(bf16)
    desc = ops.make_desc(N, H, H, C, K, R, R, 1, R // 2)
    gamma, beta = (torch.rand(K, generator=g) + 0.5).cuda(), torch.randn(K, generator=g).cuda()
    ws = torch.zeros(ops.bn_workspace_floats(K)).cuda()
    outs = []
    for fused in (False, True):
        rm, rv = torch.zeros(K).cuda(), torch.ones(K).cuda()
        nbt = torch.zeros((), dtype=torch.int64).cuda()
        bufs = [torch.empty(K).cuda() for _ in range(4)]
        if fused:
            z = ops.conv_fprop(x, w, desc, bn_stats_ws=ws)
            ops.bn_finalize(z.numel() // K, K, gamma, beta, 1e-5, 0.1, rm, rv, nbt, *bufs, ws)
        else:
            z = ops.conv_fprop(x, w, desc)
            ops.bn_stats(z, gamma, beta, 1e-5, 0.1, rm, rv, nbt, *bufs, ws)
        torch.cuda.synchronize()
        outs.append((z, rm, rv, int(nbt), bufs))
    (z0, rm0, rv0, n0, b0), (z1, rm1, rv1, n1, b1) = outs
    assert torch.equal(z0, z1) and n0 == n1 == 1
    for a, b in zip(b0 + [rm0, rv0], b1 + [rm1, rv1]):
        assert rel(b, a) < 1e-5
    assert float(ws.abs().sum()) == 0.0      # the workspace is left zeroed


# ---- convolution kernels (im2col igemm, halo shift-GEMM, split-K wgrad) vs fp64 torch on bf16-rounded operands ----
def _conv_cases():
    import importlib.util, os
    spec = importlib.util.spec_from_file_location(
        'conv_diag', os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools', 'conv_diag.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


_CONV_CASE_NAMES = [
    'c3_64_64_56', 'p1_64_256_56', 'p1_1024_256_14', 'p1s2_256_512', 'c3s2_128_128_56', 'c3_512_512_7',
    'fc_2048_1000', 'stem_s2d', 'mb_24_144', 'mb_144_24', 'res_relu',
    # halo (shift-GEMM) path: 3x3 stride 1 at several map sizes / ragged last tile / residual epilogue / stem 4x4
    'halo_28_128', 'halo_14_256', 'halo_56_res', 'halo_36_odd', 'halo_18_512', 'halo_20x12', 'halo_56_128',
    'halo_8_256', 'halo_stem', 'halo_stem_67',
    # owned-n-tile (weight-stationary) walk of the igemm kernel
    'own_256_1024', 'own_1024_256', 'own_128_512_res',
    # small and ragged shapes of the diagnostic table (the 16-channel ones are in test_gpu_conv_sweep.py)
    'p1_64_64_m128', 'p1_128_256', 'p1_256_64_odd', 'c3_64_64', 'c3s2_64_128', 'c3_32_32', 'p1_512_2048_7',
    'p1_256_128_ragged', 'p1_512_512_res', 'p1_256_1024_14',
]


@pytest.mark.parametrize("case", _CONV_CASE_NAMES)
def test_conv_fprop_dgrad_wgrad(case):
    """Tolerances: bf16 outputs (fprop, dgrad) rel-L2 <= 4e-3 (one bf16 rounding of an fp32 accumulator is ~1.7e-3);
    fp32 weight gradients rel-L2 <= 2e-5, also after a second accumulating call (dw += semantics)."""
    diag = _conv_cases()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    r = diag.run(case)
    out_fp32 = diag.CASES[case][9].get('out_fp32', False)
    assert r['fprop'][0] < (2e-5 if out_fp32 else 4e-3), r
    if 'dgrad' in r:
        assert r.get('transpose_ok', True), r
        assert r['dgrad'][0] < 4e-3, r
    assert r['wgrad'][0] < 2e-5 and r['wgrad_acc'][0] < 2e-5, r


@pytest.mark.parametrize("case", ["g32_128_56", "g32_256_28s2", "g32_512_14", "g32_1024_7", "g8_256_20x12"])
def test_grouped_conv_window_mode(case):
    """Grouped 3x3 convolutions (nn.Conv2d(groups=32) of models/resnext.py:10-16) as block-diagonal 64-channel windows
    (b200_conv_desc.window): fprop / dgrad / wgrad vs F.conv2d(groups=g) in fp64 on bf16-rounded operands, same
    tolerances as the dense kernels; the dense block-diagonal expansion must give the same output."""
    diag = _conv_cases()
    r = diag.run_grouped(case)
    assert r['fprop'][0] < 4e-3 and r['dgrad'][0] < 4e-3, r
    assert r['wgrad'][0] < 2e-5, r
    assert r['dense_vs_window'][0] < 4e-3, r
