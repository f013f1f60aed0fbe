"""Parity cases of the training features around the step, all through the C ABI:
  * the sampled (Mix&Match, config C5) optimizer regime -- GradSmooth folded into the fused SGD kernel -- against the
    torch hook chain of the same regime;
  * Trainer.train with batch augmentation (duplicates D = 3, [B, D, C, H, W] inputs) and the sampled regime against
    the same Trainer driving the stock-torch fp32 model;
  * one full-size check at the benchmark shape: a layer1 bottleneck at batch 256, 56x56, forward + backward vs fp64;
  * the fused softmax-CE kernel wired through CrossEntropyLoss (label smoothing, loss scaling via a device scalar).
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from test_gpu_engine import _pair, _rel, _cos, _setup

pytestmark = pytest.mark.gpu


def test_sampled_regime_gradsmooth_folded_matches_torch_chain():
    """OptimRegime of the 'sampled' regime (GradSmooth(momentum 0.9) BEFORE WeightDecay, models/resnet.py:282-283 of
    the reference) on the B200 arenas -- device-side norm, coefficient and fused update -- vs the per-tensor torch
    chain on the torch model, fed the SAME gradients for 5 steps with a loss scale and an LR change in between
    (the reference rebuilds the RegularizerList on adjust, which resets GradSmooth's running norm: so do we)."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.utils.optim import OptimRegime
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20, regime='sampled'), (3, 32, 32), 10, batch=32)
    regime = copy.deepcopy(ref.regime)
    regime.insert(1, {'epoch': 1, 'lr': 0.05})          # phase change at "epoch 1": adjust() fires again
    o_ref = OptimRegime(ref, copy.deepcopy(regime))
    o_mine = OptimRegime(mine, copy.deepcopy(regime))
    names = [type(r).__name__ for r in o_ref.regularizer.regularization_list] if hasattr(
        o_ref.regularizer, 'regularization_list') else []
    g = torch.Generator().manual_seed(5)
    loss_scale = 4.0
    for step in range(5):
        epoch = 0 if step < 3 else 1
        for o in (o_ref, o_mine):
            o.zero_grad()
            o.update(epoch, step)
        if step == 0:
            names = [type(r).__name__ for r in o_ref.regularizer.regularization_list]
            assert names == ['GradSmooth', 'WeightDecay']
        amp = float(torch.rand(1, generator=g)) * 3 + 0.3      # very different norms from step to step
        with torch.no_grad():
            for p, q in zip(mine.parameters(), ref.parameters()):
                gr = torch.randn(q.shape, generator=g).cuda() * amp
                q.grad = gr.clone()                              # unscaled gradient on the torch side
                p.grad.copy_(gr * loss_scale)                    # scaled on ours: the kernel folds 1/loss_scale
        o_mine.set_grad_unscale(loss_scale, 1)
        o_ref.step()
        o_mine.step()
        torch.cuda.synchronize()
        with torch.no_grad():
            for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
                assert _rel(p, q) < 2e-6, '%s after step %d: %.3e' % (n, step, _rel(p, q))
    assert o_mine.get_lr()[0] == 0.05 == o_ref.get_lr()[0]


def _run_trainer(model, batches, regime, b200, loss_scale=1.0, smooth_eps=None, adapt=None):
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    if b200:
        convert_b200(model, 'cuda')
    else:
        model.cuda()
    opt = OptimRegime(model, copy.deepcopy(regime))
    tr = Trainer(model, CrossEntropyLoss(smooth_eps=smooth_eps).cuda(), opt, device_ids=[0], device='cuda',
                 print_freq=10 ** 9, loss_scale=loss_scale, adapt_grad_norm=adapt)
    losses = []
    for b in batches:
        res = tr.train([b])
        losses.append(res['loss'])
    return tr, losses


def test_trainer_duplicates_sampled_regime_and_fused_loss():
    """Trainer.train on [B, D=3, C, H, W] batch-augmentation inputs (flattened sample-major as trainer.py:17-29 of the
    reference) with the sampled regime (GradSmooth + WeightDecay), label smoothing (fused softmax-CE kernel) and a
    loss scale of 8 (device-scalar upstream gradient): B200 path vs the same Trainer on the stock-torch fp32 model.
    5 steps: per-step loss within the bf16 band, parameters move the same way."""
    from convnet.pytorch_b200.models import resnet
    _setup()
    g = torch.Generator().manual_seed(3)
    batches = [(torch.randn(24, 3, 3, 64, 64, generator=g), torch.randint(0, 1000, (24,), generator=g))
               for _ in range(5)]
    out = []
    for b200 in (False, True):
        torch.manual_seed(123)
        model = resnet(dataset='imagenet', depth=18, regime='sampled')
        init = {k: v.detach().clone() for k, v in model.state_dict().items()}
        tr, losses = _run_trainer(model, batches, model.regime, b200, loss_scale=8.0, smooth_eps=0.1)
        out.append((losses, {k: v.detach().float().cpu() for k, v in model.state_dict().items()}, init, tr))
    (l_ref, s_ref, init, _), (l_mine, s_mine, _, tr) = out
    print('duplicates/sampled: losses torch %s  b200 %s' % (l_ref, l_mine))
    assert tr.graph_replays > 0, 'the captured-graph path (with the device-side loss scale) was not exercised'
    for a, b in zip(l_mine, l_ref):
        assert abs(a - b) < 5e-2 * max(1.0, abs(b))
    upd_m = torch.cat([(s_mine[k] - init[k].float().cpu()).flatten() for k in s_ref if 'num_batches' not in k
                       and 'running' not in k])
    upd_r = torch.cat([(s_ref[k] - init[k].float().cpu()).flatten() for k in s_ref if 'num_batches' not in k
                       and 'running' not in k])
    print('duplicates/sampled: update cos %.5f rel %.3e' % (_cos(upd_m, upd_r), _rel(upd_m, upd_r)))
    assert _cos(upd_m, upd_r) > 0.99 and _rel(upd_m, upd_r) < 0.15


def test_adapt_grad_norm_uses_clean_gradients():
    """--adapt-grad-norm (trainer.py:200-210 of the reference): the per-copy / joint gradient norms must be computed
    on freshly zeroed gradients (round-1 advisor finding: nn.Module.zero_grad() does not clear the arena)."""
    from convnet.pytorch_b200.models import resnet
    _setup()
    g = torch.Generator().manual_seed(4)
    batches = [(torch.randn(16, 2, 3, 32, 32, generator=g), torch.randint(0, 10, (16,), generator=g))
               for _ in range(3)]
    scales = []
    for b200 in (False, True):
        torch.manual_seed(123)
        model = resnet(dataset='cifar10', depth=20)
        tr, _ = _run_trainer(model, batches, model.regime, b200, adapt=1)
        scales.append(tr.grad_scale)
    print('adapt_grad_norm grad_scale torch %.5f b200 %.5f' % tuple(scales))
    assert abs(scales[0] - scales[1]) < 3e-2 * scales[0]


def test_full_size_bottleneck_at_benchmark_shape():
    """One check at the benchmark's own shape (batch 256, 56x56): the second bottleneck of layer1 of ResNet-50
    (1x1 256->64, 3x3 64->64, 1x1 64->256, identity skip; 802 816 pixels per BN) forward + backward through the
    kernels vs the same block under torch in fp64 on bf16-rounded operands."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    _setup()
    torch.manual_seed(123)
    model = resnet(dataset='imagenet', depth=50)
    with torch.no_grad():                                   # leave the vacuous zero-gamma init of the last BN
        model.layer1[1].bn3.weight.fill_(0.5)
        for p in model.parameters():
            p.copy_(p.to(torch.bfloat16).float())
    blk = copy.deepcopy(model.layer1[1]).double().cuda().train()
    convert_b200(model, 'cuda')
    rt = model._b200
    model.train()
    g = torch.Generator().manual_seed(11)
    x = torch.randn(256, 56, 56, 256, generator=g).to(torch.bfloat16).cuda()
    dy = (torch.randn(256, 56, 56, 256, generator=g) * 1e-3).to(torch.bfloat16).cuda()
    spec = rt.blocks[1]
    rt.arena.zero_grad()
    rt._transpose_weights()
    y, saved = rt._block_fwd(spec, x, True)
    dx = rt._block_bwd(spec, saved, dy)
    rt._wgrad_join()
    torch.cuda.synchronize()
    xr = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yr = blk(xr)
    yr.backward(dy.double().permute(0, 3, 1, 2))
    torch.cuda.synchronize()
    ry, rdx = _rel(y.float().permute(0, 3, 1, 2), yr), _rel(dx.float().permute(0, 3, 1, 2), xr.grad)
    print('full-size bottleneck: y rel %.3e dx rel %.3e' % (ry, rdx))
    # the reference is fp64 end to end (no storage emulation): T1 bounds of SURVEY.md section 8c apply -- the ideal
    # bf16-storage pipeline itself sits at rel-L2 ~4.4e-2 on gradients after three conv+BN units
    assert ry < 1e-2 and rdx < 8e-2
    mine = dict(model.layer1[1].named_parameters())
    for n, q in blk.named_parameters():
        c, r = _cos(mine[n].grad, q.grad), _rel(mine[n].grad, q.grad)
        print('   %-14s cos %.6f rel %.3e' % (n, c, r))
        assert c > 0.99 and r < 1e-1, n            # T1 asks every tensor for cos >= 0.95
    # pixel subsample, element-wise: 2 bf16 ulp of the channel maximum on 4096 random pixels
    idx = torch.randint(0, 256 * 56 * 56, (4096,), generator=g).cuda()
    a = y.float().view(-1, 256)[idx]
    b = yr.permute(0, 2, 3, 1).reshape(-1, 256)[idx]
    assert float(((a - b).abs() / b.abs().amax(0, keepdim=True)).max()) < 2 ** -6


@pytest.mark.parametrize("eps,scale", [(0.0, 1.0), (0.1, 8.0)])
def test_fused_cross_entropy_on_the_path(eps, scale):
    """CrossEntropyLoss on B200 logits runs the fused softmax-CE kernel (no ATen loss kernels): loss and every
    parameter gradient equal the torch formula (utils/cross_entropy.py:20-24,46-52 of the reference) applied to the
    same logits; the upstream loss scale is honoured."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss, cross_entropy
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, batch=32)
    crit = CrossEntropyLoss(smooth_eps=eps if eps else None)
    mine.train()
    arena = mine._b200.arena
    arena.zero_grad()
    logits = mine(x)
    assert getattr(logits, '_b200_head', None) is not None
    loss = crit(logits, y)
    assert type(loss.grad_fn).__name__.startswith('_FusedCE')
    up = torch.full((), scale, device='cuda')
    torch.autograd.backward(loss, grad_tensors=[up])
    g_fused = arena.g32.clone()
    want = cross_entropy(logits.detach().double(), y, smooth_eps=eps if eps else None)
    assert abs(float(loss) - float(want)) < 1e-5 * max(1.0, abs(float(want)))
    # same step through the torch definition of the loss (generic autograd path into the same network backward)
    arena.zero_grad()
    logits2 = mine(x)
    loss2 = cross_entropy(logits2.float() * 1.0, y, smooth_eps=eps if eps else None) * scale
    loss2.backward()
    torch.cuda.synchronize()
    # the only difference is one bf16 rounding of dlogits (fused: rounded once in-kernel; generic: fp32 -> cast)
    assert _rel(g_fused, arena.g32) < 2e-3 and _cos(g_fused, arena.g32) > 0.99999


def test_eval_mode_forward_carries_no_autograd_history():
    """model.eval() with grad enabled (round-1 advisor finding): the B200 path has no running-statistics BatchNorm
    backward, so the logits must not pretend to be differentiable."""
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, batch=32)
    mine.eval()
    out = mine(x)
    assert not out.requires_grad
    with pytest.raises(RuntimeError):
        F.cross_entropy(out, y).backward()


def test_uint8_input_pipeline_matches_normalised_fp32():
    """(f2) uint8 NHWC network input, normalised inside the stem's relayout kernel, vs the reference contract -- the
    same images as a normalised fp32 NCHW batch ((u8/255 - mean)/std, preprocess.py:20-24): identical logits up to the
    bf16 rounding of the input (ImageNet stem: space-to-depth layouts; CIFAR stem: padded NHWC)."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    for cfg, size in ((dict(dataset='imagenet', depth=18), 64), (dict(dataset='cifar10', depth=20), 32)):
        torch.manual_seed(123)
        m = convert_b200(resnet(**cfg), 'cuda').train()
        g = torch.Generator().manual_seed(2)
        u8 = torch.randint(0, 256, (32, size, size, 3), generator=g, dtype=torch.uint8)
        mean = torch.tensor(m._b200.input_mean).view(1, 3, 1, 1)
        std = torch.tensor(m._b200.input_std).view(1, 3, 1, 1)
        xf = (u8.permute(0, 3, 1, 2).float() / 255.0 - mean) / std
        with torch.no_grad():
            a = m(u8.cuda())
            b = m(xf.cuda())
        r = _rel(a, b)
        print('uint8 input vs fp32 (%s): logits rel %.3e' % (cfg['dataset'], r))
        assert r < 5e-3


def test_lazy_meters_match_torch_accuracy():
    """Trainer.train on the fused path reads {loss, prec1, prec5} from the loss kernel asynchronously; the averages must
    equal the reference's per-step float(loss) / accuracy(output, target) meters (trainer.py:224-227,
    utils/meters.py:59-72) computed with torch on the same logits."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.meters import accuracy
    torch.manual_seed(123)
    model = convert_b200(resnet(dataset='cifar10', depth=20), 'cuda')
    tr = Trainer(model, CrossEntropyLoss().cuda(), OptimRegime(model, model.regime), device='cuda', print_freq=3)
    g = torch.Generator().manual_seed(9)
    batches = [(torch.randn(64, 3, 32, 32, generator=g), torch.randint(0, 10, (64,), generator=g)) for _ in range(12)]
    seen = []
    orig = tr._step

    def spy(inputs, target, **kw):
        out, loss, grad = orig(inputs, target, **kw)
        p1, p5 = accuracy(out.float(), target.cuda(), topk=(1, 5))
        lo = torch.nn.functional.cross_entropy(out.float(), target.cuda())
        seen.append((float(lo), float(p1), float(p5), torch.is_tensor(loss)))
        return out, loss, grad
    tr._step = spy
    res = tr.train(batches)
    assert all(s[3] for s in seen), 'fused statistics were not used'
    for k, j in (('loss', 0), ('prec1', 1), ('prec5', 2)):
        want = sum(s[j] for s in seen) / len(seen)
        assert abs(res[k] - want) < 1e-3 * max(1.0, abs(want)), (k, res[k], want)


def test_evaluate_cli_on_the_kernel_path(tmp_path):
    """(f1) evaluate.py on the B200 path: --absorb-bn runs the conv kernels with BatchNorm folded into weights + bias
    (one launch per conv+BN+ReLU unit) and must reproduce the unfolded evaluation; --calibrate-bn re-estimates the
    running statistics with cumulative momentum through the training-mode statistics kernels (trainer.py:277-285)."""
    import os
    from convnet.pytorch_b200 import evaluate as ev
    from convnet.pytorch_b200.models import resnet
    torch.manual_seed(123)
    m = resnet(dataset='cifar10', depth=20)
    g = torch.Generator().manual_seed(0)
    x, y = torch.randn(64, 3, 32, 32, generator=g), torch.randint(0, 10, (64,), generator=g)
    opt = torch.optim.SGD(m.parameters(), lr=0.05, momentum=0.9)
    m.train()
    for _ in range(5):                                    # leave the vacuous init, move the running statistics
        opt.zero_grad(); F.cross_entropy(m(x), y).backward(); opt.step()
    ck = str(tmp_path / 'ck.pth.tar')
    torch.save({'epoch': 1, 'model': 'resnet', 'config': "{'depth': 20}", 'state_dict': m.state_dict()}, ck)
    os.environ['B200_SYNTHETIC_LENGTH'] = '256'
    try:
        common = [ck, '--dataset', 'synthetic_cifar10', '-b', '64', '--workers', '0', '--b200', 'on']
        base = ev.main(common)
        absorbed = ev.main(common + ['--absorb-bn'])
        calib = ev.main(common + ['--absorb-bn', '--calibrate-bn', '--calibrate-steps', '3'])
        m.eval()
        ref = ev.main([ck, '--dataset', 'synthetic_cifar10', '-b', '64', '--workers', '0', '--b200', 'off',
                       '--device', 'cuda'])
    finally:
        del os.environ['B200_SYNTHETIC_LENGTH']
    print('evaluate: unfolded %s | folded %s | calibrated %s | torch %s' % (base['loss'], absorbed['loss'],
                                                                          calib['loss'], ref['loss']))
    assert abs(base['loss'] - absorbed['loss']) < 2e-2 * max(1.0, base['loss'])
    assert abs(base['loss'] - ref['loss']) < 2e-2 * max(1.0, ref['loss'])
    assert abs(base['prec1'] - ref['prec1']) <= 2.0 and abs(absorbed['prec1'] - ref['prec1']) <= 2.0
    assert calib['loss'] > 0 and calib['loss'] == calib['loss']
