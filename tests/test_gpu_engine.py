"""End-to-end parity of the B200 pipeline against the same model executed by stock torch (fp32) on the
same device: logits, loss, every parameter gradient, BN running statistics and the post-step parameters.

Test-net state: default init followed by a few fp32 SGD steps ("state B" of SURVEY.md section 8c) -- at
init 2/3 of the gradients are exactly zero (last-BN gamma = 0), which would make the comparison vacuous.
Tolerances are the calibrated T1 tier of SURVEY.md section 8c (bf16 storage vs fp32 reference).
"""
import copy

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _setup():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _warm(model, x, y, steps, lr=0.05):
    opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=0.9)
    model.train()
    for _ in range(steps):
        opt.zero_grad()
        F.cross_entropy(model(x), y).backward()
        opt.step()


def _pair(factory, cfg, shape, classes, steps=5, batch=16):
    from convnet.pytorch_b200.engine import convert_b200
    _setup()
    torch.manual_seed(123)
    ref = factory(**cfg).cuda()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(batch, *shape, generator=g).cuda()
    y = torch.randint(0, classes, (batch,), generator=g).cuda()
    _warm(ref, x, y, steps)
    mine = factory(**cfg)
    mine.load_state_dict(copy.deepcopy(ref.state_dict()))
    convert_b200(mine)
    # the B200 path computes with bf16-rounded weights: give the reference the same rounded values
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(p.to(torch.bfloat16).float())
        for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
            p.copy_(q)
    mine._b200.arena.sync_shadow()
    return ref, mine, x, y


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _global(grads, names):
    return torch.cat([grads[n].detach().double().cpu().flatten() for n in names])


def _check_step(ref, mine, x, y, logit_tol=1e-2, loss_tol=3e-2, cos_min=0.95, gcos=0.998, grel=8e-2):
    """T1 of SURVEY.md section 8c (semantic tier): the bf16 pipeline vs the same model in fp32 under stock torch on
    identical bf16-rounded parameters and inputs, batches >= 32.  The survey's bounds -- logits rel-L2 <= 1e-2,
    |d loss| <= 3e-2, global gradient cos >= 0.998 and rel-L2 <= 8e-2, every gradient tensor cos >= 0.95 -- are "the
    inherent bf16-storage drift of an ideal pipeline x 1.5-2" for the state the survey calibrated (there: 0.044).  The
    drift of the IDEAL pipeline depends on the network state (the stem's weight gradient carries most of it); so when a
    gradient bound is exceeded the ideal drift is measured for this very state -- the CPU oracle with bf16 rounding at
    the kernels' storage points vs the same oracle in fp32 -- and the pipeline must stay within 1.25 x of it.  Tighter
    than the ideal pipeline is not attainable at bf16 storage and is not claimed."""
    assert x.shape[0] >= 32, 'parity tests run at >= 32 samples (tiny batches create near-dead BN channels)'
    ref.train(); mine.train()
    xq = x.to(torch.bfloat16).float()
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    ref.zero_grad()
    lo_r = ref(xq)
    loss_r = F.cross_entropy(lo_r, y)
    loss_r.backward()
    mine._b200.arena.zero_grad()
    lo_m = mine(x)
    loss_m = F.cross_entropy(lo_m, y)
    loss_m.backward()
    torch.cuda.synchronize()
    assert lo_m.shape == lo_r.shape
    names = [n for n, _ in mine.named_parameters()]
    gm = _global({n: p.grad for n, p in mine.named_parameters()}, names)
    gr = _global({n: p.grad for n, p in ref.named_parameters()}, names)
    per = sorted((_cos(p.grad, q.grad), n) for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters())
                 if float(q.grad.norm()) > 0)
    print('T1 logits rel %.3e  dloss %.3e  grad cos %.5f rel %.3e  worst tensors %s'
          % (_rel(lo_m, lo_r), abs(float(loss_m) - float(loss_r)), _cos(gm, gr), _rel(gm, gr), per[:3]))
    assert _rel(lo_m, lo_r) < logit_tol, 'logits rel-L2 %.3e' % _rel(lo_m, lo_r)
    assert abs(float(loss_m) - float(loss_r)) < loss_tol
    if not (_cos(gm, gr) > gcos and _rel(gm, gr) < grel and per[0][0] > cos_min):
        from oracle import ref_model
        _, _, g_q, _ = ref_model.loss_and_grads(sd, x.cpu(), y.cpu(), quant=True)
        _, _, g_f, _ = ref_model.loss_and_grads(sd, xq.cpu(), y.cpu(), quant=False)
        iq, jf = _global(g_q, names), _global(g_f, names)
        ideal_rel, ideal_cos = _rel(iq, jf), _cos(iq, jf)
        ideal_worst = min(_cos(g_q[n], g_f[n]) for n in names if float(g_f[n].norm()) > 0)
        print('T1 ideal bf16-storage pipeline in this state: grad cos %.5f rel %.3e worst tensor cos %.4f'
              % (ideal_cos, ideal_rel, ideal_worst))
        assert _rel(gm, gr) < max(grel, 1.25 * ideal_rel), 'global grad rel %.3e (ideal %.3e)' % (_rel(gm, gr), ideal_rel)
        assert 1.0 - _cos(gm, gr) < max(1.0 - gcos, 1.5 * (1.0 - ideal_cos)), 'global grad cos %.5f (ideal %.5f)' % (
            _cos(gm, gr), ideal_cos)
        assert 1.0 - per[0][0] < max(1.0 - cos_min, 1.5 * (1.0 - ideal_worst)), 'grad cos of %s = %.4f' % (per[0][1], per[0][0])
    for (n, b), (_, c) in zip(mine.named_buffers(), ref.named_buffers()):
        if 'num_batches' in n:
            assert int(b) == int(c)
        else:
            assert _rel(b, c) < 2e-2, 'buffer %s rel %.3e' % (n, _rel(b, c))
    return per[0][0]


def test_resnet20_cifar_step():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, batch=64)
    _check_step(ref, mine, x, y)


def test_resnet18_imagenet_step():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=18), (3, 128, 128), 1000, batch=64)
    _check_step(ref, mine, x, y)


def _check_against_bf16_oracle(mine, ref, x, y, logit_tol=1e-3, grad_tol=1e-2, cos_min=0.999):
    """T2 of SURVEY.md section 8c (bit-level intent): the CPU oracle with bf16 rounding at exactly the points where the
    kernels store bf16; batches >= 32.  The survey's bounds are logits rel-L2 <= 1e-3, global gradient rel-L2 <= 1e-2,
    every gradient tensor cos >= 0.999 ("differences come only from accumulation order").  A bf16-storage network is,
    however, sensitive to WHICH way individual roundings fall: nudging 0.1 % of the input pixels by one bf16 ulp moves
    the oracle's own conv-weight gradients by several percent (measured: ResNet-18, 5-7 %).  The test therefore also
    measures that self-sensitivity for the state at hand and accepts max(survey bound, 1.5 x self-sensitivity): the
    pipeline may be no farther from the oracle than the oracle is from itself under a perturbation far below bf16
    resolution.  Both numbers are printed."""
    from oracle import ref_model
    assert x.shape[0] >= 32
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    mine.train()
    mine._b200.arena.zero_grad()
    lo = mine(x)
    loss = F.cross_entropy(lo, y)
    loss.backward()
    torch.cuda.synchronize()
    names = [n for n, _ in mine.named_parameters()]
    xc, yc = x.cpu(), y.cpu()
    o_logits, o_loss, o_grads, o_bufs = ref_model.loss_and_grads(sd, xc, yc, quant=True)
    gq = torch.Generator().manual_seed(99)
    xb = xc.to(torch.bfloat16)
    nudge = torch.rand(xc.shape, generator=gq) < 1e-3
    xp = torch.where(nudge, (xb.float() * (1 + 2 ** -8)).to(torch.bfloat16), xb).float()
    p_logits, _, p_grads, _ = ref_model.loss_and_grads(sd, xp, yc, quant=True)
    gm = _global({n: p.grad for n, p in mine.named_parameters()}, names)
    go, gp = _global(o_grads, names), _global(p_grads, names)
    per = sorted((_cos(p.grad.cpu(), o_grads[n]), n) for n, p in mine.named_parameters() if float(o_grads[n].norm()) > 0)
    self_worst = min(_cos(p_grads[n], o_grads[n]) for n in names if float(o_grads[n].norm()) > 0)
    s_log, s_grad = _rel(p_logits, o_logits), _rel(gp, go)
    print('T2 logits rel %.3e  dloss %.3e  grad rel %.3e  worst tensors %s | oracle self-sensitivity: logits %.3e '
          'grad rel %.3e worst tensor cos %.5f' % (_rel(lo.cpu(), o_logits), abs(float(loss) - float(o_loss)),
                                                   _rel(gm, go), per[:3], s_log, s_grad, self_worst))
    assert _rel(lo.cpu(), o_logits) < max(logit_tol, 1.5 * s_log), 'logits vs bf16 oracle %.3e' % _rel(lo.cpu(), o_logits)
    assert abs(float(loss) - float(o_loss)) < 5e-3
    assert _rel(gm, go) < max(grad_tol, 1.5 * s_grad), 'global grad rel vs bf16 oracle %.3e (self %.3e)' % (_rel(gm, go), s_grad)
    assert 1.0 - per[0][0] < max(1.0 - cos_min, 1.5 * (1.0 - self_worst)), 'grad cos of %s vs bf16 oracle = %.5f' % (
        per[0][1], per[0][0])
    for n, b in mine.named_buffers():
        if 'running' in n:
            assert _rel(b.cpu(), o_bufs[n]) < 1e-3, n


def test_resnet20_against_bf16_oracle():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, batch=32)
    _check_against_bf16_oracle(mine, ref, x, y)


def test_resnet18_imagenet_against_bf16_oracle():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=18), (3, 64, 64), 1000, batch=32)
    _check_against_bf16_oracle(mine, ref, x, y)


def test_resnet50_imagenet_against_bf16_oracle():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=50), (3, 64, 64), 1000, batch=32)
    _check_against_bf16_oracle(mine, ref, x, y)


def test_resnet50_imagenet_step_and_eval():
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=50), (3, 224, 224), 1000, batch=64)
    _check_step(ref, mine, x, y)
    ref.eval(); mine.eval()
    with torch.no_grad():
        a, b = mine(x), ref(x.to(torch.bfloat16).float())
    assert _rel(a, b) < 2e-2


def test_optimizer_step_matches_reference_chain():
    """OptimRegime on the B200 arenas vs torch SGD + WeightDecay hooks on the torch model, same gradients."""
    _optimizer_chain('resnet20')


@pytest.mark.parametrize('name', ['mobilenet_v2', 'mobilenet_v1'])
def test_mobilenet_optimizer_step_matches_reference_chain(name):
    """the same for MobileNet: the dense convolution weights and the classifier weight are decayed, the depthwise
    weights, the depthwise biases, the BatchNorm parameters and the classifier bias are not"""
    _optimizer_chain(name)


def _optimizer_chain(name):
    """three steps of OptimRegime on the arenas and on the torch model from the same gradients: every parameter agrees.
    The WeightDecay filter folds into the fused SGD as an arena prefix; that prefix must be the reference's decayed set
    (oracle.ref_model.is_decayed)."""
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from oracle import ref_model
    factory, cfg, shape, classes = {
        'resnet20': (models.resnet, dict(dataset='cifar10', depth=20), (3, 32, 32), 10),
        'mobilenet_v2': (models.mobilenet_v2, dict(dataset='imagenet'), (3, 64, 64), 1000),
        'mobilenet_v1': (models.mobilenet, dict(dataset='imagenet'), (3, 64, 64), 1000)}[name]
    ref, mine, x, y = _pair(factory, cfg, shape, classes, batch=32)
    o_ref = OptimRegime(ref, copy.deepcopy(ref.regime))
    o_mine = OptimRegime(mine, copy.deepcopy(mine.regime))
    for step in range(3):
        for o in (o_ref, o_mine):
            o.zero_grad()
            o.update(0, step)
        F.cross_entropy(ref(x.to(torch.bfloat16).float()), y).backward()
        # feed the SAME gradients to both optimizers so that only the update rule is compared
        with torch.no_grad():
            for p, q in zip(mine.parameters(), ref.parameters()):
                p.grad.copy_(q.grad)
        o_ref.step()
        o_mine.step()
        with torch.no_grad():
            worst = max((_rel(p, q), n) for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()))
            print('optimizer chain %s step %d: worst parameter rel-L2 %.3e (%s)' % ((name, step) + worst))
            for (n, p), (_, q) in zip(mine.named_parameters(), ref.named_parameters()):
                assert _rel(p, q) < 1e-6, '%s after step %d: %.3e' % (n, step, _rel(p, q))
    wd, count = o_mine.optimizer.extra_wd
    sd = {k: v.cpu() for k, v in ref.state_dict().items()}
    decayed = {s.name for s in mine._b200.arena.slots if s.offset < count}
    assert wd == 1e-4 and decayed == {k for k in ref_model.param_names(sd) if ref_model.is_decayed(k, sd)}, \
        'the folded WeightDecay prefix is not the decayed set: %s' % sorted(decayed)[:8]
    sd = o_mine.state_dict()
    assert len(sd['state']) == len(list(mine.parameters()))
    k0 = sorted(sd['state'].keys())[0]
    assert 'momentum_buffer' in sd['state'][k0]


def test_state_dict_roundtrip_with_reference_layout():
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    torch.manual_seed(1)
    a = resnet(dataset='cifar10', depth=20)
    sd = copy.deepcopy(a.state_dict())
    b = convert_b200(resnet(dataset='cifar10', depth=20))
    b.load_state_dict(sd)
    for k, v in b.state_dict().items():
        assert v.shape == sd[k].shape and torch.equal(v.cpu().float(), sd[k].float()), k


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16).cuda()


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).cpu()


def _mobilenet_parity(factory, stem_name, size=128, batch=32):
    """Shared body of the MobileNet-v2 / v1 parity tests.

    Default-init MobileNets are chaotic under ANY reduced precision: the same fp32 code differs from fp64 by 3e-3..1e-2
    in its gradients and an ideal bf16-storage pipeline reaches only cos ~0.5 against fp32 (oracle/make_golden.py).  A
    whole-network gradient bound would therefore say nothing, so the check has three parts:
      1. whole-network FORWARD vs the bf16-storage oracle: logits, loss, running statistics, eval-mode logits;
      2. TEACHER-FORCED unit parity: every conv+BN(+ReLU/ReLU6)(+skip) unit is run through the kernels on the oracle's
         own input / skip / output-gradient tensors and compared with a local fp64 reference of that unit (output, input
         gradient, weight gradient, d gamma, d beta) -- well posed, no error compounding;
      3. whole-network gradient drift from stock torch fp32 no larger than twice the ideal bf16 pipeline's own drift."""
    from oracle import ref_model
    ref, mine, x, y = _pair(factory, dict(dataset='imagenet'), (3, size, size), 1000, steps=0, batch=batch)
    rt = mine._b200
    sd = {k: v.detach().cpu().clone() for k, v in ref.state_dict().items()}
    o_logits, o_loss, units = ref_model.mobilenet_v2_unit_trace(sd, x.cpu(), y.cpu())

    # ---- 1. whole-network forward (+ 3: gradients) -----------------------------------------------------------
    xq = x.to(torch.bfloat16).float()
    mine.train(); rt.arena.zero_grad()
    lo_m = mine(x)
    loss_m = F.cross_entropy(lo_m, y)
    loss_m.backward()
    torch.cuda.synchronize()
    names = [n for n, _ in mine.named_parameters()]
    gm = torch.cat([p.grad.flatten() for p in mine.parameters()]).clone()
    fwd_rel, fwd_dloss = _rel(lo_m.cpu(), o_logits), abs(float(loss_m) - float(o_loss))
    print('MobileNet forward vs oracle: logits rel %.3e  dloss %.3e' % (fwd_rel, fwd_dloss))
    _, _, o_grads, o_bufs = ref_model.loss_and_grads(sd, x.cpu(), y.cpu(), quant=True)

    # running means can sit near zero: measure the error against the scale of the statistic (its own norm or the
    # typical activation scale sqrt(running_var))
    def _buf_err(n, b):
        ref_b = o_bufs[n]
        scale = ref_b.double().norm() if 'var' in n else o_bufs[n.replace('running_mean', 'running_var')].double().sqrt().norm()
        return float((b.cpu().double() - ref_b.double()).norm() / (scale + 1e-30))
    buf_worst = max((_buf_err(n, b), n) for n, b in mine.named_buffers() if 'running' in n)
    print('MobileNet running statistics vs oracle: worst scaled error %.3e (%s)' % buf_worst)
    ref.train(); ref.zero_grad()
    F.cross_entropy(ref(xq), y).backward()
    gr = torch.cat([p.grad.flatten() for p in ref.parameters()]).cpu()
    go = torch.cat([o_grads[n].flatten() for n in names])
    drift = (_cos(gm.cpu(), gr), _cos(go, gr), _cos(gm.cpu(), go))
    print('MobileNet grad cos: mine/fp32 %.4f  oracle-bf16/fp32 %.4f  mine/oracle-bf16 %.4f' % drift)
    # eval mode on IDENTICAL running statistics (copied from the torch model): BN folded / conv biases folded into the
    # BN shift must reproduce torch's eval forward up to bf16 storage
    with torch.no_grad():
        for (n, b), (_, c) in zip(mine.named_buffers(), ref.named_buffers()):
            b.copy_(c)
    rt.arena.version += 1
    ref.eval(); mine.eval()
    with torch.no_grad():
        ev_rel = _rel(mine(x), ref(xq))
    print('MobileNet eval-mode logits vs torch (same running statistics): rel %.3e' % ev_rel)

    # ---- 2. teacher-forced units ------------------------------------------------------------------------------
    mine.train()
    flat = [(None, None, rt.stem_bn, None, stem_name)]
    for spec in rt.blocks:
        for conv, bn, act in spec['units']:
            flat.append((conv.kind, conv, bn, act, conv.slot.name[:-len('.weight')]))
    assert len(flat) == len(units) and all(f[4] == u['conv'] for f, u in zip(flat, units))
    params = dict(mine.named_parameters())
    rt._transpose_weights()
    worst = {}
    for (kind, conv, bn, act, cname), u in zip(flat, units):
        vjp = ref_model.mobilenet_v2_unit_vjp(sd, u)
        y_ref, dx_ref, dw_ref, dg_ref, db_ref = vjp[:5]
        rt.arena.zero_grad()
        dy = _nhwc(u['dy'])
        if kind is None:                                   # stem: NCHW fp32 network input, no input gradient
            out, st = rt._stem_fwd(u['x'].cuda(), True)
            rt._stem_bwd(st, dy)
            dx = None
        else:
            skip = _nhwc(u['skip']) if u['skip'] is not None else None
            uu = rt._unit_fwd(_nhwc(u['x']), conv, bn, act, True, residual=skip)
            out = uu.y
            dz, _ = rt._bn_bwd(uu, dy, None, act)
            dx = rt._conv_bwd(uu, dz)
        rt._wgrad_join()
        torch.cuda.synchronize()
        # d gamma and d beta are measured on ONE scale, the norm of the larger of the two: where a depthwise conv + BN
        # follows (MobileNet-v1), the loss is invariant to a per-channel rescaling of this unit's output, so with
        # beta = 0 at initialisation d gamma is a near-total cancellation (its own norm is rounding noise) while d beta
        # is not
        affine = max(float(dg_ref.double().norm()), float(db_ref.double().norm())) + 1e-30
        got = {'y': _rel(_nchw(out), y_ref), 'dw': _rel(params[cname + '.weight'].grad.cpu(), dw_ref),
               'dgamma': float((params[u['bn'] + '.weight'].grad.cpu().double() - dg_ref.double()).norm()) / affine,
               'dbeta': float((params[u['bn'] + '.bias'].grad.cpu().double() - db_ref.double()).norm()) / affine}
        if dx is not None:
            got['dx'] = _rel(_nchw(dx), dx_ref)
        if len(vjp) > 5:        # conv bias in front of a training-mode BN: the true gradient is sum(dz) == 0; the local
            # reference sums bf16-ROUNDED dz (storage emulation), i.e. pure rounding noise -- we write exact zeros
            assert float(params[cname + '.bias'].grad.abs().max()) == 0.0
            assert float(vjp[5].abs().max()) < 2e-2 * max(1.0, float(dw_ref.abs().max()))
        if max(got.values()) > 1e-2:
            print('  unit %s (%s, x %s): %s' % (cname, kind, tuple(u['x'].shape), {k: '%.2e' % v for k, v in got.items()}))
        for k, v in got.items():
            if v > worst.get(k, (0.0, ''))[0]:
                worst[k] = (v, cname)
    print('MobileNet teacher-forced units, worst rel-L2 per quantity: %s' % worst)
    # whole-network forward: every unit re-rounds to bf16 after a BatchNorm whose input has |mean| >> std (post-ReLU
    # depthwise stacks), so single flipped roundings are amplified layer by layer -- the bound is looser than T2's
    # 1e-3 for ResNets; the unit-level bounds below are the tight ones
    assert fwd_rel < 3e-1 and fwd_dloss < 3e-2, (fwd_rel, fwd_dloss)
    assert buf_worst[0] < 2e-2, buf_worst
    assert drift[0] > 1.0 - 2.0 * (1.0 - drift[1]) - 1e-3, drift
    assert worst['y'][0] < 1e-2, worst           # bf16 outputs: one rounding on top of the unit's own arithmetic
    assert worst['dx'][0] < 2e-2, worst
    assert worst['dw'][0] < 1e-2 and worst['dgamma'][0] < 1e-2 and worst['dbeta'][0] < 1e-2, worst
    assert ev_rel < 5e-2, ev_rel
    return ev_rel


def test_mobilenet_v2_against_reference_pinned_oracle():
    """MobileNet-v2 (config C4, depthwise path) against oracle.ref_model.forward_mobilenet_v2, which
    tests/test_oracle_golden.py pins to the unmodified reference.  Dropout is disabled so both sides see one network."""
    from convnet.pytorch_b200.models import mobilenet_v2

    def factory(**cfg):
        m = mobilenet_v2(**cfg)
        m.classifier[0].p = 0.0
        return m
    _mobilenet_parity(factory, 'features.conv0.0')


def test_mobilenet_v1_neighbour_family():
    """SURVEY.md section 8(f) row 4: MobileNet-v1 (models/mobilenet.py:39-156 of the reference; depthwise 3x3 WITH bias +
    BN + ReLU, 1x1 + BN + ReLU) on the MobileNet-v2 kernels -- same three-part check (the oracle restates the family;
    initialisation and parameter names are pinned to the reference by test_model_factories_match_reference_init).  The
    depthwise biases sit in front of a training-mode BatchNorm: zero gradient, folded into the running mean and into the
    eval-mode BN shift."""
    from convnet.pytorch_b200.models import mobilenet
    _mobilenet_parity(mobilenet, 'features.0')


@pytest.mark.parametrize("family", ["resnet_se", "resnext_se"])
def test_squeeze_excitation_neighbour_family(family):
    """SURVEY.md section 8(f) row 4: resnet_se / resnext_se (models/resnet.py:434-436, models/modules/se.py:6-25 of the
    reference) -- a squeeze-and-excitation gate on the residual branch, one gate shared by the blocks of a stage.
    T2 against the oracle (which restates SEBlock.forward and ties the shared parameters) and a training-mode eval."""
    from convnet.pytorch_b200 import models
    factory = getattr(models, family)
    ref, mine, x, y = _pair(factory, dict(dataset='imagenet', depth=50), (3, 64, 64), 1000, steps=3, batch=32)
    n_gate = sum(1 for n, _ in mine.named_parameters() if 'residual_block' in n)
    assert n_gate == 4 * 4, 'one SE gate (2 weights + 2 biases) per stage, shared by its blocks'
    _check_against_bf16_oracle(mine, ref, x, y)
    ref.eval(); mine.eval()
    with torch.no_grad():
        a, b = mine(x), ref(x.to(torch.bfloat16).float())
    assert _rel(a, b) < 3e-2


def test_resnext50_grouped_against_bf16_oracle():
    """ResNeXt (32 groups, via block-diagonal dense expansion) vs the bf16-emulating oracle."""
    from convnet.pytorch_b200.models import resnext
    ref, mine, x, y = _pair(resnext, dict(dataset='imagenet', depth=50), (3, 64, 64), 1000, steps=3, batch=32)
    _check_against_bf16_oracle(mine, ref, x, y)


def test_resnext20_cifar_against_bf16_oracle():
    """CIFAR ResNeXt (groups 4 / 8 / 16): the C != K stage entries (16 -> 64, 64 -> 128 and 128 -> 256) run on the dense
    block-diagonal expansion of b200_group_weight_pack, the other grouped convolutions as well (C % 128 != 0 or
    64 % (C/g) != 0), vs the bf16-emulating oracle."""
    from convnet.pytorch_b200.models import resnext
    ref, mine, x, y = _pair(resnext, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, batch=32)
    _check_against_bf16_oracle(mine, ref, x, y)


def test_resnext101_32x4d_config_c3():
    """BASELINE config C3's model (ResNeXt-101 32x4d: depth 101, 32 groups, C/g = 4..32): T2 against the bf16 oracle
    at 64 px and T1 against stock torch fp32 (cuDNN grouped convolutions) at the full 224 px resolution."""
    from convnet.pytorch_b200.models import resnext
    ref, mine, x, y = _pair(resnext, dict(dataset='imagenet', depth=101), (3, 64, 64), 1000, steps=3, batch=32)
    _check_against_bf16_oracle(mine, ref, x, y)
    del ref, mine
    ref, mine, x, y = _pair(resnext, dict(dataset='imagenet', depth=101), (3, 224, 224), 1000, steps=3, batch=32)
    _check_step(ref, mine, x, y)


@pytest.mark.parametrize("size,batch", [(128, 97), (160, 67), (256, 196), (288, 155)])
def test_resnet50_mixmatch_shapes(size, batch):
    """Mix&Match input sizes with odd / B+ batches (BASELINE config C5: 196 @ 256 px and 155 @ 288 px are the B+
    batches of mixsize_config at base_device_batch=256): no shape-specialised code path may break, T1 bounds."""
    from convnet.pytorch_b200.models import resnet
    ref, mine, x, y = _pair(resnet, dict(dataset='imagenet', depth=50), (3, size, size), 1000, steps=3, batch=batch)
    _check_step(ref, mine, x, y)


def test_trainer_cuda_graph_replay_matches_eager():
    """Trainer.train on the B200 path replays forward+loss+backward from a CUDA graph after two eager steps;
    parameters, BN statistics and meters after 6 steps must match a run with graphs disabled."""
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    _setup()
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(16, 3, 64, 64, generator=g), torch.randint(0, 1000, (16,), generator=g))
               for _ in range(6)]
    results = []
    for use_graphs in (False, True):
        torch.manual_seed(123)
        model = resnet(dataset='imagenet', depth=18)
        convert_b200(model, 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9)
        tr.use_graphs = use_graphs
        res = tr.train(batches)
        assert (tr.graph_replays > 0) == use_graphs, 'graph path %s' % ('not taken' if use_graphs else 'taken')
        if use_graphs:
            assert tr.graph_replays == len(batches) - 2 and tr.graph_replayed_launches > 100
        results.append((res, {k: v.detach().float().clone() for k, v in model.state_dict().items()}))
    (r0, s0), (r1, s1) = results
    assert abs(r0['loss'] - r1['loss']) < 2e-3 * max(1.0, abs(r0['loss']))
    for k in s0:
        assert _rel(s1[k], s0[k]) < 2e-3, '%s: %.3e' % (k, _rel(s1[k], s0[k]))


@pytest.mark.parametrize("family", ["resnet50", "resnext50", "resnext20_cifar"])
def test_eval_with_folded_batchnorm(family):
    """Inference path: BN folded into the conv weights + epilogue bias (utils/absorb_bn.py:18-48 of the reference)
    must agree with the unfolded kernels and with stock torch eval; the folded-weight cache must follow parameter
    and running-statistics updates.  Grouped weights are folded through b200_group_weight_pack (CIFAR ResNeXt: also
    its dense C != K expansion)."""
    from convnet.pytorch_b200 import engine
    from convnet.pytorch_b200.models import resnet, resnext
    if family == "resnext20_cifar":
        ref, mine, x, y = _pair(resnext, dict(dataset='cifar10', depth=20), (3, 32, 32), 10, steps=3, batch=8)
    else:
        factory = resnet if family == "resnet50" else resnext
        ref, mine, x, y = _pair(factory, dict(dataset='imagenet', depth=50), (3, 64, 64), 1000, steps=3, batch=8)
    saved = engine.FOLD_BN_EVAL
    try:
        ref.eval(); mine.eval()
        with torch.no_grad():
            engine.FOLD_BN_EVAL = False
            a0 = mine(x)
            engine.FOLD_BN_EVAL = True
            a1 = mine(x)
            a2 = mine(x)                      # second call: cached folded weights
            b = ref(x.to(torch.bfloat16).float())
        assert torch.equal(a1, a2)
        assert _rel(a1, a0) < 2e-2, 'folded vs unfolded %.3e' % _rel(a1, a0)
        assert _rel(a1, b) < 3e-2, 'folded vs torch eval %.3e' % _rel(a1, b)
        # one training forward/backward moves the running statistics: the cache must be rebuilt
        mine.train()
        mine._b200.arena.zero_grad()
        F.cross_entropy(mine(x), y).backward()
        mine.eval()
        with torch.no_grad():
            engine.FOLD_BN_EVAL = False
            c0 = mine(x)
            engine.FOLD_BN_EVAL = True
            c1 = mine(x)
        assert _rel(c1, c0) < 2e-2, 'after update: folded vs unfolded %.3e' % _rel(c1, c0)
        assert _rel(c1, a1) > 1e-4, 'folded weights were not refreshed after the running statistics changed'
    finally:
        engine.FOLD_BN_EVAL = saved
