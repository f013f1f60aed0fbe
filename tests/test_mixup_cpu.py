"""MixUp / CutMix (reference utils/mixup.py, trainer.py:44-51,119-138) on the CPU: the Trainer against the draws, mixed
inputs, losses and gradients the unmodified reference produced (tests/golden/mixup.npz, written by
tools/make_mixup_golden.py), the oracle with the soft target, and the command line.  CPU only."""
import hashlib
import os
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
FLAGS = {'mixup': dict(mixup=0.2), 'cutmix': dict(cutmix=1.0), 'both': dict(mixup=0.2, cutmix=1.0)}
SAMPLES_PER_PARAM = 64          # tools/make_mixup_golden.py


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def soft_target(target, n_cls, soft):
    """The reference's mixed target (utils/mixup.py:37-45, trainer.py:137-138): soft = (t2, lam) ->
    lam*onehot(target) + (1-lam)*onehot(t2), formed in fp32 with the fp32 lam."""
    t2, lam = soft
    lam = torch.tensor([float(lam)], dtype=torch.float32).view(1, 1)
    return lam * F.one_hot(target, n_cls).float() + (1. - lam) * F.one_hot(t2, n_cls).float()


def soft_cross_entropy(logits, target, soft):
    """-sum_c q_c log_softmax_c, mean over the batch (utils/cross_entropy.py:53-54 of the reference: the float-target
    branch, where label smoothing does not apply)."""
    q = soft_target(target, logits.size(-1), soft).to(logits.dtype)
    return (-(q * F.log_softmax(logits, dim=-1)).sum(-1)).mean()


def oracle_soft_loss_and_grads(sd, x, y, soft, quant=False):
    """oracle.ref_model's forward with the soft-target loss of a mixed step (``x`` is the mixed batch): logits, loss,
    {param: grad}, updated BN buffers -- the shape of ref_model.loss_and_grads."""
    from oracle import ref_model
    names = ref_model.param_names(sd)
    work = {k: (v.detach().clone().requires_grad_(True) if k in names else v) for k, v in sd.items()}
    bufs = {}
    logits = ref_model.forward(work, x, training=True, buffers_out=bufs, quant=quant)
    loss = soft_cross_entropy(logits, y, soft)
    grads = torch.autograd.grad(loss, [work[k] for k in names])
    return logits.detach(), loss.detach(), dict(zip(names, grads)), bufs


def _digest(t):
    return hashlib.sha256(t.detach().contiguous().float().numpy().tobytes()).hexdigest()


def _fixture():
    z = np.load(os.path.join(GOLD, 'mixup.npz'))
    xs = [torch.from_numpy(c).float() / 16 for c in z['x_codes']]      # exact: the pixels are multiples of 1/16
    ys = [torch.from_numpy(y) for y in z['y']]
    return z, xs, ys


def _grad_samples(grads, names):
    """the fixture's sample of every gradient: seeded indices, up to SAMPLES_PER_PARAM per parameter."""
    g = torch.Generator().manual_seed(17)
    out = []
    for n in names:
        idx = torch.randperm(grads[n].numel(), generator=g)[:SAMPLES_PER_PARAM].sort().values
        out.append(grads[n].flatten()[idx])
    return torch.cat(out)


def _check_grads(grads, z, tol=2e-4):
    """every gradient's norm and its seeded sample of entries within ``tol`` relative."""
    names = [str(n) for n in z['grad_names']]
    assert sorted(names) == sorted(grads)
    ref_norms = z['grad_norms']
    for n, r in zip(names, ref_norms):
        assert abs(float(grads[n].double().norm()) - r) <= tol * r + 1e-12, n
    mine = _grad_samples(grads, names)
    ref = torch.from_numpy(z['grad_samples'])
    off = 0
    for n in names:
        k = min(SAMPLES_PER_PARAM, grads[n].numel())
        a, b = mine[off:off + k], ref[off:off + k]
        assert float((a - b).double().norm()) <= tol * max(float(b.double().norm()), 1e-3 * float(ref.double().norm())), n
        off += k
    assert _rel(mine, ref) < tol


def _run_trainer(z, xs, ys):
    """Our Trainer on the stock-torch ResNet-20 over the fixture's batches and seeds: per step the module that drew
    the mixing, the mixed input the model received and the loss; the parameters and buffers before the fixture's
    recorded step and the gradients it produced."""
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.manual_seed(123)
    model = models.resnet(dataset='cifar10', depth=20)
    opt = OptimRegime(model, model.regime)
    seen, out = [], []
    model.register_forward_pre_hook(lambda m, inp: seen.append(inp[0].detach().clone()))
    grad_step, grads, state = int(z['grad_step']), {}, None
    random.seed(5)
    np.random.seed(5)
    torch.manual_seed(5)
    for i, kind in enumerate(str(k) for k in z['steps']):
        tr = Trainer(model, CrossEntropyLoss(), opt, device_ids=None, device='cpu', dtype=torch.float, print_freq=1000,
                     **FLAGS[kind])
        tr.training_steps = i
        x, y = xs[i].clone(), ys[i]
        if i == grad_step:
            state = {k: v.detach().clone() for k, v in model.state_dict().items()}
            step = opt.step

            def rec_step(*a, **kw):
                grads.update({n: p.grad.clone() for n, p in model.named_parameters()})
                return step(*a, **kw)
            opt.step = rec_step
        _, loss, _ = tr._step(x, y, training=True)
        if i == grad_step:
            del opt.step
        assert torch.equal(x, xs[i]), 'the caller\'s batch was modified'
        out.append((tr.last_mix, seen[-1], float(loss)))
    return out, grads, state


def test_trainer_reproduces_reference_mixup_and_cutmix_steps():
    """Draws equal step by step, mixed inputs bit for bit (SHA-256 of the fp32 bytes), losses within 1e-5, the
    recorded step's gradients within 2e-4 relative (the bound of test_oracle_reproduces_reference_step_resnet20; here
    on every gradient's norm and on a fixed sample of its entries)."""
    from convnet.pytorch_b200.utils.mixup import CutMix
    z, xs, ys = _fixture()
    steps, grads, _ = _run_trainer(z, xs, ys)
    for i, (mixer, mixed, loss) in enumerate(steps):
        assert torch.equal(mixer.mix_index, torch.from_numpy(z['perm/%d' % i])), i
        assert torch.equal(mixer.mix_values, torch.from_numpy(z['lam/%d' % i])), i
        assert isinstance(mixer, CutMix) == bool(z['cutmix/%d' % i]), i
        if isinstance(mixer, CutMix):
            assert list(mixer.box) == [int(v) for v in z['box/%d' % i]], i
        assert _digest(mixed) == str(z['mixed_sha256/%d' % i]), 'mixed input of step %d' % i
        assert abs(loss - float(z['loss/%d' % i])) < 1e-5, (i, loss, float(z['loss/%d' % i]))
    _check_grads(grads, z)


def test_both_flags_use_cutmix_with_the_mixup_alpha():
    """mix_val = mixup or cutmix with a CutMix module when cutmix is set: the fixture's last step ran with both flags
    (CutMix, alpha 0.2) and the Trainer reproduced it above; here the selection itself."""
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.mixup import CutMix, MixUp
    tr = Trainer(torch.nn.Linear(2, 2), None, device_ids=None, device='cpu', mixup=0.2, cutmix=1.0)
    seen = []
    orig = CutMix.sample
    CutMix.sample = lambda self, alpha, n, sample_batch=False: (seen.append(alpha), orig(self, alpha, n))[1]
    try:
        m = tr._draw_mix(4)
    finally:
        CutMix.sample = orig
    assert isinstance(m, CutMix) and seen == [0.2]
    assert type(Trainer(torch.nn.Linear(2, 2), None, device_ids=None, device='cpu', mixup=0.2)._draw_mix(4)) is MixUp


def test_oracle_soft_target_reproduces_reference_step():
    """oracle.ref_model's forward with the soft target (t2, lam), on the state before the recorded step and its mixed
    input (both pinned by the test above): the reference's loss and gradients."""
    from convnet.pytorch_b200.utils.mixup import CutMix
    z, xs, ys = _fixture()
    steps, _, state = _run_trainer(z, xs, ys)
    i = int(z['grad_step'])
    mixer, mixed, _ = steps[i]
    assert isinstance(mixer, CutMix) and _digest(mixed) == str(z['mixed_sha256/%d' % i])
    y = ys[i]
    perm = torch.from_numpy(z['perm/%d' % i])
    _, loss, g, _ = oracle_soft_loss_and_grads(state, mixed, y, (y[perm], float(z['lam/%d' % i][0])))
    assert abs(float(loss) - float(z['loss/%d' % i])) < 1e-5
    _check_grads(g, z)


def test_cutmix_box_edges():
    """The box of utils/mixup.py:57-73: half-widths int(H*sqrt(1-lam))//2, clipped; lam -> uncovered fraction."""
    from convnet.pytorch_b200.utils.mixup import CutMix
    m = CutMix()
    for lam, H, W in ((1.0, 32, 32), (0.0, 32, 32), (0.37, 31, 17), (0.9, 7, 64)):
        m.mix_values = torch.tensor([lam])
        state = np.random.get_state()
        cy, cx = np.random.randint(H), np.random.randint(W)
        np.random.set_state(state)
        r0, r1, c0, c1 = m.draw_box(H, W)
        hh, hw = int(H * np.sqrt(1.0 - np.float32(lam).item())) // 2, int(W * np.sqrt(1.0 - np.float32(lam).item())) // 2
        assert (r0, r1, c0, c1) == (max(cy - hh, 0), min(cy + hh, H), max(cx - hw, 0), min(cx + hw, W))
        assert float(m.mix_values) == np.float32(1 - (r1 - r0) * (c1 - c0) / (H * W))
    x1, x2 = torch.zeros(2, 3, 8, 8), torch.ones(2, 3, 8, 8)
    m.mix_values = torch.tensor([0.0])
    out = m.mix_image(x1, x2)
    r0, r1, c0, c1 = m.box
    assert float(out.sum()) == 2 * 3 * (r1 - r0) * (c1 - c0)


def test_mixing_applies_only_when_training():
    """validate / calibrate_bn never mix; eval-mode modules are the identity."""
    from convnet.pytorch_b200.utils.mixup import MixUp
    m = MixUp()
    m.sample(0.2, 4)
    x = torch.randn(4, 3)
    m.eval()
    assert m(x) is x
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.manual_seed(0)
    model = models.resnet(dataset='cifar10', depth=8)
    tr = Trainer(model, CrossEntropyLoss(), device_ids=None, device='cpu', mixup=0.2)
    g = torch.Generator().manual_seed(1)
    batches = [(torch.randn(4, 3, 32, 32, generator=g), torch.randint(0, 10, (4,), generator=g))]
    state = np.random.get_state()
    tr.validate(batches)
    assert tr.last_mix is None and np.array_equal(np.random.get_state()[1], state[1])


def test_unsupported_mixing_combinations_raise():
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.lib import B200Error
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.manual_seed(0)
    model = models.resnet(dataset='cifar10', depth=8)
    opt = OptimRegime(model, model.regime)
    tr = Trainer(model, CrossEntropyLoss(), opt, device_ids=None, device='cpu', mixup=0.2)
    x, y = torch.randn(4, 2, 3, 32, 32), torch.randint(0, 10, (4,))
    with pytest.raises(NotImplementedError, match='average_output'):
        tr.train([(x, y)], average_output=True)
    with pytest.raises(B200Error, match='uint8'):
        tr._step(torch.zeros(4, 3, 32, 32, dtype=torch.uint8), y, training=True)
    # duplicates without averaging: the permutation runs over all B*D rows
    res = tr.train([(x, y)])
    assert tr.last_mix.mix_index.numel() == 8 and res['loss'] > 0
    with pytest.raises(NotImplementedError):
        models.resnet(dataset='cifar10', depth=20, mixup=True)


@pytest.mark.parametrize('extra', [['--mixup', '0.2'], ['--cutmix', '1.0'], ['--mixup', '0.2', '--cutmix', '1.0']])
def test_cli_cpu_run_with_mixing(tmp_path, extra):
    """Config C1 (ResNet-20, synthetic CIFAR-10, CPU) through main.py with --mixup / --cutmix."""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 20}", '--dataset', 'synthetic_cifar10',
              '--device', 'cpu', '-b', '16', '--epochs', '1', '--max-steps', '2', '--workers', '0',
              '--results-dir', str(tmp_path), '--save', 'mix'] + extra)
    import csv
    rows = list(csv.DictReader(open(tmp_path / 'mix' / 'results.csv')))
    assert len(rows) == 1 and float(rows[0]['training loss']) > 0


def test_cli_cpu_run_with_cutmix_regime(tmp_path):
    """regime='cutmix' (the 300-epoch step schedule of models/resnet.py) with --cutmix, CPU, small ImageNet ResNet."""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 18, 'regime': 'cutmix'}", '--dataset',
              'synthetic_imagenet', '--input-size', '32', '--device', 'cpu', '-b', '8', '--epochs', '1',
              '--max-steps', '2', '--workers', '0', '--results-dir', str(tmp_path), '--save', 'cutmix', '--cutmix', '1.0'])
    import csv
    rows = list(csv.DictReader(open(tmp_path / 'cutmix' / 'results.csv')))
    assert len(rows) == 1 and float(rows[0]['training loss']) > 0


def test_evaluate_accepts_mixup_flag(tmp_path, monkeypatch):
    """evaluate.py takes --mixup for CLI parity with the reference (evaluate.py:70-71); evaluation never mixes."""
    from convnet.pytorch_b200 import main as cli
    from convnet.pytorch_b200 import evaluate as ev
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 8}", '--dataset', 'synthetic_cifar10',
              '--device', 'cpu', '-b', '16', '--epochs', '1', '--max-steps', '1', '--workers', '0',
              '--results-dir', str(tmp_path), '--save', 'run'])
    ck = str(tmp_path / 'run' / 'checkpoint.pth.tar')
    monkeypatch.setenv('B200_SYNTHETIC_LENGTH', '32')
    args = [ck, '--dataset', 'synthetic_cifar10', '--device', 'cpu', '-b', '16', '--workers', '0']
    base, mixed = ev.main(args), ev.main(args + ['--mixup', '0.2'])
    assert base['loss'] == mixed['loss'] and base['prec1'] == mixed['prec1']
