"""L1 batch normalization (``resnet(bn_norm='L1')``, reference models/modules/lp_norm.py:238-291) on the CPU: the model
against what the unmodified reference produced (tests/golden/l1_norm.npz, written by tools/make_l1_norm_golden.py) --
init, state_dict layout, parameter order, the weight-decay set and an fp64 training step -- the L1 oracle
(tests/l1_oracle.py), the combinations that raise, and the command line.  CPU only."""
import hashlib
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'l1_norm.npz')
MODELS = {'resnet20': dict(dataset='cifar10', depth=20), 'resnet18': dict(dataset='imagenet', depth=18)}


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD))


def bn_state(name, C):
    """tools/make_l1_norm_golden.py: deterministic BN parameters / buffers of the fp64 step"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name)) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def _model(tag):
    from convnet.pytorch_b200 import models
    torch.manual_seed(123)
    return models.resnet(bn_norm='L1', **MODELS[tag])


@pytest.mark.parametrize('tag', sorted(MODELS))
def test_init_layout_and_order_match_reference(gold, tag):
    model = _model(tag)
    sd = model.state_dict()
    assert list(sd.keys()) == list(gold[tag + '/keys'])
    assert [','.join(map(str, v.shape)) for v in sd.values()] == list(gold[tag + '/shapes'])
    got = [hashlib.sha256(v.contiguous().numpy().tobytes()).hexdigest() for v in sd.values()]
    bad = [k for k, a, b in zip(sd.keys(), got, gold[tag + '/sha256']) if a != b]
    assert not bad, 'init differs from the reference in %s' % bad[:5]
    assert [n for n, _ in model.named_parameters()] == list(gold[tag + '/params'])


@pytest.mark.parametrize('tag', sorted(MODELS))
def test_weight_decay_set_matches_reference(gold, tag):
    from convnet.pytorch_b200.utils import regularization
    model = _model(tag)
    reg = dict(model.regime[0]['regularizer'])
    reg.pop('name')
    wd = regularization.WeightDecay(model, **reg)
    assert [n for n, _ in wd.named_parameters()] == list(gold[tag + '/decayed'])


def _step_inputs(gold):
    x = torch.from_numpy(gold['step/x_codes']).double() / 16
    return x, torch.from_numpy(gold['step/target'])


def _step_model(gold):
    from convnet.pytorch_b200.models.modules.lp_norm import L1BatchNorm2d
    model = _model('resnet20').double()
    with torch.no_grad():
        for n, m in model.named_modules():
            if isinstance(m, L1BatchNorm2d):
                for k, v in bn_state(n, m.num_features).items():
                    getattr(m, k).copy_(v)
    return model


def _close(a, b, tol=1e-9):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.all(np.abs(a - b) <= tol * np.maximum(np.abs(b), 1.0)), float(np.max(np.abs(a - b)))


def test_fp64_step_module_matches_reference(gold):
    model = _step_model(gold)
    x, y = _step_inputs(gold)
    model.train()
    logits = model(x)
    loss = nn.functional.cross_entropy(logits, y)
    loss.backward()
    _close(logits.detach().numpy(), gold['step/logits'])
    _close(loss.item(), gold['step/loss'])
    assert [n for n, _ in model.named_parameters()] == list(gold['step/grad_names'])
    _close([p.grad.norm().item() for _, p in model.named_parameters()], gold['step/grad_norms'])
    sd = model.state_dict()
    _close(np.concatenate([sd[k].numpy().ravel() for k in gold['step/buffer_names']]), gold['step/buffers'])


def test_fp64_step_oracle_matches_reference(gold):
    import l1_oracle
    sd = {k: v.clone() for k, v in _step_model(gold).state_dict().items()}
    x, y = _step_inputs(gold)
    logits, loss, grads, bufs = l1_oracle.loss_and_grads(sd, x, y)
    _close(logits.numpy(), gold['step/logits'])
    _close(float(loss), gold['step/loss'])
    _close([grads[n].norm().item() for n in gold['step/grad_names']], gold['step/grad_norms'])
    _close(np.concatenate([bufs[k].numpy().ravel() for k in gold['step/buffer_names']]), gold['step/buffers'])


def test_eval_mode_and_absorb_fold():
    """zero running buffers: an untrained model's L1 layers output their bias; --absorb-bn folds with the L1 formula"""
    from convnet.pytorch_b200.models.modules.lp_norm import L1BatchNorm2d
    from convnet.pytorch_b200.evaluate import absorb_bn_torch
    bn = L1BatchNorm2d(8).double().eval()
    with torch.no_grad():
        bn.bias.copy_(torch.arange(8.0))
    x = torch.randn(2, 8, 3, 3, dtype=torch.float64)
    assert torch.equal(bn(x), torch.arange(8.0, dtype=torch.float64).view(1, 8, 1, 1).expand(2, 8, 3, 3))
    torch.manual_seed(0)
    net = nn.Sequential(nn.Conv2d(3, 8, 3, bias=False), L1BatchNorm2d(8)).double()
    with torch.no_grad():
        net[1].running_mean.uniform_(-1, 1)
        net[1].running_var.uniform_(0.5, 2)
        net[1].weight.uniform_(0.5, 1.5)
        net[1].bias.uniform_(-1, 1)
    net.eval()
    x = torch.randn(2, 3, 9, 9, dtype=torch.float64)
    ref = net(x)
    folded = absorb_bn_torch(net)
    assert isinstance(folded[1], nn.Identity)
    assert torch.allclose(folded(x), ref, rtol=1e-12, atol=1e-12)


def test_factory_leaves_torch_untouched():
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.models.modules.lp_norm import L1BatchNorm2d
    bn_class = nn.BatchNorm2d
    for make in (models.resnet, models.resnet_se):
        m = make(dataset='cifar10', depth=8, bn_norm='L1')
        kinds = {type(x) for x in m.modules() if isinstance(x, (nn.BatchNorm2d, L1BatchNorm2d))}
        assert kinds == {L1BatchNorm2d}
    assert nn.BatchNorm2d is bn_class and torch.nn.modules.batchnorm.BatchNorm2d is bn_class
    m = models.resnet(dataset='cifar10', depth=8)
    assert not any(isinstance(x, L1BatchNorm2d) for x in m.modules())
    assert sum(isinstance(x, nn.BatchNorm2d) for x in m.modules()) == 9     # stem, 3 blocks x 2, 2 downsamples


def test_out_of_scope_combinations_raise(tmp_path):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200 import main as cli
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.optim import OptimRegime
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    with pytest.raises(NotImplementedError):
        models.resnet(dataset='cifar10', depth=8, bn_norm='TopK')
    with pytest.raises(NotImplementedError):
        models.resnet(dataset='cifar10', depth=8, quantize=True)
    with pytest.raises(NotImplementedError):
        models.resnet(dataset='cifar10', depth=8, bn_norm='L1', quantize=True)
    model = models.resnet(dataset='cifar10', depth=8, bn_norm='L1')
    tr = Trainer(model, CrossEntropyLoss(), OptimRegime(model, model.regime), device_ids=None, device='cpu',
                 print_freq=1000)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(NotImplementedError):
        tr.calibrate_bn([(torch.randn(4, 3, 32, 32), torch.randint(0, 10, (4,)))], num_steps=1)
    assert all(torch.equal(before[k], v) for k, v in model.state_dict().items())
    with pytest.raises(NotImplementedError):
        cli.main(['--model', 'resnet', '--model-config', "{'depth': 8, 'bn_norm': 'L1'}", '--dataset',
                  'synthetic_cifar10', '--device', 'cpu', '-b', '8', '--epochs', '1', '--max-steps', '1', '--workers',
                  '0', '--sync-bn', '--results-dir', str(tmp_path), '--save', 'sync'])


def test_cli_l1_run(tmp_path):
    """configuration C1 with bn_norm L1 through the command line: two training steps, validation, checkpoint"""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 20, 'bn_norm': 'L1'}", '--dataset',
              'synthetic_cifar10', '--device', 'cpu', '-b', '16', '--epochs', '1', '--max-steps', '2', '--workers', '0',
              '--results-dir', str(tmp_path), '--save', 'l1'])
    ck = torch.load(tmp_path / 'l1' / 'checkpoint.pth.tar', map_location='cpu', weights_only=False)
    sd = ck['state_dict']
    assert 'bn1.num_batches_tracked' not in sd and list(k for k in sd if k.startswith('bn1.')) == \
        ['bn1.bias', 'bn1.weight', 'bn1.running_mean', 'bn1.running_var']
    assert float(sd['bn1.running_var'].abs().sum()) > 0      # the running scale moved off its zero start
