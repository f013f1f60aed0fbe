"""Activation checkpointing (``checkpoint_segments`` of the ImageNet ResNets, reference models/resnet.py:236-239 and
models/modules/checkpoint.py) on the CPU: the model against what the unmodified reference produced
(tests/golden/checkpoint_segments.npz, written by tools/make_checkpoint_golden.py) -- init, state_dict layout,
parameter order, the weight-decay set and an fp64 training step whose checkpointed BatchNorms update their running
statistics twice -- the segment plan, the command line, and the combination that raises.  CPU only."""
import hashlib
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'checkpoint_segments.npz')


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD))


def bn_state(name, C):
    """tools/make_checkpoint_golden.py: deterministic BN parameters / buffers of the fp64 step"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name)) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def _close(a, b, tol=1e-9):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    assert np.all(np.abs(a - b) <= tol * np.maximum(np.abs(b), 1.0)), float(np.max(np.abs(a - b)))


@pytest.mark.parametrize('s', [1, 2, 4])
def test_init_layout_order_and_decay_match_reference(gold, s):
    from convnet.pytorch_b200 import models
    from convnet.pytorch_b200.utils import regularization
    tag = 'resnet50_s%d' % s
    torch.manual_seed(123)
    model = models.resnet(dataset='imagenet', depth=50, checkpoint_segments=s)
    sd = model.state_dict()
    assert list(sd.keys()) == list(gold[tag + '/keys'])
    assert [','.join(map(str, v.shape)) for v in sd.values()] == list(gold[tag + '/shapes'])
    got = [hashlib.sha256(v.contiguous().numpy().tobytes()).hexdigest() for v in sd.values()]
    bad = [k for k, a, b in zip(sd.keys(), got, gold[tag + '/sha256']) if a != b]
    assert not bad, 'init differs from the reference in %s' % bad[:5]
    assert [n for n, _ in model.named_parameters()] == list(gold[tag + '/params'])
    reg = dict(model.regime[0]['regularizer'])
    reg.pop('name')
    wd = regularization.WeightDecay(model, **reg)
    assert [n for n, _ in wd.named_parameters()] == list(gold[tag + '/decayed'])


@pytest.mark.parametrize('s', [1, 2])
def test_fp64_step_matches_reference(gold, s):
    """logits, loss, gradients and the running buffers after one step; BNs inside checkpointed segments were updated
    twice (num_batches_tracked 2), the others once"""
    from convnet.pytorch_b200 import models
    tag = 'step_s%d' % s
    torch.manual_seed(123)
    model = models.resnet(dataset='imagenet', depth=18, checkpoint_segments=s).double()
    with torch.no_grad():
        for n, m in model.named_modules():
            if isinstance(m, nn.BatchNorm2d):
                for k, v in bn_state(n, m.num_features).items():
                    getattr(m, k).copy_(v)
    x = torch.from_numpy(gold['step/x_codes']).double() / 16
    y = torch.from_numpy(gold['step/target'])
    model.train()
    logits = model(x)
    loss = nn.functional.cross_entropy(logits, y)
    loss.backward()
    _close(logits.detach().numpy(), gold[tag + '/logits'])
    _close(loss.item(), gold[tag + '/loss'])
    assert [n for n, _ in model.named_parameters()] == list(gold[tag + '/grad_names'])
    _close([p.grad.norm().item() for _, p in model.named_parameters()], gold[tag + '/grad_norms'])
    sd = model.state_dict()
    _close(np.concatenate([sd[k].numpy().ravel() for k in gold[tag + '/buffer_names']]), gold[tag + '/buffers'])
    assert [int(sd[k]) for k in gold[tag + '/tracked_names']] == gold[tag + '/tracked'].tolist()


def test_segment_plan():
    """the [start, end) block ranges torch.utils.checkpoint.checkpoint_sequential recomputes, per stage"""
    from convnet.pytorch_b200.models.modules.checkpoint import CheckpointModule
    seq = nn.Sequential(*[nn.Identity() for _ in range(6)])
    assert CheckpointModule(seq, 1).segments() == [(0, 6)]
    assert CheckpointModule(seq, 2).segments() == [(0, 3)]
    assert CheckpointModule(seq, 4).segments() == [(0, 1), (1, 2), (2, 3)]
    assert CheckpointModule(nn.Sequential(*seq[:3]), 3).segments() == [(0, 1), (1, 2)]
    with pytest.raises(ValueError):
        CheckpointModule(nn.Identity(), 2)


def test_eval_and_no_grad_forwards_do_not_recompute():
    from convnet.pytorch_b200 import models
    model = models.resnet(dataset='imagenet', depth=18, checkpoint_segments=1)
    x = torch.randn(2, 3, 32, 32)
    model.eval()
    model(x)
    model.train()
    with torch.no_grad():
        model(x)
    assert all(int(m.num_batches_tracked) == 1 for m in model.modules() if isinstance(m, nn.BatchNorm2d))


def test_sync_bn_with_checkpointing_raises(tmp_path):
    from convnet.pytorch_b200 import main as cli
    with pytest.raises(NotImplementedError):
        cli.main(['--model', 'resnet', '--model-config', "{'depth': 18, 'checkpoint_segments': 1}", '--dataset',
                  'synthetic_imagenet', '--input-size', '32', '--device', 'cpu', '-b', '8', '--epochs', '1',
                  '--max-steps', '1', '--workers', '0', '--sync-bn', '--results-dir', str(tmp_path), '--save', 'sync'])


def test_cli_run_and_evaluate(tmp_path, monkeypatch):
    """the C1 command line (CPU, stock torch layers) on a checkpointed ImageNet ResNet: two training steps, validation,
    a checkpoint with the reference's keys, then evaluate.py on it with and without --absorb-bn"""
    from convnet.pytorch_b200 import main as cli
    from convnet.pytorch_b200 import evaluate as ev
    from convnet.pytorch_b200 import models
    monkeypatch.setenv('B200_SYNTHETIC_LENGTH', '32')
    cli.main(['--model', 'resnet', '--model-config', "{'depth': 18, 'checkpoint_segments': 2}", '--dataset',
              'synthetic_imagenet', '--input-size', '32', '--device', 'cpu', '-b', '8', '--epochs', '1',
              '--max-steps', '2', '--workers', '0', '--results-dir', str(tmp_path), '--save', 'ckpt'])
    path = tmp_path / 'ckpt' / 'checkpoint.pth.tar'
    sd = torch.load(path, map_location='cpu', weights_only=False)['state_dict']
    assert list(sd) == list(models.resnet(dataset='imagenet', depth=18, checkpoint_segments=2).state_dict())
    assert int(sd['layer1.module.0.bn1.num_batches_tracked']) == 2 * int(sd['layer1.module.1.bn1.num_batches_tracked'])
    args = [str(path), '--dataset', 'synthetic_imagenet', '--input-size', '32', '--device', 'cpu', '-b', '8',
            '--workers', '0']
    base = ev.main(args)
    absorbed = ev.main(args + ['--absorb-bn'])
    assert abs(base['loss'] - absorbed['loss']) < 1e-4 * max(1.0, base['loss']) and base['prec1'] == absorbed['prec1']
