"""In-block dropout of CIFAR ResNets (``resnet(dropout=p)``, reference models/resnet.py:81-118) on the CPU: the Philox
mask stream of csrc/dropout.cu restated in numpy (tests/dropout_oracle.py) against the Random123 known-answer vectors
and a scalar restatement, the host-side threshold, an fp64 training step of the module and of the dropout oracle
against what the unmodified reference produced with the same masks (tests/golden/wrn_dropout.npz, written by
tools/make_wrn_dropout_golden.py), and the Wide-ResNet command line.  CPU only."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

import dropout_oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'wrn_dropout.npz')
MODELS = {'wrn16_4': dict(dataset='cifar10', depth=16, width=[64, 128, 256], dropout=0.3),
          'resnet20': dict(dataset='cifar10', depth=20, dropout=0.3)}

# Random123 known-answer vectors of philox4x32-10: counter, key -> output
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD))


@pytest.mark.parametrize('i', range(len(KAT)))
def test_philox_known_answers(i):
    ctr, key, want = KAT[i]
    got = dropout_oracle.philox4x32_10(np.array([ctr], dtype=np.uint32), key)[0]
    assert tuple(int(v) for v in got) == want


def _philox_scalar(ctr, key):
    M = 0xffffffff
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M, (p0 >> 32) ^ c3 ^ k1, p0 & M
        k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
    return c0, c1, c2, c3


@pytest.mark.parametrize('key,layer,C,M,p', [(0, 0, 8, 3, 0.3), (-1, 7, 16, 5, 0.5), (0x0123456789abcdef, 2, 24, 7, 0.1),
                                             (-0x7edcba9876543210, 31, 160, 2, 0.9), (1 << 40, 1, 64, 9, 0.3)])
def test_mask_matches_scalar_restatement(key, layer, C, M, p):
    T, _ = dropout_oracle.threshold(p)
    got = dropout_oracle.keep_mask(key, layer, M, C, T)
    k = key & 0xffffffffffffffff
    kw = (k & 0xffffffff, k >> 32)
    for row in range(M):
        for c in range(C):
            g = (row * C + c) // 8
            w = _philox_scalar((g & 0xffffffff, g >> 32, layer, 0), kw)
            j = c % 8
            assert got[row, c] == (((w[j >> 1] >> (16 * (j & 1))) & 0xffff) < T), (row, c)


def test_threshold_and_scale():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    for p in (0.0, 0.1, 0.3, 0.5, 0.9, 1e-6, 0.999):
        T, c = ops.dropout_threshold(p)
        assert (T, c) == dropout_oracle.threshold(p)
        assert abs(T / 65536.0 - (1.0 - p)) <= 2.0 ** -17           # realised keep rate vs 1 - p
        assert c == float(np.float32(1.0 / (1.0 - p)))
    for p in (1.0, 1.5, -0.1):
        with pytest.raises(B200Error):
            ops.dropout_threshold(p)


def bn_state(name, C):
    """tools/make_wrn_dropout_golden.py: deterministic BN parameters / buffers of the fp64 step"""
    i = torch.arange(C, dtype=torch.float64)
    h = (sum(map(ord, name)) % 97) / 97.0
    return {'weight': 1.0 + 0.25 * torch.sin(i + h * 7), 'bias': 0.1 * torch.cos(1.3 * i + h * 5),
            'running_mean': 0.05 * torch.sin(0.7 * i + h), 'running_var': 1.0 + 0.2 * torch.cos(0.3 * i + h * 3)}


def _step_model(tag):
    from convnet.pytorch_b200 import models
    torch.manual_seed(123)
    model = models.resnet(**MODELS[tag]).double()
    with torch.no_grad():
        for n, m in model.named_modules():
            if isinstance(m, nn.BatchNorm2d):
                for k, v in bn_state(n, m.num_features).items():
                    getattr(m, k).copy_(v)
    return model


def _masks(gold, tag):
    out = {}
    for n in gold[tag + '/mask_names']:
        shape = tuple(gold[tag + '/mask_shape/' + n])
        bits = np.unpackbits(gold[tag + '/mask/' + n])[:int(np.prod(shape))]
        out[str(n)] = torch.from_numpy(bits.reshape(shape).astype(bool))
    return out


def _close(a, b, tol=1e-9):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert np.all(np.abs(a - b) <= tol * np.maximum(np.abs(b), 1.0)), float(np.max(np.abs(a - b)))


@pytest.mark.parametrize('tag', sorted(MODELS))
def test_fp64_step_module_matches_reference(gold, tag, monkeypatch):
    model = _step_model(tag)
    masks = _masks(gold, tag)
    by_module = {id(m.dropout): masks[n] for n, m in model.named_modules() if n in masks}
    assert len(by_module) == len(masks)
    monkeypatch.setattr(nn.Dropout, 'forward', lambda self, x: x * (by_module[id(self)].to(x.dtype) / (1 - self.p)))
    x = torch.from_numpy(gold[tag + '/x_codes']).double() / 16
    y = torch.from_numpy(gold[tag + '/target'])
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


@pytest.mark.parametrize('tag', sorted(MODELS))
def test_fp64_step_oracle_matches_reference(gold, tag):
    model = _step_model(tag)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    x = torch.from_numpy(gold[tag + '/x_codes']).double() / 16
    y = torch.from_numpy(gold[tag + '/target'])
    masks = _masks(gold, tag)
    spec = dropout_oracle.block_spec(model, *x.shape[:1], *x.shape[2:])
    assert sorted(s[0] for s in spec) == sorted(masks)
    assert all(tuple(masks[s[0]].shape) == (x.shape[0], s[2], s[3], s[4]) for s in spec)
    logits, loss, grads, bufs = dropout_oracle.loss_and_grads(sd, x, y, masks, 0.3)
    _close(logits.numpy(), gold[tag + '/logits'])
    _close(float(loss), gold[tag + '/loss'])
    _close([grads[n].norm().item() for n in gold[tag + '/grad_names']], gold[tag + '/grad_norms'])
    _close(np.concatenate([bufs[k].numpy().ravel() for k in gold[tag + '/buffer_names']]), gold[tag + '/buffers'])


def test_cli_wide_resnet_dropout_run(tmp_path):
    """the Wide-ResNet command of the README (WRN-28-10, 'wide-resnet' regime, dropout 0.3) through the command line:
    two training steps, validation, checkpoint"""
    from convnet.pytorch_b200 import main as cli
    cli.main(['--model', 'resnet', '--model-config',
              "{'depth': 28, 'width': [160, 320, 640], 'regime': 'wide-resnet', 'dropout': 0.3}", '--dataset',
              'synthetic_cifar10', '--device', 'cpu', '-b', '4', '--epochs', '1', '--max-steps', '2', '--workers', '0',
              '--results-dir', str(tmp_path), '--save', 'wrn'])
    ck = torch.load(tmp_path / 'wrn' / 'checkpoint.pth.tar', map_location='cpu', weights_only=False)
    sd = ck['state_dict']
    assert sd['layer3.3.conv2.weight'].shape == (640, 640, 3, 3)
    assert float(sd['bn1.running_var'].sub(1).abs().sum()) > 0     # the two steps trained
