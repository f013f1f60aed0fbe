"""GPU tier of the device JPEG decode: the kernels' regions against Pillow's decode bit for bit (the CPU tier's corpus,
~2000x1500 images, batches mixing device and host-decoded files; resized-crop regions at D = 1 and 4 and scale-crop
support regions), whole training and evaluation runs with and without ``device_decode``, and the status of a truncated
file."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_jpeg_cpu import device_corpus, encode, fallback_corpus, picture  # noqa: E402
from convnet.pytorch_b200.lib import B200Error  # noqa: E402
from convnet.pytorch_b200.utils.augment import JpegCollate, JpegDecode, ResizedCrop, ScaleCrop  # noqa: E402

pytestmark = pytest.mark.gpu


def _decode_on_device(spec, files, seed=0):
    """-> (device regions, PIL regions, status) of one JpegBatch of ``files``."""
    torch.manual_seed(seed)
    batch, _ = JpegCollate(spec)([(JpegDecode(spec)(f), i) for i, f in enumerate(files)])
    dev = batch.replace(tuple(t.cuda() for t in batch.tensors))
    decoded, status = dev.decode()
    return decoded.regions[:decoded.nbytes].cpu(), batch.regions(), status.cpu(), batch


def _assert_regions_equal(got, ref, batch):
    if torch.equal(got, ref):
        return
    bad = []
    for b, (off, h, w) in enumerate(batch.index.tolist()):
        if not torch.equal(got[off:off + 3 * h * w], ref[off:off + 3 * h * w]):
            bad.append(b)
    raise AssertionError('regions of images %s differ from Pillow' % bad)


def _corpus():
    files = [d for _, d in device_corpus()]
    files += [encode(picture(1500, 2000, 3), quality=q, subsampling=ss) for q, ss in ((92, 2), (75, 0), (85, 1))]
    files.append(encode(picture(1500, 2000, 4), quality=90, restart_marker_rows=2))
    fb = [d for _, d in fallback_corpus()]
    return files[:40] + fb[:1] + files[40:90] + fb[1:] + files[90:]


@pytest.mark.parametrize('spec', [ResizedCrop(64, duplicates=1), ResizedCrop(64, duplicates=4), ScaleCrop(64, 73)],
                         ids=['rrc-d1', 'rrc-d4', 'scale-crop'])
def test_kernel_regions_equal_pillow(spec):
    torch.cuda.set_device(0)
    files = _corpus()
    got, ref, status, batch = _decode_on_device(spec, files, seed=3)
    assert not status.any(), status
    assert (batch.layout['desc'][:, 0] == 2).sum() == 3
    _assert_regions_equal(got, ref, batch)


def test_whole_image_regions_equal_pillow():
    """Regions that are whole images (scale crop without a resize, input size above the images): every pixel, every
    edge and padding case of the upsampling."""
    torch.cuda.set_device(0)
    files = [d for _, d in device_corpus(large=True)]
    got, ref, status, batch = _decode_on_device(ScaleCrop(600, 600), files)
    assert not status.any(), status
    assert batch.layout['desc'][:, 24].tolist() == [min(600, s) for s in batch.layout['desc'][:, 1]]
    _assert_regions_equal(got, ref, batch)


def test_truncated_file_raises_with_its_index():
    from convnet.pytorch_b200 import ops
    torch.cuda.set_device(0)
    good = encode(picture(200, 300, 1), quality=90)
    cut = good[:len(good) * 3 // 10]
    spec = ScaleCrop(32, 36)
    batch, _ = JpegCollate(spec)([(JpegDecode(spec)(f), i) for i, f in enumerate([good, cut, good])])
    assert (batch.layout['desc'][:, 0] == 0).all()              # the header is intact: the device takes the file
    _, status = batch.replace(tuple(t.cuda() for t in batch.tensors)).decode()
    status = status.cpu()
    assert status.tolist()[0] == 0 and status.tolist()[2] == 0 and status.tolist()[1] & 2
    with pytest.raises(B200Error, match=r'sample\(s\) \[1\]'):
        ops.check_jpeg_status(status)


def _image_folder(root, n, seed):
    """An ImageFolder of n files named .JPEG: baseline JPEGs of several kinds and, as ImageNet has, a few files the
    workers decode (progressive, PNG bytes)."""
    rng = np.random.default_rng(seed)
    for i in range(n):
        d = root / 'imagenet' / 'train' / ('c%d' % (i % 3))
        d.mkdir(parents=True, exist_ok=True)
        h, w = (int(v) for v in rng.integers(80, 260, 2))
        a = picture(h, w, seed + i)
        kind = i % 8
        if kind == 5:
            data = encode(a, quality=80, progressive=True)
        elif kind == 7:
            data = encode(a, fmt='PNG')
        elif kind == 3:
            data = encode(a[:, :, 0], quality=85)
        else:
            data = encode(a, quality=int(rng.integers(60, 96)), subsampling=kind % 3,
                          **({'restart_marker_blocks': 4} if kind == 6 else {}))
        (d / ('%03d.JPEG' % i)).write_bytes(data)
    (root / 'imagenet' / 'val').symlink_to(root / 'imagenet' / 'train')


def test_trainer_resnet18_device_decode_matches_host_decode_bitwise(tmp_path):
    """ResNet-18, 64 px, B=8, D=2: four Trainer.train steps through the prefetch ring with captured graphs, fed by
    device_decode and by the workers' PIL decode: logits, losses and updated parameters bitwise equal."""
    from convnet.pytorch_b200.data import DataRegime
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    from convnet.pytorch_b200.utils.optim import OptimRegime
    torch.cuda.set_device(0)
    _image_folder(tmp_path, 32, seed=9)
    runs = []
    for decode in (True, False):
        torch.manual_seed(123)
        model = convert_b200(resnet(dataset='imagenet', depth=18), 'cuda')
        opt = OptimRegime(model, copy.deepcopy(model.regime))
        tr = Trainer(model, CrossEntropyLoss().cuda(), opt, device='cuda', print_freq=10 ** 9)
        data = DataRegime(None, {'name': 'imagenet', 'datasets_path': str(tmp_path), 'split': 'train',
                                 'augment': True, 'input_size': 64, 'batch_size': 8, 'shuffle': False,
                                 'num_workers': 0, 'duplicates': 2, 'device_resized_crop': True,
                                 'device_decode': decode}).get_loader()
        record, step = [], tr._step

        def recording_step(inputs, target, **kw):
            out, loss, grad = step(inputs, target, **kw)
            record.append((out.detach().clone(), loss.detach().clone()))
            return out, loss, grad
        tr._step = recording_step
        tr.train(data)
        torch.cuda.synchronize()
        runs.append(([(o.cpu(), l.cpu()) for o, l in record], model._b200.arena.p32.detach().clone().cpu(),
                     tr.graph_replays))
    (r0, p0, g0), (r1, p1, g1) = runs
    assert len(r0) == len(r1) == 4 and g0 == g1 >= 1
    for (o0, l0), (o1, l1) in zip(r0, r1):
        assert torch.equal(o0, o1) and torch.equal(l0, l1)
    assert torch.equal(p0, p1)


def test_evaluate_cli_device_decode_matches_host_decode(tmp_path, monkeypatch):
    """evaluate.py --device-scale-crop with and without --device-decode on an ImageFolder of mixed files: equal
    results, and the decode kernel ran."""
    from convnet.pytorch_b200 import engine, evaluate, models, ops
    monkeypatch.setattr(engine, 'FOLD_BN_EVAL', engine.FOLD_BN_EVAL)   # evaluate.main sets it; restored at teardown
    torch.manual_seed(0)
    _image_folder(tmp_path, 20, seed=4)
    model = models.resnet(dataset='imagenet', depth=18)
    ckpt = tmp_path / 'checkpoint.pth.tar'
    torch.save({'epoch': 1, 'model': 'resnet', 'config': "{'depth': 18}", 'state_dict': model.state_dict()}, ckpt)
    calls = []
    launch = ops.jpeg_decode
    monkeypatch.setattr(ops, 'jpeg_decode', lambda *a, **kw: calls.append(1) or launch(*a, **kw))
    res = []
    for extra in ([], ['--device-decode']):
        res.append(evaluate.main([str(ckpt), '--dataset', 'imagenet', '--datasets-dir', str(tmp_path),
                                  '--input-size', '64', '-b', '8', '--workers', '0', '--device-scale-crop',
                                  '--save', 'e%d_%s' % (len(extra), tmp_path.name)] + extra))
    assert len(calls) == 3
    assert [res[0][k] for k in ('loss', 'prec1', 'prec5')] == [res[1][k] for k in ('loss', 'prec1', 'prec5')]
