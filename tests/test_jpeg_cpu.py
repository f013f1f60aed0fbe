"""CPU tier of the device JPEG decode (data.py ``device_decode``): the header classifier, the numpy restatement of the
kernels (tests/jpeg_oracle.py) against Pillow's decode, the worker draws and JpegBatch.apply() against the PIL paths
of the device crops, and the settings that raise."""
import io
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import jpeg_oracle  # noqa: E402
from convnet.pytorch_b200.utils import jpeg  # noqa: E402
from convnet.pytorch_b200.utils.augment import JpegCollate, JpegDecode, ResizedCrop, ResizedCropCollate, \
    ScaleCrop, ScaleCropCollate  # noqa: E402


def picture(h, w, seed, gray=False, noise=False):
    """A seeded test picture: smooth gradients plus noise (or pure uniform noise)."""
    rng = np.random.default_rng(seed)
    if noise:
        a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        y, x = np.mgrid[0:h, 0:w]
        a = np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), (x * 3 + y * 5) % 256], -1)
        a = (a + rng.integers(-24, 25, a.shape)).clip(0, 255).astype(np.uint8)
    return a[:, :, 0] if gray else a


def encode(a, fmt='JPEG', mode=None, **kw):
    from PIL import Image
    img = Image.fromarray(a)
    if mode:
        img = img.convert(mode)
    buf = io.BytesIO()
    img.save(buf, fmt, **kw)
    return buf.getvalue()


def device_corpus(large=True):
    """(name, bytes) of files the device decodes: every quality, optimised tables, 4:4:4 / 4:2:2 / 4:2:0 and
    grayscale, restart markers by blocks and by rows, odd sizes, q=100 noise for the IDCT clamp."""
    out = [('q%d' % q, encode(picture(17, 33, q), quality=q, subsampling=q % 3)) for q in range(1, 101)]
    sizes = [(1, 1), (7, 9), (17, 33), (2, 5), (33, 17)] + ([(375, 500)] if large else [])
    for i, (h, w) in enumerate(sizes):
        for ss in (0, 1, 2):
            out.append(('%dx%d ss%d' % (h, w, ss), encode(picture(h, w, i), quality=85, subsampling=ss)))
        out.append(('%dx%d optimize' % (h, w), encode(picture(h, w, i), quality=75, optimize=True)))
        out.append(('%dx%d gray' % (h, w), encode(picture(h, w, i, gray=True), quality=80)))
        out.append(('%dx%d noise' % (h, w), encode(picture(h, w, i, noise=True), quality=100, subsampling=0)))
        out.append(('%dx%d rst blocks' % (h, w), encode(picture(h, w, i), quality=90, restart_marker_blocks=3)))
        out.append(('%dx%d rst rows' % (h, w), encode(picture(h, w, i), quality=90, subsampling=1,
                                                        restart_marker_rows=1)))
    return out


def fallback_corpus():
    a = picture(40, 52, 7)
    return [('progressive', encode(a, quality=80, progressive=True)),
            ('cmyk', encode(a, mode='CMYK', quality=80)),
            ('png', encode(a, fmt='PNG'))]


def pil_rgb(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)).convert('RGB'))


def test_classifier_sends_each_file_to_its_side():
    for name, data in device_corpus(large=False):
        info = jpeg.parse(data)
        assert info.device, (name, info.reason)
        assert (info.height, info.width) == pil_rgb(data).shape[:2], name
    for name, data in fallback_corpus():
        assert not jpeg.parse(data).device, name
    assert not jpeg.parse(b'').device and not jpeg.parse(b'\xff\xd8\xff').device


def test_oracle_equals_pillow_bitwise():
    for name, data in device_corpus():
        got = jpeg_oracle.decode(data)
        assert np.array_equal(got, pil_rgb(data)), name


def test_restart_markers_are_located():
    data = encode(picture(48, 64, 3), quality=90, restart_marker_blocks=2)
    info = jpeg.parse(data)
    mx, my = info.mcus
    assert info.restart == 2 and len(info.rst) == -(-mx * my // 2) - 1
    assert all(data[p - 2] == 0xFF and data[p - 1] == 0xD0 + (k & 7) for k, p in enumerate(info.rst))


def _files(n=6, seed=0):
    """Device and fallback files of varied sizes, in a fixed order."""
    out = []
    for i in range(n):
        h, w = 60 + 37 * i, 90 + 23 * i
        out.append(encode(picture(h, w, seed + i), quality=70 + 4 * i, subsampling=i % 3))
    out.insert(2, fallback_corpus()[0][1])
    out.insert(5, fallback_corpus()[2][1])
    return out


@pytest.mark.parametrize('D', [1, 4])
def test_resized_crop_draws_and_apply_equal_the_pil_path(D):
    from PIL import Image
    spec = ResizedCrop(32, duplicates=D)
    files = _files()
    torch.manual_seed(5)
    samples = [(JpegDecode(spec)(f), i) for i, f in enumerate(files)]
    torch.manual_seed(5)
    ref = [(spec(Image.open(io.BytesIO(f)).convert('RGB')), i) for i, f in enumerate(files)]
    for (s, _), ((region, draws), _) in zip(samples, ref):
        assert torch.equal(s[2], draws)
        assert (s[1][2], s[1][3]) == tuple(region.shape[:2])
    batch, target = JpegCollate(spec)(samples)
    ref_batch, ref_target = ResizedCropCollate(spec)(ref)
    assert torch.equal(target, ref_target) and batch.rows == ref_batch.rows == len(files) * D
    assert torch.equal(batch.index, ref_batch.index) and batch.nbytes == ref_batch.nbytes
    assert torch.equal(batch.regions(), ref_batch.regions)
    assert torch.equal(batch.apply(), ref_batch.apply())
    kinds = batch.layout['desc'][:, 0]
    assert list(np.flatnonzero(kinds == 2)) == [2, 5]


def test_scale_crop_geometry_and_apply_equal_the_pil_path():
    from PIL import Image
    spec = ScaleCrop(32, 40)
    files = _files(seed=11)
    samples = [(JpegDecode(spec)(f), i) for i, f in enumerate(files)]
    ref = [(spec(Image.open(io.BytesIO(f)).convert('RGB')), i) for i, f in enumerate(files)]
    batch, _ = JpegCollate(spec)(samples)
    ref_batch, _ = ScaleCropCollate(spec)(ref)
    assert torch.equal(batch.table, ref_batch.geom) and torch.equal(batch.index, ref_batch.index)
    assert torch.equal(batch.regions(), ref_batch.regions)
    assert torch.equal(batch.apply(), ref_batch.apply())


def test_layout_validation_rejects_a_corrupt_descriptor():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    spec = ScaleCrop(32, 40)
    batch, _ = JpegCollate(spec)([(JpegDecode(spec)(f), i) for i, f in enumerate(_files(3))])
    n = batch.payload.numel()
    ops.check_jpeg_layout(batch.layout, n, batch.nbytes)
    with pytest.raises(B200Error, match='payload'):
        ops.check_jpeg_layout(batch.layout, n, batch.nbytes - 1)
    bad = dict(batch.layout, desc=batch.layout['desc'].copy())
    bad['desc'][0, 10] = n + 1                      # the segment's end past the payload
    with pytest.raises(B200Error, match=r'image\(s\) \[0\]'):
        ops.check_jpeg_layout(bad, n, batch.nbytes)
    with pytest.raises(B200Error, match='sample\\(s\\) \\[1\\]'):
        ops.check_jpeg_status(torch.tensor([0, 2, 0], dtype=torch.int32))


def test_synthetic_loader_yields_jpeg_batches():
    from convnet.pytorch_b200.data import DataRegime
    from convnet.pytorch_b200.utils.augment import JpegBatch
    dr = DataRegime(None, {'name': 'synthetic_imagenet', 'split': 'train', 'augment': True, 'input_size': 32,
                           'batch_size': 4, 'synthetic_length': 8, 'device_resized_crop': True,
                           'device_decode': True})
    batch, target = next(iter(dr.get_loader()))
    assert isinstance(batch, JpegBatch) and target.shape == (4,)
    assert (batch.layout['desc'][:, 0] == 0).all()                  # PIL's 4:2:0 files: all decoded on the device
    assert batch.apply().shape == (4, 3, 32, 32)


def test_unsupported_combinations_raise(tmp_path):
    from convnet.pytorch_b200 import evaluate, main as cli
    from convnet.pytorch_b200.data import DataRegime
    with pytest.raises(NotImplementedError, match='device_resized_crop or device_scale_crop'):
        DataRegime(None, {'name': 'synthetic_imagenet', 'split': 'train', 'augment': True, 'batch_size': 4,
                          'synthetic_length': 8, 'device_decode': True})
    common = ['--model', 'resnet', '--model-config', "{'depth': 18}", '--dataset', 'synthetic_imagenet',
              '--device', 'cpu', '-b', '4', '--epochs', '1', '--max-steps', '1', '--workers', '0',
              '--input-size', '32', '--results-dir', str(tmp_path)]
    with pytest.raises(NotImplementedError, match='--device-resized-crop or'):
        cli.main(common + ['--save', 'a', '--device-decode'])
    with pytest.raises(NotImplementedError, match='CUDA'):
        cli.main(common + ['--save', 'b', '--device-decode', '--device-resized-crop'])
    with pytest.raises(NotImplementedError, match='--device-scale-crop; set it'):
        evaluate.main([str(tmp_path / 'missing.pth'), '--dataset', 'synthetic_imagenet', '--device', 'cpu',
                       '--device-decode', '--save', str(tmp_path / 'e')])
