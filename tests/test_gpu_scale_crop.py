"""Resize + CenterCrop on the kernel path: the scale-crop relayout (b200_input_prep_u8_scale_crop) against
b200_input_prep of ScaleCropBatch.apply() -- torchvision's own PIL transform -- bit for bit, its table checks and memory
safety, and Trainer.validate fed ScaleCropBatches against the same evaluation fed the applied fp32 batches."""

import numpy as np
import pytest
import torch

from convnet.pytorch_b200.utils.augment import ScaleCrop, ScaleCropBatch, ScaleCropCollate

pytestmark = pytest.mark.gpu

GUARD = 4096


def _image(h, w, c, seed):
    from PIL import Image
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(0, 256, (h, w, c), generator=g, dtype=torch.uint8).numpy()
    return Image.fromarray(a if c == 3 else a[:, :, 0], 'RGB' if c == 3 else 'L')


def _batch(size, scale, C, sizes, seed):
    """ScaleCropBatch of seeded uniform images of ``sizes`` [(h, w)] through the loader's own per-image work"""
    stats = {'mean': [0.485, 0.456, 0.406][:C], 'std': [0.229, 0.224, 0.225][:C]}
    spec = ScaleCrop(size, scale, normalize=stats)
    samples = [(spec(_image(h, w, C, seed + k)), k) for k, (h, w) in enumerate(sizes)]
    return ScaleCropCollate(spec)(samples)[0]


def _tables(batch):
    from convnet.pytorch_b200 import ops
    return ops.ScaleCropTables(batch.index.cuda(), batch.geom.cuda(), batch.spec.lut(batch.channels).cuda(),
                               batch.spec.size, (batch.index, batch.geom, batch.nbytes))


def _random_sizes(n, seed, lo=20, hi=900):
    g = torch.Generator().manual_seed(seed)
    return [(int(h), int(w)) for h, w in torch.randint(lo, hi, (n, 2), generator=g)]


def _cases():
    return [  # name, size, scale, C, image sizes, cpad, s2d
        ('224-256-mode2', 224, 256, 3, [(375, 500), (500, 375), (300, 300), (256, 341), (100, 120), (2000, 2300)],
         16, True),                                                # the fixture's shapes: >16 taps, upscale, identity
        ('224-224-pad-c1', 224, 224, 1, [(150, 200), (301, 180), (224, 224), (225, 226), (90, 400)], 8, False),
        ('128-146-c1-mode2', 128, 146, 1, [(333, 417), (146, 146), (77, 1000)], 16, True),
        ('288-329-cpad16', 288, 329, 3, [(480, 640), (329, 500), (1200, 300)], 16, False),
        ('64-73-odd-b', 64, 73, 3, _random_sizes(7, 1), 8, False),
        ('64-73-mode2', 64, 73, 3, _random_sizes(5, 2), 16, True),
        ('96-110-random', 96, 110, 3, _random_sizes(9, 3, 10, 1500), 16, True),
        ('48-40-downscale-crop', 48, 40, 3, _random_sizes(5, 4), 8, False),    # scale < size: padded after Resize
    ]


@pytest.mark.parametrize('name,size,scale,C,sizes,cpad,s2d', _cases(), ids=[c[0] for c in _cases()])
def test_input_prep_u8_scale_crop_is_exact(name, size, scale, C, sizes, cpad, s2d):
    from convnet.pytorch_b200 import ops
    batch = _batch(size, scale, C, sizes, seed=len(sizes) * 11 + C)
    want = ops.input_prep(batch.apply().cuda(), cpad, s2d=s2d, border=s2d)
    sc = _tables(batch)
    regions = batch.regions.cuda()
    n = want.numel()
    outs = []
    for _ in range(2):
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=torch.bfloat16, device='cuda')
        out = buf[GUARD:GUARD + n].view(want.shape)
        ops.input_prep_u8_scale_crop(regions, cpad, sc, s2d=s2d, border=s2d, out=out)
        torch.cuda.synchronize()
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + n:].float()).all(), 'wrote outside'
        assert not torch.isnan(out.float()).any(), 'left elements unwritten'
        bad = (out.view(torch.int16) != want.view(torch.int16))
        assert not bad.any(), 'differs from input_prep(apply()) at %d elements, first %s' % (
            int(bad.sum()), bad.nonzero()[0].tolist())
        outs.append(out.clone())
    assert torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))


def test_input_prep_u8_scale_crop_rejects_bad_tables():
    from convnet.pytorch_b200 import ops
    from convnet.pytorch_b200.lib import B200Error
    batch = _batch(64, 73, 3, [(375, 500), (90, 60)], seed=0)
    regions = batch.regions.cuda()
    ops.input_prep_u8_scale_crop(regions, 16, _tables(batch))
    for col, value, match in ((0, 0, 'misses'), (6, 0, 'misses'), (4, 0, 'outside 1'), (0, 10 ** 4, 'outside its')):
        geom = batch.geom.clone()
        geom[0, col] = value
        with pytest.raises(B200Error, match=match):
            ops.input_prep_u8_scale_crop(regions, 16, _tables(ScaleCropBatch(batch.regions, batch.index, geom,
                                                                              batch.spec, 3)))
    ix = batch.index.clone()
    ix[1, 0] = batch.nbytes
    with pytest.raises(B200Error, match='buffer'):
        ops.input_prep_u8_scale_crop(regions, 16, _tables(ScaleCropBatch(batch.regions, ix, batch.geom, batch.spec, 3)))
    with pytest.raises(B200Error, match='Cpad'):
        ops.input_prep_u8_scale_crop(regions, 12, _tables(batch))
    with pytest.raises(B200Error, match='border'):
        ops.input_prep_u8_scale_crop(regions, 16, _tables(batch), s2d=True, border=False)


def test_out_of_range_tables_stay_memory_safe():
    """tables the host check refuses, handed straight to the kernel: every read is clamped to its region and the
    buffer, every write lands in the output, the work stays bounded (sizes clamp to 65535)"""
    from convnet.pytorch_b200 import lib
    regions = torch.randint(0, 256, (5000,), dtype=torch.uint8, device='cuda')
    index = torch.tensor([[-100, 0, 7], [10 ** 12, 3, 10 ** 9], [4000, 40, 40], [0, 10, 10]], dtype=torch.int64,
                         device='cuda')
    geom = torch.tensor([[-10 ** 9, 10 ** 9, 50, -3, 0, 999, -2 ** 31 + 1, 2 ** 31 - 1],
                         [5, 5, 300, 200, 1, 1, 10, -10],
                         [-7, 3, 60, 80, 500, 700, 200, 300],
                         [2 ** 31 - 1, -2 ** 31, 30, 30, 64, 64, -5, 5]], dtype=torch.int32, device='cuda')
    lut = torch.rand(3, 256, device='cuda')
    for mode, shape in ((0, (4, 64, 64, 8)), (2, (4, 35, 35, 16))):
        n = int(np.prod(shape))
        buf = torch.full((n + 2 * GUARD,), float('nan'), dtype=torch.bfloat16, device='cuda')
        out = buf[GUARD:GUARD + n]
        lib.check(lib.load().b200_input_prep_u8_scale_crop(regions.data_ptr(), regions.numel(), index.data_ptr(),
                                                           geom.data_ptr(), 4, 3, 64, 64, shape[-1], mode,
                                                           lut.data_ptr(), out.data_ptr(),
                                                           torch.cuda.current_stream().cuda_stream),
                  'b200_input_prep_u8_scale_crop')
        torch.cuda.synchronize()
        assert torch.isnan(buf[:GUARD].float()).all() and torch.isnan(buf[GUARD + n:].float()).all()
        assert not torch.isnan(out.float()).any()


def _val_batches(steps, B, size, scale, seed):
    """(ScaleCropBatch, target) of images of the synthetic ImageNet pool through the loader's per-image work"""
    from convnet.pytorch_b200.data import synthetic_imagenet_pool
    pool = synthetic_imagenet_pool(n=steps * B, lo=40, hi=400, seed=seed)
    spec = ScaleCrop(size, scale)
    g = torch.Generator().manual_seed(seed)
    collate = ScaleCropCollate(spec)
    return [collate([(spec(img), int(torch.randint(0, 1000, (1,), generator=g))) for img in pool[s * B:(s + 1) * B]])
            for s in range(steps)]


def _validate_pair(model_fn, batches, monkeypatch):
    """Trainer.validate of the ScaleCropBatches and of their applied fp32 batches, BN folded and not: logits bitwise
    equal and meters equal; the device run never calls apply()"""
    from convnet.pytorch_b200 import engine, ops
    from convnet.pytorch_b200.engine import convert_b200
    from convnet.pytorch_b200.trainer import Trainer
    from convnet.pytorch_b200.utils.cross_entropy import CrossEntropyLoss
    torch.cuda.set_device(0)
    torch.manual_seed(123)
    model = convert_b200(model_fn(), 'cuda')
    tr = Trainer(model, CrossEntropyLoss().cuda(), device='cuda', print_freq=10 ** 9)
    fp32 = [(b.apply(), t) for b, t in batches]
    outputs, step = [], tr._step
    kernel_calls = []
    launch = ops.input_prep_u8_scale_crop

    def recording_step(inputs, target, **kw):
        out = step(inputs, target, **kw)
        outputs.append(out[0].detach().clone())
        return out

    def counted(*a, **kw):
        kernel_calls.append(1)
        return launch(*a, **kw)

    def no_apply(self):
        raise AssertionError('the device evaluation called ScaleCropBatch.apply()')
    tr._step = recording_step
    saved = engine.FOLD_BN_EVAL
    try:
        for fold in (False, True):
            engine.FOLD_BN_EVAL = fold
            runs = []
            for form in ('device', 'fp32'):
                outputs.clear()
                with monkeypatch.context() as m:
                    if form == 'device':
                        m.setattr(ScaleCropBatch, 'apply', no_apply)
                        m.setattr(ops, 'input_prep_u8_scale_crop', counted)
                    res = tr.validate(batches if form == 'device' else fp32)
                torch.cuda.synchronize()
                runs.append((torch.cat(outputs).cpu(), {k: res[k] for k in ('loss', 'prec1', 'prec5')}))
            (o0, m0), (o1, m1) = runs
            assert o0.shape == (sum(b.rows for b, _ in batches), 1000)
            assert torch.equal(o0, o1), 'fold=%s: logits differ at %d elements' % (fold, int((o0 != o1).sum()))
            assert m0 == m1, (fold, m0, m1)
    finally:
        engine.FOLD_BN_EVAL = saved
    assert len(kernel_calls) == 2 * len(batches)


def test_validate_resnet18_scale_crop_matches_applied_batch_bitwise(monkeypatch):
    """ResNet-18 (mode-2 space-to-depth stem), 64 px from scale 73, odd batches, three steps"""
    from convnet.pytorch_b200.models import resnet
    _validate_pair(lambda: resnet(dataset='imagenet', depth=18), _val_batches(3, 7, 64, 73, seed=5), monkeypatch)


def test_validate_mobilenet_v2_scale_crop_matches_applied_batch_bitwise(monkeypatch):
    """MobileNet-v2 (mode-0 3x3/s2 stem), 96 px from scale 110, two steps"""
    from convnet.pytorch_b200.models import mobilenet_v2
    _validate_pair(lambda: mobilenet_v2(dataset='imagenet'), _val_batches(2, 6, 96, 110, seed=6), monkeypatch)


def test_eval_forward_adds_library_kernels_only():
    """Profiler traces of the eval forward of a converted ResNet-18 on a ScaleCropBatch and on its applied fp32 batch:
    the first runs the scale-crop relayout in place of the fp32 one and no kernel outside the library that the second
    does not run"""
    from torch.profiler import ProfilerActivity, profile
    from convnet.pytorch_b200.models import resnet
    from convnet.pytorch_b200.engine import convert_b200
    torch.cuda.set_device(0)
    torch.manual_seed(3)
    batch, _ = _val_batches(1, 16, 64, 73, seed=7)[0]
    model = convert_b200(resnet(dataset='imagenet', depth=18), 'cuda')
    model.eval()
    rt = model._b200
    traces = []
    for x, kw in ((batch.regions.cuda(), dict(aug=_tables(batch))), (batch.apply().cuda(), {})):
        with torch.no_grad():
            rt.run_forward(x, False, False, **kw)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(2):
                    rt.run_forward(x, False, False, **kw)
                torch.cuda.synchronize()
        traces.append({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    fused, plain = traces

    def other(names):
        return {n for n in names if 'b200::' not in n and 'memset' not in n.lower()}
    print('\nscale-crop eval forward: kernels outside the library: %s' % sorted(other(fused)))
    assert len(fused) > 5 and other(fused) <= other(plain), other(fused) - other(plain)
    assert any('input_prep_scale_crop_kernel' in n for n in fused), sorted(fused)
    assert not any('input_prep_kernel' in n for n in fused) and any('input_prep_kernel' in n for n in plain)


def test_evaluate_cli_with_device_scale_crop(tmp_path, monkeypatch):
    """evaluate.py --device-scale-crop on a ResNet-18 checkpoint, synthetic ImageNet at 64 px: the relayout runs"""
    from convnet.pytorch_b200 import engine, evaluate, models, ops
    from convnet.pytorch_b200.main import _model_dataset_name
    torch.manual_seed(0)
    model = models.resnet(dataset=_model_dataset_name('synthetic_imagenet'), depth=18)
    ckpt = tmp_path / 'checkpoint.pth.tar'
    torch.save({'epoch': 1, 'model': 'resnet', 'config': "{'depth': 18}", 'state_dict': model.state_dict()}, ckpt)
    monkeypatch.setenv('B200_SYNTHETIC_LENGTH', '24')
    calls = []
    launch = ops.input_prep_u8_scale_crop
    monkeypatch.setattr(ops, 'input_prep_u8_scale_crop', lambda *a, **kw: calls.append(1) or launch(*a, **kw))
    monkeypatch.setattr(ScaleCropBatch, 'apply', lambda self: (_ for _ in ()).throw(AssertionError('apply() ran')))
    saved = engine.FOLD_BN_EVAL
    try:
        res = evaluate.main([str(ckpt), '--dataset', 'synthetic_imagenet', '--input-size', '64', '-b', '8',
                             '--workers', '0', '--absorb-bn', '--device-scale-crop', '--save', 'sc_%s' % tmp_path.name])
    finally:
        engine.FOLD_BN_EVAL = saved
    assert len(calls) == 3 and res['loss'] > 0 and 0 <= res['prec1'] <= 100
