"""Row-range bookkeeping of gradient accumulation (``chunk_batch``) on the fused path, on the host: torch.chunk's row
ranges, device-augmentation chunks whose boundaries split one image's copies (the host apply() is the oracle), the
per-chunk loss-gradient scale and the meter weights."""
import types

import pytest
import torch

from convnet.pytorch_b200 import ops


@pytest.mark.parametrize('rows', [1, 2, 5, 7, 16, 31, 32, 33, 128, 250])
@pytest.mark.parametrize('chunks', [1, 2, 3, 4, 5, 8])
def test_chunk_rows_follow_torch_chunk(rows, chunks):
    want = [(int(c[0]), int(c[-1]) + 1) for c in torch.arange(rows).chunk(chunks)]
    assert ops.chunk_rows(rows, chunks) == want


def _aug_batch(B, D, resize=None, seed=0):
    from convnet.pytorch_b200.utils.augment import AugmentedBatch, BatchAugment
    spec = BatchAugment(padding=4, cutout={'holes': 1, 'length': 8}, duplicates=D, resize=resize)
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    images = torch.randint(0, 256, (B, 16, 16, 3), generator=g, dtype=torch.uint8)
    return AugmentedBatch(images, spec.sample(B, 16, 16), spec)


@pytest.mark.parametrize('B,D,N,resize', [(5, 4, 3, None), (7, 4, 3, None), (6, 3, 4, None), (5, 4, 2, (12, 12)),
                                          (3, 1, 2, None)])
def test_augment_row_range_against_host_apply(B, D, N, resize):
    from convnet.pytorch_b200.utils.augment import AugmentedBatch
    batch = _aug_batch(B, D, resize)
    whole = batch.apply()
    P = batch.params.shape[-1]
    aug = ops.Aug(batch.params.reshape(B * D, P), batch.spec.lut(3), D, batch.spec.padding, resize)
    seen = []
    for r0, r1 in ops.chunk_rows(B * D, N):
        a, b0, b1 = aug.row_range(r0, r1)
        p, n = a.window
        assert n == r1 - r0 == a.rows and 0 <= p < D and p + n <= (b1 - b0) * D
        assert b0 * D <= r0 and r1 <= b1 * D and (b1 - b0 - 1) * D < p + n
        sub = AugmentedBatch(batch.images[b0:b1], a.params.reshape(b1 - b0, D, P), batch.spec).apply()
        assert torch.equal(sub[p:p + n], whole[r0:r1]), (r0, r1)
        assert a.key != aug.key
        seen.append((r0, r1))
    assert seen[0][0] == 0 and seen[-1][1] == B * D


def test_resized_crop_row_range_against_host_apply():
    from PIL import Image
    from convnet.pytorch_b200.utils.augment import ResizedCrop, ResizedCropBatch, ResizedCropCollate
    g = torch.Generator().manual_seed(2)
    torch.manual_seed(2)
    spec = ResizedCrop(16, duplicates=2)
    samples = []
    for _ in range(5):
        h, w = (int(v) for v in torch.randint(8, 40, (2,), generator=g))
        img = Image.fromarray(torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).numpy(), 'RGB')
        samples.append((spec(img), 0))
    batch, _ = ResizedCropCollate(spec)(samples)
    whole = batch.apply()
    rrc = ops.Rrc(batch.index, batch.draws, spec.lut(3), 2, spec.size, batch.host + (batch.nbytes,))
    ranges = ops.chunk_rows(10, 4)            # 3, 3, 3, 1 rows: boundaries inside images 1 and 4
    assert any(r0 % 2 for r0, _ in ranges)
    for r0, r1 in ranges:
        a, b0, b1 = rrc.row_range(r0, r1)
        p, n = a.window
        assert a.index.shape[0] == b1 - b0 and a.draws.shape[0] == 2 * (b1 - b0) and a.rows == n == r1 - r0
        h_index, h_draws, nbytes = a.host
        assert torch.equal(h_index, a.index) and torch.equal(h_draws, a.draws) and nbytes == batch.nbytes
        ops.check_rrc_tables(h_index, h_draws, nbytes, 3, 2)
        sub = ResizedCropBatch(batch.regions, a.index, a.draws, spec, 3, batch.nbytes).apply()
        assert torch.equal(sub[p:p + n], whole[r0:r1]), (r0, r1)


def test_trainer_chunks_split_device_rows():
    from convnet.pytorch_b200.trainer import Trainer
    batch = _aug_batch(5, 4)
    P = batch.params.shape[-1]
    aug = ops.Aug(batch.params.reshape(20, P), batch.spec.lut(3), 4, 4)
    target = torch.arange(20)
    chunks = Trainer._chunks(batch.images, target, 3, aug)
    assert [int(t[0]) for _, t, _ in chunks] == [0, 7, 14]
    for (x, t, a), (r0, r1) in zip(chunks, ops.chunk_rows(20, 3)):
        b0 = r0 // 4
        assert torch.equal(t, target[r0:r1])
        assert x.shape[0] == a.params.shape[0] // 4 and torch.equal(x[0], batch.images[b0])
    plain = Trainer._chunks(torch.zeros(10, 3, 4, 4), torch.arange(10), 4, None)
    assert [t.tolist() for _, t, _ in plain] == [[0, 1, 2], [3, 4, 5], [6, 7, 8], [9]]
    one = Trainer._chunks(batch.images, target, 1, aug)
    assert len(one) == 1 and one[0][2] is aug


def _host_trainer():
    """a Trainer whose runtime stands in with a CPU device: _upstream and _chunk_weights need nothing else"""
    from convnet.pytorch_b200.trainer import Trainer
    tr = Trainer(torch.nn.Linear(2, 2), torch.nn.CrossEntropyLoss(), device='cpu')
    tr.b200 = types.SimpleNamespace(device='cpu')
    return tr


@pytest.mark.parametrize('N', [2, 3, 4, 7])
@pytest.mark.parametrize('loss_scale', [1.0, 3.0, 0.1])
def test_chunk_upstream_is_autograd_of_loss_over_chunks(N, loss_scale):
    """what autograd hands the chunk's loss for backward((loss / N), grad=up)"""
    tr = _host_trainer()
    tr.loss_scale = loss_scale
    up = torch.tensor(float(tr._upstream()))
    loss = torch.tensor(2.5, requires_grad=True)
    torch.autograd.backward(loss / N, grad_tensors=[up])
    assert float(tr._upstream(N)) == float(loss.grad)
    assert float(tr._upstream()) == float(up)


def test_meter_weights_reproduce_the_reference_meters():
    """uneven chunks: the loss meter is the sum of each chunk's loss / N (the reference's total_loss), the accuracies
    those of the concatenated outputs"""
    from convnet.pytorch_b200.utils.meters import accuracy
    tr = _host_trainer()
    g = torch.Generator().manual_seed(0)
    B, N, classes = 30, 4, 10
    out = torch.randn(B, classes, generator=g)
    y = torch.randint(0, classes, (B,), generator=g)
    ranges = ops.chunk_rows(B, N)
    assert len({r1 - r0 for r0, r1 in ranges}) > 1
    stats, ref_loss = [], 0.0
    for r0, r1 in ranges:
        loss = torch.nn.functional.cross_entropy(out[r0:r1], y[r0:r1])
        p1, p5 = accuracy(out[r0:r1], y[r0:r1], topk=(1, 5))
        stats.append(torch.stack([loss, p1.reshape(()), p5.reshape(())]).float())
        ref_loss += float(loss / N)
    got = (torch.stack(stats) * tr._chunk_weights(ranges, N)).sum(0)
    p1, p5 = accuracy(out, y, topk=(1, 5))
    assert abs(float(got[0]) - ref_loss) < 1e-5
    assert abs(float(got[1]) - float(p1)) < 1e-4 and abs(float(got[2]) - float(p5)) < 1e-4
    assert tr._chunk_weights(ranges, N) is tr._chunk_weights(ranges, N)
