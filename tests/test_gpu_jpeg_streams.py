"""GPU tier of the device JPEG decode on streams Pillow's encoder never writes (tests/test_jpeg_streams_cpu.py's
corpus): the kernels' regions against Pillow's decode bit for bit, whole images and resized-crop draws; the Huffman
launch with 32 decoding threads per block; region boxes chosen at every MCU-row and upsampling residue; and the status
bit of each kind of damaged entropy data, which leaves the rest of the batch exact and, below the rows a region needs,
leaves that region exact too."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_gpu_jpeg import _assert_regions_equal, _decode_on_device  # noqa: E402
from test_jpeg_cpu import encode, picture  # noqa: E402
from test_jpeg_streams_cpu import YCC, _frame, damaged, stream_corpus  # noqa: E402
from convnet.pytorch_b200 import ops  # noqa: E402
from convnet.pytorch_b200.lib import B200Error  # noqa: E402
from convnet.pytorch_b200.utils import jpeg  # noqa: E402
from convnet.pytorch_b200.utils.augment import JpegCollate, JpegDecode, ResizedCrop, ScaleCrop, \
    _mcu_rows_needed  # noqa: E402

pytestmark = pytest.mark.gpu

BAD_CODE, SHORT_DATA, BAD_RESTART, BAD_INDEX = 1, 2, 4, 8
DAMAGE = {'code': BAD_CODE, 'short': SHORT_DATA, 'restart': BAD_RESTART, 'run': BAD_INDEX}


def _boxed(files_boxes):
    """-> (device regions, PIL regions, status, batch) of one JpegBatch whose i-th image is files_boxes[i][0] with
    the region box files_boxes[i][1] = (y0, x0, rh, rw)."""
    spec = ScaleCrop(32, 32)
    samples = []
    for i, (data, box) in enumerate(files_boxes):
        info, _, table, data, _ = JpegDecode(spec)(data)
        assert info is not None, info
        samples.append(((info, tuple(int(v) for v in box), table, data, None), i))
    batch, _ = JpegCollate(spec)(samples)
    decoded, status = batch.replace(tuple(t.cuda() for t in batch.tensors)).decode()
    return decoded.regions[:decoded.nbytes].cpu(), batch.regions(), status.cpu(), batch


@pytest.mark.parametrize('spec', [ScaleCrop(600, 600), ResizedCrop(48, duplicates=4)], ids=['whole', 'rrc-d4'])
def test_streams_equal_pillow(spec):
    torch.cuda.set_device(0)
    corpus = stream_corpus()
    files = [d for _, d, _ in corpus]
    got, ref, status, batch = _decode_on_device(spec, files, seed=7)
    assert not status.any(), status
    kinds = batch.layout['desc'][:, 0]
    assert [k != 2 for k in kinds] == [r == 'baseline' for _, _, r in corpus]
    if isinstance(spec, ScaleCrop):                                         # every region is its whole image
        d = batch.layout['desc']
        dev = kinds != 2
        assert (d[dev, 24] == d[dev, 1]).all() and (d[dev, 25] == d[dev, 2]).all()
    _assert_regions_equal(got, ref, batch)


def test_32_intervals_per_block_launch():
    """Restart interval 1 on large 4:2:0 images: more intervals than 32 per SM, so b200_jpeg_decode gives each block
    32 decoding threads."""
    torch.cuda.set_device(0)
    files = [encode(picture(1500, 2000, s), quality=q, subsampling=2, restart_marker_blocks=1)
             for s, q in ((1, 90), (2, 75))]
    files.append(_frame(600, 808, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 3, restart=1))
    got, ref, status, batch = _decode_on_device(ScaleCrop(2048, 2048), files)
    n = batch.layout['intervals'].shape[0]
    assert n > 32 * torch.cuda.get_device_properties(0).multi_processor_count, n
    assert not status.any(), status
    _assert_regions_equal(got, ref, batch)


def _box_files():
    """(name, bytes, MCU height, MCU width) of images 93 x 77 (odd chroma width 39 at 4:2:0 and 4:2:2)."""
    h, w = 93, 77
    mx = -(-w // 16)
    return [('4:2:0', encode(picture(h, w, 1), quality=88, subsampling=2), 16, 16),
            ('4:2:2', encode(picture(h, w, 2), quality=88, subsampling=1), 8, 16),
            ('4:4:4', encode(picture(h, w, 3), quality=88, subsampling=0), 8, 8),
            ('gray', encode(picture(h, w, 4, gray=True), quality=88), 8, 8),
            ('4:2:0 restart 2 rows', _frame(h, w, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 5, restart=2 * mx), 16, 16),
            ('4:2:0 restart row + 3', _frame(h, w, [(1, 2, 2, 0, 0, 0)] + YCC[1:], 6, restart=mx + 3), 16, 16)]


def _boxes(H, W, mh, mw):
    """Region boxes whose bottom edge y0 + rh takes every residue mod mh, near the bottom and in the middle, whose right
    edge x0 + rw takes every residue mod mw likewise, 1 x 1 boxes and 1-row boxes."""
    out = []
    for r in range(mh):
        for top in (H, H // 2 + mh):
            y1 = top - (top - r) % mh
            if y1 >= 1:
                out.append((max(0, y1 - 3), 0, min(3, y1), W))
    for r in range(mw):
        for right in (W, W // 2 + mw):
            x1 = right - (right - r) % mw
            if x1 >= 1:
                out.append((0, max(0, x1 - 2), H, min(2, x1)))
    out += [(y, x, 1, 1) for y, x in ((0, 0), (H - 1, W - 1), (H - 1, 0), (0, W - 1), (H // 2, W // 2), (15, 15),
                                      (16, 16), (31, 39))]
    out += [(y, 0, 1, W) for y in (0, 7, 8, 15, 16, 17, 31, 32, 47, 48, H - 2, H - 1)]
    return out


@pytest.mark.parametrize('case', [0, 1, 2, 3, 4, 5], ids=[n for n, _, _, _ in _box_files()])
def test_chosen_region_boxes_equal_pillow(case):
    """Regions cut at every residue of the MCU rows and columns, where the decode stops after the last MCU row the
    region needs (upsampling context row included), and the IDCT skips blocks outside it.  For the restart files the
    last needed MCU row ends a restart interval at some residues and not at others."""
    torch.cuda.set_device(0)
    _, data, mh, mw = _box_files()[case]
    info = jpeg.parse(data)
    boxes = _boxes(info.height, info.width, mh, mw)
    got, ref, status, batch = _boxed([(data, b) for b in boxes])
    assert not status.any(), status
    if case == 4:                               # some boxes end their decode exactly at a restart interval's end
        ri = info.restart
        ends = {int(r) * info.mcus[0] % ri == 0 for r in batch.layout['desc'][:, 7]}
        assert ends == {True, False}
    _assert_regions_equal(got, ref, batch)


def test_damaged_streams_set_their_status_bit():
    """Each kind of damage inside the region sets exactly its status bit for its own image; check_jpeg_status names
    those images; the good images of the batch stay exact."""
    torch.cuda.set_device(0)
    good = encode(picture(100, 120, 5), quality=85)
    kinds = list(DAMAGE)
    files = [good] + [damaged(k, 3) for k in kinds] + [good]
    boxes = [(0, 0, 100, 120)] + [(0, 0, 128, 80)] * len(kinds) + [(30, 20, 60, 90)]
    got, ref, status, batch = _boxed(list(zip(files, boxes)))
    assert status.tolist() == [0] + [DAMAGE[k] for k in kinds] + [0]
    with pytest.raises(B200Error, match=r'sample\(s\) \[1, 2, 3, 4\]'):
        ops.check_jpeg_status(status)
    for b in (0, len(files) - 1):
        off, h, w = batch.index[b].tolist()
        assert torch.equal(got[off:off + 3 * h * w], ref[off:off + 3 * h * w]), b


def test_damage_below_the_region_leaves_it_exact():
    """The same damage two MCU rows below the rows a region needs: status 0 and the region exact."""
    torch.cuda.set_device(0)
    files_boxes = []
    for k in DAMAGE:
        data = damaged(k, 5)
        info = jpeg.parse(data)
        box = (10, 4, 38, 70)                       # rows [10, 48): MCU rows 0..3, the last for upsampling context
        assert _mcu_rows_needed(info, box[0] + box[2]) == 4
        files_boxes.append((data, box))
    got, ref, status, batch = _boxed(files_boxes)
    assert not status.any(), status
    _assert_regions_equal(got, ref, batch)
