"""Baseline JPEG headers on the host: the marker parser and classifier of the device decode (data.py
``device_decode``).

``parse(data)`` walks SOI, APPn, DQT, DHT, SOF, DRI and SOS, locates the entropy-coded segment (ECS) and its restart
markers, and returns a ``JpegInfo``.  ``info.device`` says whether csrc/jpeg.cu decodes the file to the bytes Pillow
(libjpeg-turbo on x86-64: its SIMD ISLOW IDCT, fancy upsampling) gives for ``Image.open(f).convert('RGB')``:
  - SOF0 / SOF1, 8-bit samples, Huffman coding, one scan holding every component in frame order;
  - 1 component, or 3 with luma sampling 1x1, 2x1 or 2x2 and chroma 1x1;
  - a YCbCr colour space as libjpeg infers it (JFIF APP0, Adobe APP14 transform 1, or no Adobe marker and component
    ids other than 'R', 'G', 'B');
  - 8- or 16-bit quantisation tables (entries <= 32767), any restart interval.
Everything else (progressive, arithmetic, 12-bit, CMYK / YCCK, Adobe transform 0, 4:1:1, 4:4:0, multi-scan, non-JPEG
bytes) has ``device`` False with a ``reason``: the loader worker decodes it with PIL.  No PIL is needed here.
"""
import numpy as np

# natural (row-major) index of zig-zag position k (T.81 figure A.6; libjpeg's jpeg_natural_order)
NATURAL_ORDER = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27,
                          20, 13, 6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58,
                          59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

LOOKAHEAD = 9                 # bits resolved by one table lookup (libjpeg's HUFF_LOOKAHEAD is 8)
HUFF_WORDS = 36 + (1 << LOOKAHEAD) // 2 + 64   # int32 words of one packed table (see HuffTable.pack)


class HuffTable(object):
    """A canonical Huffman table (T.81 annex C; libjpeg's jpeg_make_d_derived_tbl): ``maxcode[l]`` the largest code of
    length l (-1 when none, maxcode[17] a sentinel), ``valoffset[l]`` so that value = huffval[code + valoffset[l]], and
    ``lut`` [2**LOOKAHEAD] (length << 8 | value) of every code of at most LOOKAHEAD bits (0: longer or no code)."""

    def __init__(self, bits, huffval):
        self.bits = [0] + [int(b) for b in bits]             # bits[l], l = 1..16
        self.huffval = np.zeros(256, np.uint8)
        self.huffval[:len(huffval)] = huffval
        sizes = [l for l in range(1, 17) for _ in range(self.bits[l])]
        codes, code, si, p = [], 0, sizes[0] if sizes else 0, 0
        while p < len(sizes):
            while p < len(sizes) and sizes[p] == si:
                codes.append(code)
                code += 1
                p += 1
            if code >= (1 << si):
                raise ValueError('bad Huffman table')
            code <<= 1
            si += 1
        self.maxcode = np.full(18, -1, np.int64)
        self.valoffset = np.zeros(18, np.int64)
        p = 0
        for l in range(1, 17):
            if self.bits[l]:
                self.valoffset[l] = p - codes[p]
                p += self.bits[l]
                self.maxcode[l] = codes[p - 1]
        self.maxcode[17] = 0xFFFFF
        self.lut = np.zeros(1 << LOOKAHEAD, np.int32)
        for p, (l, c) in enumerate(zip(sizes, codes)):
            if l <= LOOKAHEAD:
                s = c << (LOOKAHEAD - l)
                self.lut[s:s + (1 << (LOOKAHEAD - l))] = (l << 8) | int(self.huffval[p])

    def pack(self):
        """int32 [HUFF_WORDS]: maxcode[18], valoffset[18], the lookahead table as int16 pairs, huffval as uint8 quads --
        the layout csrc/jpeg.cu reads."""
        out = np.zeros(HUFF_WORDS, np.int32)
        out[0:18] = self.maxcode
        out[18:36] = self.valoffset
        n = (1 << LOOKAHEAD) // 2
        out[36:36 + n] = self.lut.astype(np.int16).view(np.int32)
        out[36 + n:] = self.huffval.view(np.int32)
        return out


class JpegInfo(object):
    """What the parser found.  ``height``, ``width``; ``comps``: [(id, h, v, tq)] in frame order; ``qt``: {slot: int32
    [64] natural order}; ``dc`` / ``ac``: {slot: HuffTable}; ``scan``: [(component index, td, ta)]; ``restart``: the
    restart interval in MCUs (0: none); ``ecs``: (start, end) byte offsets of the entropy-coded segment; ``rst``: int64
    offsets of the first byte after each restart marker inside it; ``device`` / ``reason``."""

    def __init__(self):
        self.height = self.width = 0
        self.comps, self.scan = [], []
        self.qt, self.dc, self.ac = {}, {}, {}
        self.restart = 0
        self.ecs = (0, 0)
        self.rst = np.zeros(0, np.int64)
        self.device, self.reason = False, 'not parsed'

    @property
    def channels(self):
        return len(self.comps)

    @property
    def sampling(self):
        """(hmax, vmax): the luma sampling of a 3-component file, (1, 1) for one component."""
        return (self.comps[0][1], self.comps[0][2]) if len(self.comps) == 3 else (1, 1)

    @property
    def mcus(self):
        """(MCU columns, MCU rows) of the scan."""
        hmax, vmax = self.sampling
        return -(-self.width // (8 * hmax)), -(-self.height // (8 * vmax))


def _fallback(info, reason):
    info.device, info.reason = False, reason
    return info


def parse(data):
    """bytes -> JpegInfo (never raises on malformed input: such a file is a fallback, PIL decides what it is)."""
    info = JpegInfo()
    try:
        return _parse(memoryview(data).cast('B'), info)
    except (IndexError, ValueError) as e:
        return _fallback(info, 'malformed: %s' % e)


def _parse(d, info):
    n = len(d)
    if n < 4 or d[0] != 0xFF or d[1] != 0xD8:
        return _fallback(info, 'not a JPEG (no SOI)')
    jfif = adobe = False
    transform = None
    sof = None
    pos = 2
    while True:
        while pos < n and d[pos] == 0xFF and pos + 1 < n and d[pos + 1] == 0xFF:
            pos += 1                                                   # fill bytes
        if pos + 4 > n or d[pos] != 0xFF:
            return _fallback(info, 'no scan')
        m = d[pos + 1]
        length = (d[pos + 2] << 8) | d[pos + 3]
        seg = d[pos + 4:pos + 2 + length]
        if length < 2 or pos + 2 + length > n:
            return _fallback(info, 'truncated header')
        if m == 0xE0 and bytes(seg[:5]) == b'JFIF\0':
            jfif = True
        elif m == 0xEE and bytes(seg[:5]) == b'Adobe' and len(seg) >= 12:
            adobe, transform = True, seg[11]
        elif m == 0xDB:
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                if pq > 1 or tq > 3:
                    return _fallback(info, 'bad DQT')
                if pq:
                    zz = np.frombuffer(bytes(seg[i + 1:i + 129]), '>u2').astype(np.int32)
                else:
                    zz = np.frombuffer(bytes(seg[i + 1:i + 65]), np.uint8).astype(np.int32)
                if zz.size != 64:
                    raise ValueError('short DQT')
                q = np.zeros(64, np.int32)
                q[NATURAL_ORDER] = zz
                info.qt[tq] = q
                i += 1 + 64 * (pq + 1)
        elif m == 0xC4:
            i = 0
            while i < len(seg):
                tc, th = seg[i] >> 4, seg[i] & 15
                bits = list(seg[i + 1:i + 17])
                cnt = sum(bits)
                vals = np.frombuffer(bytes(seg[i + 17:i + 17 + cnt]), np.uint8)
                if tc > 1 or th > 3 or len(bits) != 16 or cnt > 256 or vals.size != cnt:
                    return _fallback(info, 'bad DHT')
                if tc == 0 and cnt and vals.max() > 15:
                    return _fallback(info, 'bad DC table')
                (info.ac if tc else info.dc)[th] = HuffTable(bits, vals)
                i += 17 + cnt
        elif m == 0xDD:
            info.restart = (seg[0] << 8) | seg[1]
        elif m == 0xCC:
            return _fallback(info, 'arithmetic coding')
        elif 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            if m not in (0xC0, 0xC1):
                return _fallback(info, 'SOF%d (not baseline / extended Huffman)' % (m - 0xC0))
            if sof is not None:
                return _fallback(info, 'two frames')
            sof = m
            if seg[0] != 8:
                return _fallback(info, '%d-bit samples' % seg[0])
            info.height, info.width = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4]
            nc = seg[5]
            info.comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(nc)]
        elif m == 0xDA:
            if sof is None:
                return _fallback(info, 'scan before frame')
            ns = seg[0]
            ids = [c[0] for c in info.comps]
            scan = []
            for k in range(ns):
                cid, t = seg[1 + 2 * k], seg[2 + 2 * k]
                if cid not in ids:
                    return _fallback(info, 'scan names an unknown component')
                scan.append((ids.index(cid), t >> 4, t & 15))
            ss, se, a = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            info.scan = scan
            start = pos + 2 + length
            _locate_ecs(d, start, info)
            return _classify(info, jfif, adobe, transform, (ss, se, a))
        elif m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7:
            return _fallback(info, 'marker 0x%02X before the scan' % m)
        pos += 2 + length


def _locate_ecs(d, start, info):
    """The ECS runs from ``start`` to the first marker that is neither a stuffed 0xFF00 nor RSTn (the end of the data
    when there is none: a truncated file keeps its bytes, and the decoder reports the premature end).  0xFF fill bytes
    before a marker (T.81 B.1.1.2) stay inside it: the decoders stop reading an interval at its first 0xFF that is not
    stuffing."""
    a = np.frombuffer(d, np.uint8)
    ff = np.flatnonzero(a[start:-1] == 0xFF) + start
    nxt = a[ff + 1]
    is_rst = (nxt >= 0xD0) & (nxt <= 0xD7)
    ends = ff[(nxt != 0) & (nxt != 0xFF) & ~is_rst]
    end = int(ends[0]) if ends.size else len(a)
    info.ecs = (start, end)
    rst = ff[is_rst]
    info.rst = (rst[rst < end] + 2).astype(np.int64)
    info.after_ecs = bytes(a[end:end + 2])


def _classify(info, jfif, adobe, transform, spectral):
    comps = info.comps
    if info.height < 1 or info.width < 1:
        return _fallback(info, 'no image size in the frame (DNL)')
    if spectral != (0, 63, 0):
        return _fallback(info, 'not a sequential scan')
    if len(comps) not in (1, 3):
        return _fallback(info, '%d components' % len(comps))
    if [c for c, _, _ in info.scan] != list(range(len(comps))):
        return _fallback(info, 'the scan does not hold every component in frame order (multi-scan)')
    if info.after_ecs not in (b'\xff\xd9', b''):
        return _fallback(info, 'more than one scan')
    if len(comps) == 3:
        (i0, h0, v0, _), (i1, h1, v1, _), (i2, h2, v2, _) = comps
        if (h0, v0) not in ((1, 1), (2, 1), (2, 2)) or (h1, v1, h2, v2) != (1, 1, 1, 1):
            return _fallback(info, 'sampling %dx%d,%dx%d,%dx%d' % (h0, v0, h1, v1, h2, v2))
        if adobe and not jfif and transform != 1:
            return _fallback(info, 'Adobe transform %d' % transform)
        if not jfif and not adobe and (i0, i1, i2) == (82, 71, 66):
            return _fallback(info, 'RGB component ids')
    for (ci, td, ta) in info.scan:
        tq = comps[ci][3]
        if tq not in info.qt or td not in info.dc or ta not in info.ac:
            return _fallback(info, 'a table the scan uses is missing')
        if int(info.qt[tq].max()) > 32767:
            return _fallback(info, 'quantisation entries above 32767')
    info.device, info.reason = True, 'baseline'
    return info
