"""A small baseline / extended-Huffman JPEG writer for the decode tests, written from T.81 (annexes B, C, F and K).

It writes the streams Pillow's encoder never does: any component ids, sampling factors and table slots, 8- or 16-bit
DQT, the annex K Huffman tables or any canonical table built from code lengths (codes up to 16 bits, code space left
unused), DRI with fill bytes before the markers, extra APPn / COM segments, JFIF and Adobe markers, SOF0 or SOF1 --
and, on request, damaged entropy-coded data: a code from the unused code space, an AC run past coefficient 63, an
out-of-sequence RSTn, or a segment that ends in the middle of an MCU.

``encode(comps, blocks, width, height, qt, dc, ac, ...)`` takes the quantised coefficients of every block of every
component (int [block rows, block columns, 64], natural order) and returns the file bytes.  ``fdct(plane, q)`` makes
such blocks from a sample plane.
"""
import numpy as np

# zig-zag position k -> natural (row-major) index (T.81 figure A.6)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                   31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

SOS, DQT, DHT, DRI, COM = 0xDA, 0xDB, 0xC4, 0xDD, 0xFE


class Huff(object):
    """A canonical Huffman table (T.81 annex C): ``bits`` [16] the number of codes of each length 1..16, ``vals`` the
    symbols in code order; ``codes`` {symbol: (code, length)}."""

    def __init__(self, bits, vals):
        self.bits, self.vals = [int(b) for b in bits], [int(v) for v in vals]
        assert len(self.bits) == 16 and sum(self.bits) == len(self.vals)
        self.codes, code, k = {}, 0, 0
        for l in range(1, 17):
            for _ in range(self.bits[l - 1]):
                self.codes[self.vals[k]] = (code, l)
                code, k = code + 1, k + 1
            assert code <= (1 << l), 'over-full code lengths'
            code <<= 1
        self.spare = (1 << 16) - (code >> 1)       # unused 16-bit code space (in units of 2**-16)

    def unused_code(self):
        """(code, 16): a 16-bit string no code of the table is a prefix of (the table must leave space unused)."""
        assert self.spare > 0
        return (1 << 16) - 1, 16

    @classmethod
    def from_lengths(cls, lengths):
        """{symbol: code length} -> the canonical table, symbols ordered by length and then by value."""
        order = sorted(lengths, key=lambda s: (lengths[s], s))
        bits = [0] * 16
        for s in order:
            bits[lengths[s] - 1] += 1
        return cls(bits, order)


def spread(symbols, long=(), long_lengths=(10, 11, 12, 13, 14, 15, 16)):
    """A table of ``symbols``: those in ``long`` get code lengths cycling over ``long_lengths`` (the decoders' paths
    past their lookahead), every other symbol the shortest common length that still leaves code space unused."""
    long = [s for s in symbols if s in set(long)]
    lengths = {s: long_lengths[i % len(long_lengths)] for i, s in enumerate(long)}
    used = sum(2.0 ** -l for l in lengths.values())
    short = [s for s in symbols if s not in lengths]
    L = 1
    while short and len(short) * 2.0 ** -L + used >= 1.0:
        L += 1
    lengths.update({s: L for s in short})
    return Huff.from_lengths(lengths)


DC_SYMBOLS = list(range(16))                                              # size categories 0..15
AC_SYMBOLS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)]   # EOB, ZRL, every run / size


# T.81 annex K.3: the example tables (K.3 / K.4 DC, K.5 / K.6 AC), luminance and chrominance
K_DC_LUMA = Huff([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], range(12))
K_DC_CHROMA = Huff([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], range(12))


def _k_ac_luma():
    head = [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
            0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0,
            0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28,
            0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A]
    rest = [(hi << 4) | lo for hi in (4, 5, 6, 7, 8) for lo in range(3, 11)]
    rest += [(hi << 4) | lo for hi in (9, 10, 11, 12, 13) for lo in range(2, 11)]
    rest += [(hi << 4) | lo for hi in (14, 15) for lo in range(1, 11)]
    return Huff([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], head + rest)


def _k_ac_chroma():
    head = [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
            0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0,
            0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26,
            0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A]
    rest = [(hi << 4) | lo for hi in (4, 5, 6, 7) for lo in range(3, 11)]
    rest += [(hi << 4) | lo for hi in (8, 9, 10, 11, 12, 13, 14, 15) for lo in range(2, 11)]
    return Huff([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], head + rest)


K_AC_LUMA, K_AC_CHROMA = _k_ac_luma(), _k_ac_chroma()
FULL_DC, FULL_AC = spread(DC_SYMBOLS), spread(AC_SYMBOLS)       # every symbol a baseline scan may use


def fdct(plane, q):
    """uint8 [8R, 8C] samples, int [64] quantisation (natural order) -> int64 [R, C, 64] quantised coefficients of the
    T.81 A.3.3 FDCT, rounded to nearest."""
    R, C = plane.shape[0] // 8, plane.shape[1] // 8
    k = np.arange(8)
    m = np.cos((2 * k[None, :] + 1) * k[:, None] * np.pi / 16) * np.where(k == 0, np.sqrt(0.5), 1.0)[:, None] / 2
    b = plane[:8 * R, :8 * C].astype(np.float64).reshape(R, 8, C, 8).transpose(0, 2, 1, 3) - 128
    f = np.einsum('ux,rcxy,vy->rcuv', m, b, m).reshape(R, C, 64)
    return np.round(f / np.asarray(q, np.float64)).astype(np.int64)


def pad_plane(a, rows, cols):
    """Replicate a plane's last row and column out to rows x cols samples."""
    return np.pad(a, ((0, rows - a.shape[0]), (0, cols - a.shape[1])), mode='edge')


class _Bits(object):
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, code, length):
        for i in range(length - 1, -1, -1):
            self.acc = (self.acc << 1) | ((code >> i) & 1)
            self.n += 1
            if self.n == 8:
                self.out.append(self.acc)
                if self.acc == 0xFF:
                    self.out.append(0)                  # byte stuffing (F.1.2.3)
                self.acc, self.n = 0, 0

    def flush(self, pad=1):
        """Pad to a byte boundary with ``pad`` bits (1 as T.81 F.1.2.3 asks)."""
        if self.n:
            self.put((1 << (8 - self.n)) - 1 if pad else 0, 8 - self.n)


def _size(v):
    return int(abs(int(v))).bit_length()


def _put_value(w, v, s):
    w.put(int(v) if v >= 0 else int(v) + (1 << s) - 1, s)


def _segment(marker, payload, fill=0):
    assert len(payload) + 2 < 65536
    return b'\xff' * fill + bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, 'big') + bytes(payload)


def jfif():
    return (0xE0, b'JFIF\0\x01\x01\x00\x00\x01\x00\x01\x00\x00')


def adobe(transform):
    return (0xEE, b'Adobe\x00\x64\x00\x00\x00\x00' + bytes([transform]))


def dqt(slot, q, wide=False):
    """DQT payload of one table (q natural order), 8-bit entries or 16-bit (Pq = 1)."""
    zz = np.asarray(q, np.int64)[ZIGZAG]
    if wide:
        return bytes([0x10 | slot]) + zz.astype('>u2').tobytes()
    assert zz.min() >= 1 and zz.max() <= 255
    return bytes([slot]) + zz.astype(np.uint8).tobytes()


def dht(tc, slot, t):
    return bytes([(tc << 4) | slot] + t.bits + t.vals)


def encode(comps, blocks, width, height, qt, dc, ac, sof=0xC0, markers=(jfif(),), restart=0, fill=0, rst_fill=0,
           wide_q=(), extra=(), tables_after_sof=False, redefine=False, damage=None):
    """-> JPEG bytes of one interleaved scan (one block per MCU for a single component, whatever its sampling).

    comps: [(id, h, v, tq, td, ta)] in frame order; blocks: [int [rows, cols, 64] natural order] per component, at
    least (MCU rows * v) x (MCU columns * h) blocks (DC values absolute, so a predictor may run past int16 as long as
    each difference fits in 15 bits); qt: {slot: int [64]}; dc / ac: {slot: Huff}; markers: APPn / COM segments
    (marker, payload) after SOI; restart: DRI interval in MCUs; fill / rst_fill: 0xFF fill bytes before each header
    marker and EOI / before each RSTn; wide_q: DQT slots written with 16-bit entries; extra: (position, marker,
    payload) segments inserted at that position of the table segments; tables_after_sof: DQT after the frame header;
    redefine: define every table first with other contents, then again with its own; damage: (kind, MCU) with kind
    'code' (a code from the unused space for the MCU's first DC), 'run' (an AC run past coefficient 63 in the MCU's
    last block), 'restart' (the restart marker ending the MCU's interval gets the next marker's number) or 'short'
    (the segment ends, zero-padded, just after the MCU's first DC code)."""
    nc = len(comps)
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    samp = [(1, 1)] if nc == 1 else [(c[1], c[2]) for c in comps]
    if nc == 1:
        hmax = vmax = 1
    mcux, mcuy = -(-width // (8 * hmax)), -(-height // (8 * vmax))
    kind, at = damage if damage else (None, -1)

    tables = []
    for slot in sorted(qt):
        if redefine:
            tables.append((DQT, dqt(slot, np.full(64, 7 + slot), slot in wide_q)))
        tables.append((DQT, dqt(slot, qt[slot], slot in wide_q)))
    huffs = []
    for tc, ts in ((0, dc), (1, ac)):
        for slot in sorted(ts):
            if redefine:
                huffs.append((DHT, dht(tc, slot, FULL_AC if tc else FULL_DC)))
            huffs.append((DHT, dht(tc, slot, ts[slot])))
    frame = bytes([8]) + height.to_bytes(2, 'big') + width.to_bytes(2, 'big') + bytes([nc]) + \
        b''.join(bytes([c[0], (c[1] << 4) | c[2], c[3]]) for c in comps)
    segs = tables + huffs if not tables_after_sof else huffs
    for pos, m, p in sorted(extra, key=lambda e: e[0], reverse=True):
        segs.insert(pos, (m, p))
    segs = list(markers) + segs + [(sof, frame)] + (tables if tables_after_sof else [])
    if restart:
        segs.append((DRI, restart.to_bytes(2, 'big')))
    scan = bytes([nc]) + b''.join(bytes([c[0], (c[4] << 4) | c[5]]) for c in comps) + b'\x00\x3f\x00'
    segs.append((SOS, scan))

    w, ecs, pred, n_rst = _Bits(), bytearray(), [0] * nc, 0
    total = mcux * mcuy
    for m in range(total):
        my, mx = divmod(m, mcux)
        for c, (h, v) in enumerate(samp):
            hd, ha = dc[comps[c][4]], ac[comps[c][5]]
            for bv in range(v):
                for bh in range(h):
                    blk = blocks[c][my * v + bv, mx * h + bh]
                    first = m == at and c == 0 and bv == 0 and bh == 0
                    last = m == at and c == nc - 1 and bv == v - 1 and bh == h - 1
                    diff = int(blk[0]) - pred[c]
                    pred[c] = int(blk[0])
                    s = _size(diff)
                    assert s <= 15, 'DC difference %d does not fit' % diff
                    if first and kind == 'code':
                        w.put(*hd.unused_code())
                    w.put(*hd.codes[s])
                    _put_value(w, diff, s)
                    if first and kind == 'short':
                        w.flush(pad=0)
                        ecs += w.out
                        return _assemble(segs, fill, bytes(ecs))
                    if last and kind == 'run':
                        for _ in range(3):
                            w.put(*ha.codes[0xF0])               # ZRL x3: the next coefficient is k = 49
                        w.put(*ha.codes[0xF1])                   # run 15 -> k = 64
                        w.put(1, 1)
                    zz = np.asarray(blk, np.int64)[ZIGZAG]
                    run = 0
                    for k in range(1, 64):
                        a = int(zz[k])
                        if a == 0:
                            run += 1
                            continue
                        while run > 15:
                            w.put(*ha.codes[0xF0])
                            run -= 16
                        s = _size(a)
                        assert 1 <= s <= 15, 'AC value %d does not fit' % a
                        w.put(*ha.codes[(run << 4) | s])
                        _put_value(w, a, s)
                        run = 0
                    if run:
                        w.put(*ha.codes[0x00])
        if restart and (m + 1) % restart == 0 and m + 1 < total:
            w.flush()
            ecs += w.out
            w.out = bytearray()
            num = n_rst + (1 if kind == 'restart' and at // restart == n_rst else 0)
            ecs += b'\xff' * rst_fill + bytes([0xFF, 0xD0 + (num & 7)])
            n_rst += 1
            pred = [0] * nc
    w.flush()
    ecs += w.out
    return _assemble(segs, fill, bytes(ecs))


def _assemble(segs, fill, ecs):
    return b'\xff\xd8' + b''.join(_segment(m, p, fill) for m, p in segs) + ecs + b'\xff' * fill + b'\xff\xd9'
