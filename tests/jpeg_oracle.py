"""numpy restatement of the device JPEG decode (csrc/jpeg.cu): baseline Huffman decode, the integer ISLOW IDCT as
libjpeg-turbo's x86-64 SIMD code computes it (16-bit dequantisation and sums, saturating stores), fancy upsampling
(h2v1, h2v2) and libjpeg's fixed-point YCbCr -> RGB.  It is the spec the
kernels are written against; the CPU tests pin it to Pillow's decode and the GPU tests pin the kernels to Pillow.

decode(data) -> uint8 [H, W, 3], the bytes of np.asarray(Image.open(f).convert('RGB')), for a file whose
utils.jpeg.parse(data).device is True.
"""
import numpy as np

from convnet.pytorch_b200.utils import jpeg


def _huff_decode(bits, pos, t):
    """(value, new pos) of one Huffman symbol of table t read from the '0'/'1' string ``bits`` at ``pos``."""
    code, l = 0, 0
    while l < 17:
        code = (code << 1) | (1 if bits[pos + l] == '1' else 0) if pos + l < len(bits) else code << 1
        l += 1
        if l <= 16 and t.maxcode[l] >= 0 and code <= t.maxcode[l]:
            return int(t.huffval[code + t.valoffset[l]]), pos + l
    raise ValueError('bad Huffman code')


def _receive(bits, pos, s):
    if s == 0:
        return 0, pos
    if pos + s > len(bits):
        raise ValueError('premature end of data')
    v = int(bits[pos:pos + s], 2)
    if v < (1 << (s - 1)):
        v += (-1 << s) + 1
    return v, pos + s


def _unstuff(seg):
    a = np.frombuffer(seg, np.uint8)
    keep = np.ones(a.size, bool)
    keep[1:] = ~((a[:-1] == 0xFF) & (a[1:] == 0x00))
    return ''.join(np.unpackbits(a[keep]).astype(str))


def entropy_decode(data, info):
    """-> [int16 [rows, cols, 64] natural-order coefficient blocks per component]."""
    hmax, vmax = info.sampling
    mx, my = info.mcus
    samp = [(1, 1)] if info.channels == 1 else [(c[1], c[2]) for c in info.comps]
    blocks = [np.zeros((my * v, mx * h, 64), np.int16) for h, v in samp]
    total = mx * my
    ri = info.restart or total
    starts = [info.ecs[0]] + [int(p) for p in info.rst]
    for k in range(-(-total // ri)):
        if k >= len(starts):
            raise ValueError('missing restart marker')
        end = info.ecs[1] if k + 1 >= len(starts) else starts[k + 1] - 2
        bits, pos = _unstuff(bytes(data[starts[k]:end])), 0
        pred = [0] * len(samp)
        for m in range(k * ri, min((k + 1) * ri, total)):
            my_, mx_ = divmod(m, mx)
            for c, (h, v) in enumerate(samp):
                _, td, ta = info.scan[c]
                for bv in range(v):
                    for bh in range(h):
                        blk = blocks[c][my_ * v + bv, mx_ * h + bh]
                        s, pos = _huff_decode(bits, pos, info.dc[td])
                        diff, pos = _receive(bits, pos, s)
                        pred[c] = pred[c] + diff
                        blk[0] = np.int32(pred[c]).astype(np.int16)
                        i = 1
                        while i < 64:
                            rs, pos = _huff_decode(bits, pos, info.ac[ta])
                            r, s = rs >> 4, rs & 15
                            if s:
                                i += r
                                if i > 63:
                                    raise ValueError('coefficient index past 63')
                                blk[jpeg.NATURAL_ORDER[i]], pos = _receive(bits, pos, s)
                                i += 1
                            elif r == 15:
                                i += 16
                            else:
                                break
    return blocks


_F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
          f1961=16069, f2053=16819, f2562=20995, f3072=25172)


def s16(x):
    """The low 16 bits of int64 values, as a signed int16 (two's-complement wrap)."""
    return ((x + 32768) & 0xFFFF) - 32768


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7, descale):
    """One pass of libjpeg-turbo's SIMD ISLOW IDCT (jidctint-sse2 / -avx2) over int64 arrays of int16 values -> the 8
    outputs, DESCALEd by ``descale`` and saturated to int16.  It is jidctint.c's algorithm with the products paired
    as its comments rewrite them (pmaddwd), and with x0 +- x4 and the odd part's z3 = x7 + x3, z4 = x5 + x1 added in
    16 bits (paddw, wrapping)."""
    f = _F
    tmp3 = x2 * (f['f0541'] + f['f0765']) + x6 * f['f0541']
    tmp2 = x2 * f['f0541'] + x6 * (f['f0541'] - f['f1847'])
    tmp0 = s16(x0 + x4) << 13
    tmp1 = s16(x0 - x4) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    z3, z4 = s16(x7 + x3), s16(x5 + x1)
    z3, z4 = z3 * (f['f1175'] - f['f1961']) + z4 * f['f1175'], z3 * f['f1175'] + z4 * (f['f1175'] - f['f0390'])
    t0 = x7 * (f['f0298'] - f['f0899']) + x1 * -f['f0899'] + z3
    t3 = x7 * -f['f0899'] + x1 * (f['f1501'] - f['f0899']) + z4
    t1 = x5 * (f['f2053'] - f['f2562']) + x3 * -f['f2562'] + z4
    t2 = x5 * -f['f2562'] + x3 * (f['f3072'] - f['f2562']) + z3
    r = 1 << (descale - 1)
    return [np.clip((v + r) >> descale, -32768, 32767) for v in (tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0,
                                                                tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3)]


def idct(blocks, q):
    """int16 [..., 64] coefficient blocks, int [64] quantisation (natural order) -> uint8 [..., 8, 8] samples, as
    libjpeg-turbo's x86-64 SIMD ISLOW makes them: dequantisation keeps the low 16 bits of coef * q; a block whose
    coefficient rows 1..7 are all zero takes the shortcut of pass 1, every column s16(dq0 << 2); the final store
    saturates to [-128, 127] and adds 128."""
    raw = blocks.astype(np.int64).reshape(-1, 8, 8)
    c = s16(raw * np.asarray(q, np.int64).reshape(8, 8))
    ws = np.stack(_idct_1d(*[c[:, k, :] for k in range(8)], 13 - 2), axis=1)    # pass 1: columns -> [N, row, col]
    flat = ~raw[:, 1:, :].any(axis=(1, 2))
    ws[flat] = s16(c[flat, 0:1, :] << 2)
    rows = _idct_1d(*[ws[:, :, k] for k in range(8)], 13 + 2 + 3)              # pass 2: rows
    out = np.stack(rows, axis=2)
    return (np.clip(out, -128, 127) + 128).astype(np.uint8).reshape(blocks.shape[:-1] + (8, 8))


def planes(data, info):
    """-> [uint8 component planes, block-padded]."""
    blocks = entropy_decode(data, info)
    out = []
    for c, b in enumerate(blocks):
        tq = info.comps[info.scan[c][0]][3]
        s = idct(b, info.qt[tq])                                          # [rows, cols, 8, 8]
        out.append(s.transpose(0, 2, 1, 3).reshape(b.shape[0] * 8, b.shape[1] * 8))
    return out


def upsample(p, cw, ch, hmax, vmax, H, W):
    """uint8 chroma plane (real size ch x cw) -> int [H, W] as libjpeg-turbo's upsampler makes it: fancy h2v1 / h2v2
    with replicated edges, plain replication when the downsampled width is 2 or less."""
    p = p[:ch, :cw].astype(np.int64)
    y, x = np.arange(H), np.arange(W)
    if hmax == 1:
        return p[y][:, x]
    if cw <= 2:
        return p[(y // vmax)][:, x // 2]
    i = x >> 1
    left = np.clip(i - 1, 0, cw - 1)
    right = np.clip(i + 1, 0, cw - 1)
    if vmax == 1:
        s = p[y]
        return np.where(x % 2 == 0, (3 * s[:, i] + s[:, left] + 1) >> 2, (3 * s[:, i] + s[:, right] + 2) >> 2)
    r = y >> 1
    far = np.clip(np.where(y % 2 == 0, r - 1, r + 1), 0, ch - 1)
    col = 3 * p[r] + p[far]                                              # [H, cw]
    return np.where(x % 2 == 0, (3 * col[:, i] + col[:, left] + 8) >> 4, (3 * col[:, i] + col[:, right] + 7) >> 4)


def ycc_to_rgb(y, cb, cr):
    """libjpeg's jdcolor.c ycc_rgb_convert (16-bit fixed point, arithmetic shifts, range limit)."""
    one_half = 1 << 15
    cb, cr = cb.astype(np.int64) - 128, cr.astype(np.int64) - 128
    r = y + ((91881 * cr + one_half) >> 16)
    g = y + ((-22554 * cb + one_half - 46802 * cr) >> 16)
    b = y + ((116130 * cb + one_half) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data, info=None):
    """bytes of a device-class JPEG -> uint8 [H, W, 3]."""
    info = info or jpeg.parse(data)
    if not info.device:
        raise ValueError('not a device-class JPEG: %s' % info.reason)
    H, W = info.height, info.width
    pl = planes(data, info)
    y = pl[0][:H, :W].astype(np.int64)
    if info.channels == 1:
        return np.repeat(y[:, :, None], 3, axis=2).astype(np.uint8)
    hmax, vmax = info.sampling
    cw, ch = -(-W // hmax), -(-H // vmax)
    cb = upsample(pl[1], cw, ch, hmax, vmax, H, W)
    cr = upsample(pl[2], cw, ch, hmax, vmax, H, W)
    return ycc_to_rgb(y, cb, cr)
