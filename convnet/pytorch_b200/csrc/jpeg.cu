// Baseline JPEG decode on the device (b200_jpeg_decode): the loader workers parse headers (utils/jpeg.py) and ship the
// entropy-coded segments; three kernels turn them into the uint8 HWC regions the resized-crop and scale-crop relayouts
// read, byte for byte what Pillow (libjpeg-turbo on x86-64, SIMD ISLOW IDCT, fancy upsampling) decodes.
// tests/jpeg_oracle.py is the numpy statement of the same arithmetic.
//   1. jpeg_huffman_kernel: one thread per restart interval (the whole image without restart markers) decodes Huffman
//      codes into int16 coefficient blocks (natural order), up to the last MCU row the region needs;
//   2. jpeg_idct_kernel: one thread per 8x8 block the region's pixels (and their upsampling context) depend on runs
//      the ISLOW IDCT as libjpeg-turbo's x86-64 SIMD code computes it (16-bit dequantisation and sums, saturating
//      stores; its C jpeg_idct_islow differs on out-of-range blocks) into block-padded uint8 component planes;
//   3. jpeg_color_kernel: one thread per region pixel upsamples the chroma (h2v1 / h2v2 fancy, box when the chroma is
//      at most 2 samples wide), converts YCbCr -> RGB in libjpeg's fixed point and writes HWC RGB; grayscale images are
//      replicated to RGB, and images the workers decoded with PIL are copied from the payload.
#include <cuda_runtime.h>
#include <stdint.h>

#include "host.h"

namespace {

// descriptor words (int64 [B][kDescWords], built by utils/augment.py JpegCollate)
enum {
  D_KIND, D_H, D_W, D_HMAX, D_VMAX, D_MCUX, D_MCUY, D_MCUROWS, D_RI, D_ECS0, D_ECS1,
  D_Q0, D_Q1, D_Q2, D_DC0, D_DC1, D_DC2, D_AC0, D_AC1, D_AC2,
  D_COEF, D_PLANE, D_Y0, D_X0, D_RH, D_RW, D_OUT, D_SRC, D_PIX
};
constexpr int kDescWords = 32;
constexpr int kKindColor = 0, kKindGray = 1, kKindHost = 2;
constexpr int kLookahead = 9;                         // utils/jpeg.py LOOKAHEAD
constexpr int kLutWord = 36, kValWord = 36 + (1 << kLookahead) / 2;
constexpr int kBadCode = 1, kShortData = 2, kBadRestart = 4, kBadIndex = 8;

__constant__ unsigned char kNatural[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                           12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                           58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// MSB-first bit reader over one image's ECS bytes [pos, end): removes byte stuffing, stops at the first marker and
// feeds zero bits past the data.  `pad` counts those zero bits: consuming into them is a premature end.
struct Bits {
  const uint8_t* p;
  long long pos, end;
  unsigned long long acc;
  int nbits, pad;

  __device__ __forceinline__ void fill() {
    while (nbits <= 56) {
      unsigned b = 0;
      if (pos < end) {
        b = __ldg(p + pos);
        if (b == 0xFF) {
          const unsigned n = pos + 1 < end ? __ldg(p + pos + 1) : 0xFFu;
          if (n == 0) {
            pos += 2;
          } else {
            end = pos;          // a marker: the data of this interval ends here
            b = 0;
            pad += 8;
          }
        } else {
          pos += 1;
        }
      } else {
        pad += 8;
      }
      acc |= (unsigned long long)b << (56 - nbits);
      nbits += 8;
    }
  }
  __device__ __forceinline__ void skip(int n) {
    acc <<= n;
    nbits -= n;
  }
  // the next s (<= 16) bits as T.81's EXTEND(RECEIVE(s))
  __device__ __forceinline__ int receive(int s) {
    if (s == 0) return 0;
    int v = (int)(acc >> (64 - s));
    skip(s);
    return v < (1 << (s - 1)) ? v + (-1 << s) + 1 : v;
  }
  // one Huffman symbol of the packed table T (utils/jpeg.py HuffTable.pack); needs >= 16 buffered bits
  __device__ __forceinline__ int huff(const int* __restrict__ T, int& err) {
    const unsigned look = (unsigned)(acc >> (64 - kLookahead));
    const int e = __ldg(reinterpret_cast<const short*>(T + kLutWord) + look);
    if (e) {
      skip(e >> 8);
      return e & 255;
    }
    for (int l = kLookahead + 1; l <= 16; ++l) {
      const int code = (int)(acc >> (64 - l));
      if (code <= __ldg(T + l)) {
        skip(l);
        return __ldg(reinterpret_cast<const uint8_t*>(T + kValWord) + ((code + __ldg(T + 18 + l)) & 255));
      }
    }
    err |= kBadCode;
    return 0;
  }
};

__device__ __forceinline__ int comp_h(const long long* d, int c) { return c == 0 ? (int)d[D_HMAX] : 1; }
__device__ __forceinline__ int comp_v(const long long* d, int c) { return c == 0 ? (int)d[D_VMAX] : 1; }
__device__ __forceinline__ int ncomp(const long long* d) { return d[D_KIND] == kKindColor ? 3 : 1; }

// intervals: int64 [n][3] {image, interval number, first byte (after its RSTn marker)}
__global__ void jpeg_huffman_kernel(const uint8_t* __restrict__ payload, const long long* __restrict__ desc,
                                    const long long* __restrict__ intervals, int n_intervals, int per_block,
                                    short* __restrict__ coef, int* __restrict__ status) {
  if ((int)threadIdx.x >= per_block) return;
  const int t = blockIdx.x * per_block + threadIdx.x;
  if (t >= n_intervals) return;
  const long long* iv = intervals + 3LL * t;
  const int b = (int)iv[0];
  const long long k = iv[1], start = iv[2];
  const long long* d = desc + (long long)b * kDescWords;
  if (d[D_KIND] == kKindHost) return;
  const long long mcux = d[D_MCUX], total = mcux * d[D_MCUY];
  const long long ri = d[D_RI] > 0 ? d[D_RI] : total;
  const long long m0 = k * ri, m1 = min(min(m0 + ri, total), d[D_MCUROWS] * mcux);
  if (m0 >= m1) return;
  if (k > 0 && (start - 2 < d[D_ECS0] || payload[start - 2] != 0xFF || payload[start - 1] != 0xD0 + ((k - 1) & 7))) {
    atomicOr(status + b, kBadRestart);
    return;
  }
  const int nc = ncomp(d);
  Bits r{payload, start, d[D_ECS1], 0ULL, 0, 0};
  int pred[3] = {0, 0, 0};
  int err = 0;
  alignas(16) short blk[64];
  for (long long m = m0; m < m1; ++m) {
    const long long my = m / mcux, mx = m - my * mcux;
    long long base = d[D_COEF];
    for (int c = 0; c < nc; ++c) {
      const int h = comp_h(d, c), v = comp_v(d, c);
      const int* dc = reinterpret_cast<const int*>(payload + d[D_DC0 + c]);
      const int* ac = reinterpret_cast<const int*>(payload + d[D_AC0 + c]);
      const long long bw = mcux * h;
      for (int bv = 0; bv < v; ++bv) {
        for (int bh = 0; bh < h; ++bh) {
#pragma unroll
          for (int i = 0; i < 64; ++i) blk[i] = 0;
          r.fill();
          const int s = r.huff(dc, err);
          pred[c] += r.receive(s);       // int arithmetic wraps as libjpeg's last_dc_val does
          blk[0] = (short)pred[c];
          for (int i = 1; i < 64;) {
            r.fill();
            const int rs = r.huff(ac, err);
            const int run = rs >> 4, sz = rs & 15;
            if (sz) {
              i += run;
              if (i > 63) {
                err |= kBadIndex;
                break;
              }
              blk[kNatural[i]] = (short)r.receive(sz);
              ++i;
            } else if (run == 15) {
              i += 16;
            } else {
              break;
            }
          }
          const long long idx = base + (my * v + bv) * bw + mx * h + bh;
          int4* dst = reinterpret_cast<int4*>(coef + idx * 64);
          const int4* src = reinterpret_cast<const int4*>(blk);
#pragma unroll
          for (int i = 0; i < 8; ++i) dst[i] = src[i];
        }
      }
      base += bw * d[D_MCUY] * v;
    }
    if (err || r.nbits < r.pad) {
      atomicOr(status + b, err ? err : kShortData);
      return;
    }
  }
}

// index of the last image whose prefix word d[w] is <= x (prefixes ascend with the image index)
__device__ __forceinline__ int find_image(const long long* __restrict__ desc, int B, int w, long long x) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (desc[(long long)mid * kDescWords + w] <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// [lo, hi] sample indices of a component (sampling f of fmax) that region [a, a + n) reads, upsampling context included
__device__ __forceinline__ void comp_span(long long a, long long n, int f, int fmax, long long& lo, long long& hi) {
  if (f == fmax) {
    lo = a;
    hi = a + n - 1;
  } else {
    lo = a / fmax - 1;
    hi = (a + n - 1) / fmax + 1;
  }
}

constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ int s16(int x) { return (short)x; }        // paddw / pmullw: keep the low 16 bits
__device__ __forceinline__ short sat16(int x) { return (short)(x < -32768 ? -32768 : (x > 32767 ? 32767 : x)); }

// one pass of libjpeg-turbo's SIMD ISLOW IDCT (jidctint-sse2 / -avx2) over x[0..7] (stride s), DESCALEd by n and
// saturated to int16 (packssdw) into o[0..7]: jidctint.c's algorithm with its products paired as pmaddwd forms them,
// and x0 +- x4 and the odd part's z3 = x7 + x3, z4 = x5 + x1 summed in 16 bits.  No 32-bit sum can overflow.
__device__ __forceinline__ void idct8(const short* x, int s, short* o, int os, int n) {
  const int x0 = x[0], x1 = x[s], x2 = x[2 * s], x3 = x[3 * s], x4 = x[4 * s], x5 = x[5 * s], x6 = x[6 * s],
            x7 = x[7 * s];
  const int tmp3 = x2 * (F0541 + F0765) + x6 * F0541, tmp2 = x2 * F0541 + x6 * (F0541 - F1847);
  const int tmp0 = s16(x0 + x4) * 8192, tmp1 = s16(x0 - x4) * 8192;
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  const int z3 = s16(x7 + x3), z4 = s16(x5 + x1);
  const int z3f = z3 * (F1175 - F1961) + z4 * F1175, z4f = z3 * F1175 + z4 * (F1175 - F0390);
  const int t0 = x7 * (F0298 - F0899) + x1 * -F0899 + z3f, t3 = x7 * -F0899 + x1 * (F1501 - F0899) + z4f;
  const int t1 = x5 * (F2053 - F2562) + x3 * -F2562 + z4f, t2 = x5 * -F2562 + x3 * (F3072 - F2562) + z3f;
  const int r = 1 << (n - 1);
  o[0] = sat16((tmp10 + t3 + r) >> n); o[7 * os] = sat16((tmp10 - t3 + r) >> n);
  o[os] = sat16((tmp11 + t2 + r) >> n); o[6 * os] = sat16((tmp11 - t2 + r) >> n);
  o[2 * os] = sat16((tmp12 + t1 + r) >> n); o[5 * os] = sat16((tmp12 - t1 + r) >> n);
  o[3 * os] = sat16((tmp13 + t0 + r) >> n); o[4 * os] = sat16((tmp13 - t0 + r) >> n);
}

__global__ void jpeg_idct_kernel(const uint8_t* __restrict__ payload, const long long* __restrict__ desc, int B,
                                 long long n_blocks, const short* __restrict__ coef, uint8_t* __restrict__ planes) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_blocks) return;
  const int b = find_image(desc, B, D_COEF, t);
  const long long* d = desc + (long long)b * kDescWords;
  if (d[D_KIND] == kKindHost) return;
  long long local = t - d[D_COEF], plane = d[D_PLANE];
  const int nc = ncomp(d), hmax = (int)d[D_HMAX], vmax = (int)d[D_VMAX];
  for (int c = 0; c < nc; ++c) {
    const int h = comp_h(d, c), v = comp_v(d, c);
    const long long bw = d[D_MCUX] * h, bh = d[D_MCUY] * v;
    if (local >= bw * bh) {
      local -= bw * bh;
      plane += bw * bh * 64;
      continue;
    }
    const long long by = local / bw, bx = local - by * bw;
    if (by >= d[D_MCUROWS] * v) return;                       // below the rows the entropy decode stopped at
    long long ylo, yhi, xlo, xhi;
    comp_span(d[D_Y0], d[D_RH], v, vmax, ylo, yhi);
    comp_span(d[D_X0], d[D_RW], h, hmax, xlo, xhi);
    if (by * 8 + 7 < ylo || by * 8 > yhi || bx * 8 + 7 < xlo || bx * 8 > xhi) return;
    const int* q = reinterpret_cast<const int*>(payload + d[D_Q0 + c]);
    alignas(16) short in[64];
    const int4* src = reinterpret_cast<const int4*>(coef + t * 64);
    int ac = 0;                                               // OR of coefficient rows 1..7 (one int4 per row)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int4 w = src[i];
      reinterpret_cast<int4*>(in)[i] = w;
      if (i > 0) ac |= w.x | w.y | w.z | w.w;
    }
    short dq[64], ws[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) dq[i] = (short)((int)in[i] * __ldg(q + i));   // pmullw: the low 16 bits
    if (ac == 0) {
      // pass 1's shortcut when every AC row is zero: each column is dq0 << 2, wrapped to 16 bits (psllw)
#pragma unroll
      for (int i = 0; i < 64; ++i) ws[i] = (short)(dq[i & 7] * 4);
    } else {
#pragma unroll
      for (int col = 0; col < 8; ++col) idct8(dq + col, 8, ws + col, 8, 11);     // pass 1: columns
    }
    alignas(8) uint8_t row[8];
    short o[8];
    for (int y = 0; y < 8; ++y) {
      idct8(ws + 8 * y, 1, o, 1, 18);                                         // pass 2: rows
#pragma unroll
      for (int i = 0; i < 8; ++i) row[i] = (uint8_t)(o[i] < -128 ? 0 : (o[i] > 127 ? 255 : o[i] + 128));
      *reinterpret_cast<uint2*>(planes + plane + (by * 8 + y) * (bw * 8) + bx * 8) =
          *reinterpret_cast<const uint2*>(row);
    }
    return;
  }
}

__device__ __forceinline__ int clampi(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }

// libjpeg-turbo's upsampled chroma sample at image pixel (y, x) of a plane (row stride `stride`) with cw x ch real
// samples: h2v1 / h2v2 fancy upsampling with replicated edges, plain replication when cw <= 2
__device__ __forceinline__ int chroma(const uint8_t* __restrict__ p, long long stride, int cw, int ch, int hmax,
                                      int vmax, int y, int x) {
  if (hmax == 1) return p[(long long)y * stride + x];
  if (cw <= 2) return p[(long long)(y / vmax) * stride + (x >> 1)];
  const int i = x >> 1, j = (x & 1) ? clampi(i + 1, 0, cw - 1) : clampi(i - 1, 0, cw - 1);
  if (vmax == 1) {
    const uint8_t* row = p + (long long)y * stride;
    return (x & 1) ? (3 * row[i] + row[j] + 2) >> 2 : (3 * row[i] + row[j] + 1) >> 2;
  }
  const int r = y >> 1, far = clampi((y & 1) ? r + 1 : r - 1, 0, ch - 1);
  const uint8_t* n0 = p + (long long)r * stride;
  const uint8_t* n1 = p + (long long)far * stride;
  const int ci = 3 * n0[i] + n1[i], cj = 3 * n0[j] + n1[j];
  return (x & 1) ? (3 * ci + cj + 7) >> 4 : (3 * ci + cj + 8) >> 4;
}

__device__ __forceinline__ uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

__global__ void jpeg_color_kernel(const uint8_t* __restrict__ payload, const long long* __restrict__ desc, int B,
                                  long long n_pixels, const uint8_t* __restrict__ planes, uint8_t* __restrict__ out) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_pixels) return;
  const int b = find_image(desc, B, D_PIX, t);
  const long long* d = desc + (long long)b * kDescWords;
  const long long local = t - d[D_PIX], rw = d[D_RW];
  uint8_t* o = out + d[D_OUT] + 3 * local;
  if (d[D_KIND] == kKindHost) {
    const uint8_t* s = payload + d[D_SRC] + 3 * local;
    o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
    return;
  }
  const long long ry = local / rw;
  const int y = (int)(d[D_Y0] + ry), x = (int)(d[D_X0] + local - ry * rw);
  const int hmax = (int)d[D_HMAX], vmax = (int)d[D_VMAX];
  const long long stride0 = d[D_MCUX] * hmax * 8;
  const uint8_t* p0 = planes + d[D_PLANE];
  const int Y = p0[(long long)y * stride0 + x];
  if (d[D_KIND] == kKindGray) {
    o[0] = o[1] = o[2] = (uint8_t)Y;
    return;
  }
  const long long stride = d[D_MCUX] * 8, psize = stride * d[D_MCUY] * 8;
  const uint8_t* p1 = p0 + stride0 * d[D_MCUY] * vmax * 8;
  const int H = (int)d[D_H], W = (int)d[D_W];
  const int cw = (W + hmax - 1) / hmax, ch = (H + vmax - 1) / vmax;
  const int cb = chroma(p1, stride, cw, ch, hmax, vmax, y, x) - 128;
  const int cr = chroma(p1 + psize, stride, cw, ch, hmax, vmax, y, x) - 128;
  // jdcolor.c ycc_rgb_convert: FIX(1.40200), FIX(1.77200), -FIX(0.71414), -FIX(0.34414) at 16 fractional bits
  o[0] = clamp255(Y + ((91881 * cr + 32768) >> 16));
  o[1] = clamp255(Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16));
  o[2] = clamp255(Y + ((116130 * cb + 32768) >> 16));
}

}  // namespace

extern "C" int b200_jpeg_decode(const uint8_t* payload, long long payload_bytes, const long long* desc, int B,
                                const long long* intervals, int n_intervals, int16_t* coef, long long coef_blocks,
                                uint8_t* planes, long long plane_bytes, long long pixels, uint8_t* out,
                                long long out_bytes, int* status, b200_stream_t stream) {
  B200_REQUIRE(payload && desc && status && out && payload_bytes > 0 && B > 0 && n_intervals >= 0 && coef_blocks >= 0 &&
                   plane_bytes >= 0 && pixels > 0 && out_bytes >= 3 * pixels,
               B200_ERR_INVALID, "jpeg_decode: bad argument");
  B200_REQUIRE((coef_blocks == 0 || (coef && planes && intervals)) && plane_bytes >= 64 * coef_blocks,
               B200_ERR_INVALID, "jpeg_decode: workspaces missing or too small");
  B200_REQUIRE(((uintptr_t)payload & 15) == 0 && ((uintptr_t)coef & 15) == 0 && ((uintptr_t)planes & 7) == 0,
               B200_ERR_INVALID, "jpeg_decode: payload and coef must be 16-byte aligned, planes 8-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int) * B, s);
  B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "jpeg_decode: status reset: %s", cudaGetErrorString(e));
  if (n_intervals > 0) {
    // one decoding thread per warp while there are warps enough to fill the GPU: lanes of one warp that decode
    // different streams would serialise on every diverging branch
    const int per_block = n_intervals > 32 * b200::sm_count() ? 32 : 1;
    b200::launch(jpeg_huffman_kernel, (n_intervals + per_block - 1) / per_block, 32, 0, s, payload, desc, intervals,
                 n_intervals, per_block, coef, status);
    B200_CHECK_LAUNCH("jpeg_huffman_kernel");
  }
  if (coef_blocks > 0) {
    b200::launch(jpeg_idct_kernel, (unsigned)((coef_blocks + 127) / 128), 128, 0, s, payload, desc, B, coef_blocks, coef,
                 planes);
    B200_CHECK_LAUNCH("jpeg_idct_kernel");
  }
  b200::launch(jpeg_color_kernel, (unsigned)((pixels + 255) / 256), 256, 0, s, payload, desc, B, pixels, planes, out);
  B200_CHECK_LAUNCH("jpeg_color_kernel");
  return B200_OK;
}
