// Depthwise RxS convolution (groups == C == K) for NHWC bf16: CUDA-core, HBM-bound, 128-bit vectorised
// fprop / dgrad / wgrad.  Arithmetic intensity is ~R*S FLOP per element, far below the tensor-core
// ridge, so these are written as bandwidth kernels (no tensor cores, no im2col).
// Replaces the depthwise nn.Conv2d of the reference's inverted residual (models/mobilenet_v2.py:57-58)
// and its autograd backward.  Weight layout: [R*S][C] (bf16 for fprop/dgrad, fp32 gradient).
#include "common.cuh"
#include "host.h"

namespace b200 {

__device__ __forceinline__ void dld8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void dst8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

__global__ void __launch_bounds__(256) dw_fprop_kernel(const __nv_bfloat16* __restrict__ x,
                                                       const __nv_bfloat16* __restrict__ w, b200_conv_desc d,
                                                       __nv_bfloat16* __restrict__ y) {
  const int cv = d.C >> 3;
  const long long total = (long long)d.N * d.P * d.Q * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % cv);
    long long pix = idx / cv;
    const int q = (int)(pix % d.Q); pix /= d.Q;
    const int p = (int)(pix % d.P);
    const int n = (int)(pix / d.P);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int r = 0; r < d.R; ++r) {
      const int h = p * d.stride - d.pad_h + r;
      if (h < 0 || h >= d.H) continue;
      for (int s = 0; s < d.S; ++s) {
        const int ww = q * d.stride - d.pad_w + s;
        if (ww < 0 || ww >= d.W) continue;
        float xf[8], wf[8];
        dld8(x + (((long long)n * d.H + h) * d.W + ww) * d.C + v * 8, xf);
        dld8(w + (long long)(r * d.S + s) * d.C + v * 8, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(xf[i], wf[i], acc[i]);
      }
    }
    dst8(y + idx * 8, acc);
  }
}

__global__ void __launch_bounds__(256) dw_dgrad_kernel(const __nv_bfloat16* __restrict__ dy,
                                                       const __nv_bfloat16* __restrict__ w, b200_conv_desc d,
                                                       __nv_bfloat16* __restrict__ dx) {
  const int cv = d.C >> 3;
  const long long total = (long long)d.N * d.H * d.W * cv;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % cv);
    long long pix = idx / cv;
    const int ww = (int)(pix % d.W); pix /= d.W;
    const int h = (int)(pix % d.H);
    const int n = (int)(pix / d.H);
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int r = 0; r < d.R; ++r) {
      const int th = h + d.pad_h - r;
      if (th < 0 || th % d.stride != 0) continue;
      const int p = th / d.stride;
      if (p >= d.P) continue;
      for (int s = 0; s < d.S; ++s) {
        const int tw = ww + d.pad_w - s;
        if (tw < 0 || tw % d.stride != 0) continue;
        const int q = tw / d.stride;
        if (q >= d.Q) continue;
        float gf[8], wf[8];
        dld8(dy + (((long long)n * d.P + p) * d.Q + q) * d.C + v * 8, gf);
        dld8(w + (long long)(r * d.S + s) * d.C + v * 8, wf);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(gf[i], wf[i], acc[i]);
      }
    }
    dst8(dx + idx * 8, acc);
  }
}

constexpr int kDwThreads = 256;
constexpr int kDwMaxBlocks = 592;
constexpr int kDwMaxTaps = 9;

// partial[block][tap][C]
__global__ void __launch_bounds__(kDwThreads) dw_wgrad_partial_kernel(const __nv_bfloat16* __restrict__ x,
                                                                      const __nv_bfloat16* __restrict__ dy,
                                                                      b200_conv_desc d, int cv, int rows_per_iter,
                                                                      float* __restrict__ partial) {
  __shared__ float red[kDwThreads][9];
  const int t = threadIdx.x;
  const bool active = t < rows_per_iter * cv;
  const int r0 = t / cv, v = t - r0 * cv;
  const long long M = (long long)d.N * d.P * d.Q;
  const long long rows_per_block = (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  const int ntaps = d.R * d.S;
  float acc[kDwMaxTaps][8];
#pragma unroll
  for (int a = 0; a < kDwMaxTaps; ++a)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[a][i] = 0.f;
  if (active) {
    for (long long row = row_begin + r0; row < row_end; row += rows_per_iter) {
      const int q = (int)(row % d.Q);
      const int p = (int)((row / d.Q) % d.P);
      const int n = (int)(row / ((long long)d.Q * d.P));
      float gf[8];
      dld8(dy + row * d.C + v * 8, gf);
#pragma unroll
      for (int a = 0; a < kDwMaxTaps; ++a) {
        if (a >= ntaps) break;
        const int r = a / d.S, s = a - r * d.S;
        const int h = p * d.stride - d.pad_h + r, ww = q * d.stride - d.pad_w + s;
        if (h < 0 || h >= d.H || ww < 0 || ww >= d.W) continue;
        float xf[8];
        dld8(x + (((long long)n * d.H + h) * d.W + ww) * d.C + v * 8, xf);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[a][i] = fmaf(gf[i], xf[i], acc[a][i]);
      }
    }
  }
  float* out = partial + (long long)blockIdx.x * ntaps * d.C;
#pragma unroll
  for (int a = 0; a < kDwMaxTaps; ++a) {
    if (a >= ntaps) break;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) red[t][i] = acc[a][i];
    __syncthreads();
    for (int c = t; c < d.C; c += kDwThreads) {
      const int vv = c >> 3, e = c & 7;
      float s = 0.f;
      for (int r = 0; r < rows_per_iter; ++r) s += red[r * cv + vv][e];
      out[(long long)a * d.C + c] = s;
    }
  }
}

// dw[i] += sum over blocks of partial[b][i] (fixed order: deterministic).  A block of 256 threads owns 4 outputs x 64
// interleaved block groups -- every load is independent; the first version (one thread per output walking all the
// blocks) was a chain of L2 round trips, 0.3 ms per layer.
__global__ void __launch_bounds__(256) dw_wgrad_final_kernel(const float* __restrict__ partial, int nblocks, int n,
                                                             float* __restrict__ dw) {
  __shared__ double red[64][5];
  const int lane_o = threadIdx.x & 3, grp = threadIdx.x >> 2;
  const int o = blockIdx.x * 4 + lane_o;
  double acc = 0.0;
  if (o < n) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int b = grp;
    for (; b + 192 < nblocks; b += 256) {
      a0 += __ldcg(partial + (size_t)b * n + o);
      a1 += __ldcg(partial + (size_t)(b + 64) * n + o);
      a2 += __ldcg(partial + (size_t)(b + 128) * n + o);
      a3 += __ldcg(partial + (size_t)(b + 192) * n + o);
    }
    for (; b < nblocks; b += 64) a0 += __ldcg(partial + (size_t)b * n + o);
    acc = (double)a0 + (double)a1 + (double)a2 + (double)a3;
  }
  red[grp][lane_o] = acc;
  __syncthreads();
  if (grp == 0 && o < n) {
    double tot = 0.0;
#pragma unroll 8
    for (int g = 0; g < 64; ++g) tot += red[g][lane_o];
    dw[o] += (float)tot;
  }
}

// ================================================================================================
// 3x3 / pad 1 specialisations (stride 1 and 2: every depthwise layer of MobileNet-v1 / -v2).
// The generic kernels above issue 18 16-byte loads per output vector (9 inputs + 9 weights) and a few 64-bit
// divisions -- like the BN kernels they are bound by load requests in flight, not by bytes (measured ~25 % of the HBM
// roofline over the MobileNet-v2 step).  Here a thread owns one (image, output column, 8-channel vector) and SLIDES
// DOWN the rows: the nine weight vectors live in registers (fp32), the 3x3 input window stays in registers (packed
// bf16) and every step loads only the new rows -- 3 loads per output at stride 1, 6 at stride 2, 4 / 7 in wgrad.
// Neighbouring threads are neighbouring channel vectors / columns (coalesced rows); the column overlap between
// threads is served by L1 (ld.global.nc).
__device__ __forceinline__ uint4 dw_ldg(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void dw_fma8(const uint4& xv, const float (&w)[8], float (&acc)[8]) {
  const float2 a = unpack_bf16x2(xv.x), b = unpack_bf16x2(xv.y), c = unpack_bf16x2(xv.z), d = unpack_bf16x2(xv.w);
  acc[0] = fmaf(a.x, w[0], acc[0]); acc[1] = fmaf(a.y, w[1], acc[1]);
  acc[2] = fmaf(b.x, w[2], acc[2]); acc[3] = fmaf(b.y, w[3], acc[3]);
  acc[4] = fmaf(c.x, w[4], acc[4]); acc[5] = fmaf(c.y, w[5], acc[5]);
  acc[6] = fmaf(d.x, w[6], acc[6]); acc[7] = fmaf(d.y, w[7], acc[7]);
}

struct Dw3 {
  int N, H, W, C, P, Q;   // input map H x W, output map P x Q
  int TP;                 // output rows per work item (a column is cut into ceil(P / TP) chunks)
};

// fprop (flip = 0) and the stride-1 dgrad (flip = 1: dx = conv(dy, w rotated by 180 degrees), same geometry)
template <int STRIDE>
__global__ void __launch_bounds__(128) dw3x3_fprop_kernel(const __nv_bfloat16* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ w, const Dw3 g, int flip,
                                                          __nv_bfloat16* __restrict__ y) {
  const unsigned cv = (unsigned)g.C >> 3;
  const unsigned chunks = (unsigned)(g.P + g.TP - 1) / (unsigned)g.TP;
  const unsigned total = (unsigned)g.N * chunks * (unsigned)g.Q * cv;
  const unsigned step = gridDim.x * blockDim.x;           // a multiple of cv (host): the channel vector is per thread
  unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const unsigned v = idx % cv;
  float wf[9][8];
#pragma unroll
  for (int t = 0; t < 9; ++t) dld8(w + (size_t)(flip ? 8 - t : t) * g.C + v * 8, wf[t]);
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (; idx < total; idx += step) {
    unsigned t = idx / cv;
    const int q = (int)(t % (unsigned)g.Q); t /= (unsigned)g.Q;
    const int ch = (int)(t % chunks);
    const int n = (int)(t / chunks);
    const int p0 = ch * g.TP, p1 = min(g.P, p0 + g.TP);
    const int c0 = q * STRIDE - 1;                        // input columns c0, c0 + 1, c0 + 2
    const bool okl = c0 >= 0, okr = c0 + 2 < g.W;
    const __nv_bfloat16* xn = x + (size_t)n * g.H * g.W * g.C + v * 8;
    auto load_row = [&](int h, uint4 (&row)[3]) {
      if (h < 0 || h >= g.H) { row[0] = zero; row[1] = zero; row[2] = zero; return; }
      const __nv_bfloat16* r = xn + ((size_t)h * g.W + c0) * g.C;
      row[0] = okl ? dw_ldg(r) : zero;
      row[1] = dw_ldg(r + g.C);
      row[2] = okr ? dw_ldg(r + 2 * g.C) : zero;
    };
    uint4 win[3][3];
    int h = p0 * STRIDE - 1;
    load_row(h, win[0]);
    if (STRIDE == 1) load_row(h + 1, win[1]);
    __nv_bfloat16* yo = y + (((size_t)n * g.P + p0) * g.Q + q) * g.C + v * 8;
    for (int p = p0; p < p1; ++p) {
      if (STRIDE == 1) {
        load_row(h + 2, win[2]);
      } else {
        load_row(h + 1, win[1]);
        load_row(h + 2, win[2]);
      }
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) dw_fma8(win[r][c], wf[r * 3 + c], acc);
      dst8(yo, acc);
      yo += (size_t)g.Q * g.C;
      if (STRIDE == 1) {
#pragma unroll
        for (int c = 0; c < 3; ++c) { win[0][c] = win[1][c]; win[1][c] = win[2][c]; }
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) win[0][c] = win[2][c];
      }
      h += STRIDE;
    }
  }
}

// stride-2 dgrad: dx[h, w] = sum over (r, s) with h = 2p - 1 + r, w = 2q - 1 + s of dy[p, q] * wgt[r, s].
// Even h: r = 1, p = h/2.  Odd h: r = 0 (p = (h+1)/2) and r = 2 (p = (h-1)/2); the same in w.  A thread owns one dx
// column: it keeps dy row j in registers, loads row j + 1 and writes dx rows 2j and 2j + 1.
__global__ void __launch_bounds__(128) dw3x3_dgrad_s2_kernel(const __nv_bfloat16* __restrict__ dy,
                                                             const __nv_bfloat16* __restrict__ w, const Dw3 g,
                                                             __nv_bfloat16* __restrict__ dx) {
  const unsigned cv = (unsigned)g.C >> 3;
  const int J = (g.H + 1) >> 1;                                   // row pairs of dx
  const unsigned chunks = (unsigned)(J + g.TP - 1) / (unsigned)g.TP;
  const unsigned total = (unsigned)g.N * chunks * (unsigned)g.W * cv;
  const unsigned step = gridDim.x * blockDim.x;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += step) {
    const unsigned v = idx % cv;
    unsigned t = idx / cv;
    const int wc = (int)(t % (unsigned)g.W); t /= (unsigned)g.W;
    const int ch = (int)(t % chunks);
    const int n = (int)(t / chunks);
    // column slots: a = (qa, sa), b = (qb, sb)
    const bool odd = wc & 1;
    const int qa = odd ? (wc + 1) >> 1 : wc >> 1, sa = odd ? 0 : 1;
    const int qb = (wc - 1) >> 1, sb = 2;
    const bool oka = qa < g.Q, okb = odd && qb >= 0 && qb < g.Q;
    float wa[3][8], wb[3][8];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      dld8(w + (size_t)(r * 3 + sa) * g.C + v * 8, wa[r]);
      dld8(w + (size_t)(r * 3 + sb) * g.C + v * 8, wb[r]);
    }
    const __nv_bfloat16* gn = dy + (size_t)n * g.P * g.Q * g.C + v * 8;
    auto load_row = [&](int p, uint4& a, uint4& b) {
      a = zero; b = zero;
      if (p < 0 || p >= g.P) return;
      const __nv_bfloat16* r = gn + (size_t)p * g.Q * g.C;
      if (oka) a = dw_ldg(r + (size_t)qa * g.C);
      if (okb) b = dw_ldg(r + (size_t)qb * g.C);
    };
    const int j0 = ch * g.TP, j1 = min(J, j0 + g.TP);
    uint4 ca, cb, na, nb;
    load_row(j0, ca, cb);
    __nv_bfloat16* xo = dx + (((size_t)n * g.H + 2 * j0) * g.W + wc) * g.C + v * 8;
    for (int j = j0; j < j1; ++j) {
      load_row(j + 1, na, nb);
      float e[8], o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { e[i] = 0.f; o[i] = 0.f; }
      dw_fma8(ca, wa[1], e); dw_fma8(cb, wb[1], e);                // dx row 2j    : r = 1, p = j
      dw_fma8(na, wa[0], o); dw_fma8(nb, wb[0], o);                // dx row 2j + 1: r = 0, p = j + 1
      dw_fma8(ca, wa[2], o); dw_fma8(cb, wb[2], o);                //                r = 2, p = j
      dst8(xo, e);
      if (2 * j + 1 < g.H) dst8(xo + (size_t)g.W * g.C, o);
      xo += 2 * (size_t)g.W * g.C;
      ca = na; cb = nb;
    }
  }
}

// wgrad partials: dw[tap][c] += sum over (n, p, q) of dy[n, p, q, c] * x[n, p*stride - 1 + r, q*stride - 1 + s, c].
// A block owns a contiguous range of output columns (n, q); thread (r0, v) walks the columns r0, r0 + rows_per_iter, ...
// of that range top to bottom with the sliding window; 72 fp32 accumulators per thread, folded over the block in shared
// memory at the end -> partial[block][tap][C] (dw_wgrad_final_kernel adds the blocks in a fixed order).
template <int STRIDE>
__global__ void __launch_bounds__(kDwThreads) dw3x3_wgrad_partial_kernel(const __nv_bfloat16* __restrict__ x,
                                                                         const __nv_bfloat16* __restrict__ dy,
                                                                         const Dw3 g, int cv, int rows_per_iter,
                                                                         float* __restrict__ partial) {
  __shared__ float red[kDwThreads][9];
  const int t = threadIdx.x;
  const bool active = t < rows_per_iter * cv;
  const int r0 = t / cv, v = t - r0 * cv;
  const unsigned cols = (unsigned)g.N * (unsigned)g.Q;
  const unsigned cols_per_block = (cols + gridDim.x - 1) / gridDim.x;
  const unsigned col_begin = blockIdx.x * cols_per_block;
  const unsigned col_end = min(cols, col_begin + cols_per_block);
  float acc[9][8];
#pragma unroll
  for (int a = 0; a < 9; ++a)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[a][i] = 0.f;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  if (active) {
    for (unsigned col = col_begin + r0; col < col_end; col += rows_per_iter) {
      const int n = (int)(col / (unsigned)g.Q);
      const int q = (int)(col - (unsigned)n * (unsigned)g.Q);
      const int c0 = q * STRIDE - 1;
      const bool okl = c0 >= 0, okr = c0 + 2 < g.W;
      const __nv_bfloat16* xn = x + (size_t)n * g.H * g.W * g.C + v * 8;
      auto load_row = [&](int h, uint4 (&row)[3]) {
        if (h < 0 || h >= g.H) { row[0] = zero; row[1] = zero; row[2] = zero; return; }
        const __nv_bfloat16* r = xn + ((size_t)h * g.W + c0) * g.C;
        row[0] = okl ? dw_ldg(r) : zero;
        row[1] = dw_ldg(r + g.C);
        row[2] = okr ? dw_ldg(r + 2 * g.C) : zero;
      };
      uint4 win[3][3];
      int h = -1;
      load_row(h, win[0]);
      if (STRIDE == 1) load_row(h + 1, win[1]);
      const __nv_bfloat16* gp = dy + ((size_t)n * g.P * g.Q + q) * g.C + v * 8;
      for (int p = 0; p < g.P; ++p) {
        float gf[8];
        dld8(gp, gf);
        gp += (size_t)g.Q * g.C;
        if (STRIDE == 1) {
          load_row(h + 2, win[2]);
        } else {
          load_row(h + 1, win[1]);
          load_row(h + 2, win[2]);
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int c = 0; c < 3; ++c) dw_fma8(win[r][c], gf, acc[r * 3 + c]);
        if (STRIDE == 1) {
#pragma unroll
          for (int c = 0; c < 3; ++c) { win[0][c] = win[1][c]; win[1][c] = win[2][c]; }
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c) win[0][c] = win[2][c];
        }
        h += STRIDE;
      }
    }
  }
  float* out = partial + (size_t)blockIdx.x * 9 * g.C;
#pragma unroll
  for (int a = 0; a < 9; ++a) {
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) red[t][i] = acc[a][i];
    __syncthreads();
    for (int c = t; c < g.C; c += kDwThreads) {
      const int vv = c >> 3, e = c & 7;
      float sum = 0.f;
      for (int r = 0; r < rows_per_iter; ++r) sum += red[r * cv + vv][e];
      out[(size_t)a * g.C + c] = sum;
    }
  }
}

// the specialised path covers 3x3, pad 1, stride 1 or 2 (all of MobileNet); anything else runs the generic kernels
static inline bool dw3_ok(const b200_conv_desc* d) {
  return d->R == 3 && d->S == 3 && d->pad_h == 1 && d->pad_w == 1 && (d->stride == 1 || d->stride == 2) &&
         d->P == (d->H - 1) / d->stride + 1 && d->Q == (d->W - 1) / d->stride + 1 &&
         (long long)d->N * d->H * d->W * (d->C / 8) < (1LL << 31);
}
static inline Dw3 dw3_geom(const b200_conv_desc* d, int rows) {
  Dw3 g;
  g.N = d->N; g.H = d->H; g.W = d->W; g.C = d->C; g.P = d->P; g.Q = d->Q;
  g.TP = rows < 16 ? rows : 16;       // <= 16 output rows per work item: 2 extra row loads amortised over the chunk
  return g;
}
// grid: enough 128-thread blocks for the work items, a multiple of the channel-vector count (so that a thread keeps
// its channel vector over the grid-stride loop), capped at 16 blocks per SM
static inline int dw3_grid(long long items, int cv) {
  long long b = (items + 127) / 128;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  b = (b + cv - 1) / cv * cv;
  return (int)b;
}

static int dw_check(const b200_conv_desc* d, const char* who) {
  B200_REQUIRE(d && d->C == d->K && d->C % 8 == 0 && d->C <= 2048, B200_ERR_UNSUPPORTED,
               "%s: depthwise needs C == K, C %% 8 == 0, C <= 2048", who);
  B200_REQUIRE(d->R * d->S <= kDwMaxTaps && d->stride >= 1, B200_ERR_UNSUPPORTED, "%s: filter too large", who);
  return B200_OK;
}
static inline int dw_grid(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_dwconv_fprop(const b200_conv_desc* d, const void* x, const void* w, void* y, b200_stream_t stream) {
  int rc = dw_check(d, "dwconv_fprop");
  if (rc) return rc;
  B200_REQUIRE(x && w && y, B200_ERR_INVALID, "dwconv_fprop: null pointer");
  if (dw3_ok(d)) {
    const Dw3 g = dw3_geom(d, d->P);
    const long long items = (long long)d->N * ((d->P + g.TP - 1) / g.TP) * d->Q * (d->C / 8);
    const int grid = dw3_grid(items, d->C / 8);
    if (d->stride == 1)
      b200::launch(dw3x3_fprop_kernel<1>, grid, 128, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x,
                   (const __nv_bfloat16*)w, g, 0, (__nv_bfloat16*)y);
    else
      b200::launch(dw3x3_fprop_kernel<2>, grid, 128, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x,
                   (const __nv_bfloat16*)w, g, 0, (__nv_bfloat16*)y);
    B200_CHECK_LAUNCH("dw3x3_fprop_kernel");
    return B200_OK;
  }
  const long long total = (long long)d->N * d->P * d->Q * (d->C / 8);
  b200::launch(dw_fprop_kernel, dw_grid(total), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w,
                                                                  *d, (__nv_bfloat16*)y);
  B200_CHECK_LAUNCH("dw_fprop_kernel");
  return B200_OK;
}

extern "C" int b200_dwconv_dgrad(const b200_conv_desc* d, const void* dy, const void* w, void* dx,
                                 b200_stream_t stream) {
  int rc = dw_check(d, "dwconv_dgrad");
  if (rc) return rc;
  B200_REQUIRE(dy && w && dx, B200_ERR_INVALID, "dwconv_dgrad: null pointer");
  if (dw3_ok(d)) {
    if (d->stride == 1) {       // same geometry as fprop, filter rotated by 180 degrees
      const Dw3 g = dw3_geom(d, d->H);
      const long long items = (long long)d->N * ((d->H + g.TP - 1) / g.TP) * d->W * (d->C / 8);
      b200::launch(dw3x3_fprop_kernel<1>, dw3_grid(items, d->C / 8), 128, 0, (cudaStream_t)stream,
                   (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, g, 1, (__nv_bfloat16*)dx);
    } else {
      const int J = (d->H + 1) / 2;
      const Dw3 g = dw3_geom(d, J);
      const long long items = (long long)d->N * ((J + g.TP - 1) / g.TP) * d->W * (d->C / 8);
      b200::launch(dw3x3_dgrad_s2_kernel, dw3_grid(items, d->C / 8), 128, 0, (cudaStream_t)stream,
                   (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w, g, (__nv_bfloat16*)dx);
    }
    B200_CHECK_LAUNCH("dw3x3_dgrad_kernel");
    return B200_OK;
  }
  const long long total = (long long)d->N * d->H * d->W * (d->C / 8);
  b200::launch(dw_dgrad_kernel, dw_grid(total), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)w,
                                                                  *d, (__nv_bfloat16*)dx);
  B200_CHECK_LAUNCH("dw_dgrad_kernel");
  return B200_OK;
}

extern "C" int b200_dwconv_wgrad(const b200_conv_desc* d, const void* x, const void* dy, float* dw, float* workspace,
                                 size_t workspace_bytes, b200_stream_t stream) {
  int rc = dw_check(d, "dwconv_wgrad");
  if (rc) return rc;
  B200_REQUIRE(x && dy && dw && workspace, B200_ERR_INVALID, "dwconv_wgrad: null pointer");
  const int cv = d->C / 8;
  const int rows_per_iter = kDwThreads / cv;
  const long long M = (long long)d->N * d->P * d->Q;
  long long blocks = (M + rows_per_iter * 8 - 1) / (rows_per_iter * 8);
  if (blocks > kDwMaxBlocks) blocks = kDwMaxBlocks;
  if (blocks < 1) blocks = 1;
  const int n = d->R * d->S * d->C;
  B200_REQUIRE(workspace_bytes >= (size_t)blocks * n * sizeof(float), B200_ERR_INVALID,
               "dwconv_wgrad: workspace too small (%zu < %zu)", workspace_bytes, (size_t)blocks * n * sizeof(float));
  if (dw3_ok(d)) {
    // one column (n, q) per thread at a time; at least two columns per thread so that the block partials stay few
    const long long cols = (long long)d->N * d->Q;
    long long b3 = (cols + 2 * rows_per_iter - 1) / (2 * rows_per_iter);
    if (b3 < blocks) blocks = b3 < 1 ? 1 : b3;
    const Dw3 g = dw3_geom(d, d->P);
    if (d->stride == 1)
      b200::launch(dw3x3_wgrad_partial_kernel<1>, (int)blocks, kDwThreads, 0, (cudaStream_t)stream,
                   (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, g, cv, rows_per_iter, workspace);
    else
      b200::launch(dw3x3_wgrad_partial_kernel<2>, (int)blocks, kDwThreads, 0, (cudaStream_t)stream,
                   (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, g, cv, rows_per_iter, workspace);
  } else {
    b200::launch(dw_wgrad_partial_kernel, (int)blocks, kDwThreads, 0, (cudaStream_t)stream,
        (const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, *d, cv, rows_per_iter, workspace);
  }
  B200_CHECK_LAUNCH("dw_wgrad_partial_kernel");
  b200::launch(dw_wgrad_final_kernel, (n + 3) / 4, 256, 0, (cudaStream_t)stream, workspace, (int)blocks, n, dw);
  B200_CHECK_LAUNCH("dw_wgrad_final_kernel");
  return B200_OK;
}
