// RandomResizedCrop + RandomHorizontalFlip + ToTensor + Normalize of the ImageNet training transform (the reference's
// inception_preprocess, preprocess.py:71-77) fused into the stem relayout: uint8 regions -> bf16 stem layouts.
//
// The resample is Pillow's ImagingResample with the BILINEAR filter on 8-bit channels, applied to the crop as if the
// crop were the whole image (torchvision crops, then resizes): per axis, coefficients computed in double without
// contraction, normalised by their sum, converted to 22-bit integers; a horizontal pass into a uint8 intermediate, then
// a vertical pass over it, each accumulating in int32 from 2^21 and shifting right by 22 with a clamp to [0, 255].
//
// One block owns kRrcRows output rows of one copy and one thread owns one resampled column.  Each thread runs the
// horizontal pass of its column over the intermediate rows the band needs and feeds every finished intermediate value
// straight into its per-row vertical accumulators (registers), so the intermediate never leaves the thread.  Horizontal
// coefficients sit in a per-thread shared-memory slab of kRrcTaps taps (rebuilt per row when a column has more taps, so
// the scale is unbounded); vertical coefficients are computed per chunk of kRrcYChunk intermediate rows.  The grid
// depends only on (B*D, OH) and there is no workspace: a captured CUDA graph replays with new tables and regions.
//
// The same arithmetic (the rrc_* helpers below) serves the ImageNet evaluation transform (Resize + CenterCrop,
// input_prep_scale_crop_kernel: the crop window of the whole image's resize, on the same block shape) and the small
// fixed-size resample of the CIFAR Mix&Match transform, input_prep_aug_resize_kernel at the end of this file.
#include "common.cuh"
#include "host.h"

namespace b200 {

constexpr int kRrcRows = 8;      // output rows per block (even, so that space-to-depth row pairs stay in one block)
constexpr int kRrcTaps = 16;     // horizontal taps per coefficient slab
constexpr int kRrcYChunk = 32;   // intermediate rows per vertical-coefficient chunk
constexpr int kRrcMaxOW = 512;   // one thread per output column

struct RrcAxis { double scale, support, ss; int in; };

__device__ __forceinline__ RrcAxis rrc_axis(int in, int out) {
  RrcAxis a;
  a.in = in;
  a.scale = __ddiv_rn((double)in, (double)out);
  const double fs = a.scale < 1.0 ? 1.0 : a.scale;
  a.support = fs;                       // the bilinear filter's support (1.0) times the filter scale
  a.ss = __ddiv_rn(1.0, fs);
  return a;
}

// first source index and tap count of output index xx; center = (xx + 0.5) * scale
__device__ __forceinline__ void rrc_bounds(const RrcAxis& a, int xx, double& center, int& xmin, int& cnt) {
  center = __dmul_rn(__dadd_rn((double)xx, 0.5), a.scale);
  int lo = __double2int_rz(__dadd_rn(__dsub_rn(center, a.support), 0.5));
  int hi = __double2int_rz(__dadd_rn(__dadd_rn(center, a.support), 0.5));
  if (lo < 0) lo = 0;
  if (hi > a.in) hi = a.in;
  xmin = lo;
  cnt = hi - lo;
}

// un-normalised weight of source index x: tri((x - center + 0.5) * ss)
__device__ __forceinline__ double rrc_tri(const RrcAxis& a, double center, int x) {
  double t = __dmul_rn(__dadd_rn(__dsub_rn((double)x, center), 0.5), a.ss);
  if (t < 0.0) t = -t;
  return t < 1.0 ? __dsub_rn(1.0, t) : 0.0;
}

__device__ __forceinline__ double rrc_sum(const RrcAxis& a, double center, int xmin, int cnt) {
  double ww = 0.0;
  for (int x = 0; x < cnt; ++x) ww = __dadd_rn(ww, rrc_tri(a, center, xmin + x));
  return ww;
}

__device__ __forceinline__ int rrc_coef(double w, double ww) {
  const double k = ww != 0.0 ? __ddiv_rn(w, ww) : w;
  return __double2int_rz(__dadd_rn(0.5, __dmul_rn(k, 4194304.0)));     // (int)(0.5 + k * 2^22)
}

__device__ __forceinline__ int rrc_clip8(int acc) {
  const int v = acc >> 22;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

struct RrcRow { double center, ww; int ymin, cnt; };

__global__ void __launch_bounds__(kRrcMaxOW) input_prep_rrc_kernel(
    const uint8_t* __restrict__ regions, long long region_bytes, const long long* __restrict__ index,
    const int* __restrict__ draws, int D, int C, int OH, int OW, int Cpad, int mode, const float* __restrict__ lut,
    __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char rrc_smem[];
  int* ktab = reinterpret_cast<int*>(rrc_smem);                                  // [kRrcTaps][blockDim.x]
  uint8_t* tile = rrc_smem + (size_t)kRrcTaps * blockDim.x * sizeof(int);        // [kRrcRows][OW][C], output columns
  __shared__ RrcRow rows[kRrcRows];
  __shared__ int vtab[kRrcRows * kRrcYChunk];

  const int n = blockIdx.y;                     // output row n: copy n % D of image n / D
  const int o0 = blockIdx.x * kRrcRows;
  const int tb = min(kRrcRows, OH - o0);
  const int xx = threadIdx.x;
  const int nt = blockDim.x;

  // the image's region and the copy's crop box, clamped: any table values read inside the region and the buffer
  const long long* ix = index + (long long)(n / D) * 3;
  const int* dr = draws + (long long)n * 5;
  const long long off = min(max(__ldg(ix + 0), 0LL), region_bytes - 1);
  const int rh = (int)min(max(__ldg(ix + 1), 1LL), 65535LL), rw = (int)min(max(__ldg(ix + 2), 1LL), 65535LL);
  const int cy = min(max(__ldg(dr + 0), 0), rh - 1), cx = min(max(__ldg(dr + 1), 0), rw - 1);
  const int ch = min(max(__ldg(dr + 2), 1), rh - cy), cw = min(max(__ldg(dr + 3), 1), rw - cx);
  const bool flip = __ldg(dr + 4) != 0;

  const RrcAxis ay = rrc_axis(ch, OH), ax = rrc_axis(cw, OW);
  if (xx < tb) {
    RrcRow r;
    rrc_bounds(ay, o0 + xx, r.center, r.ymin, r.cnt);
    r.ww = rrc_sum(ay, r.center, r.ymin, r.cnt);
    rows[xx] = r;
  }
  double xc = 0.0, xww = 0.0;
  int xmin = 0, xcnt = 0;
  if (xx < OW) {
    rrc_bounds(ax, xx, xc, xmin, xcnt);
    xww = rrc_sum(ax, xc, xmin, xcnt);
  }
  __syncthreads();
  int ybeg = rows[0].ymin, yend = rows[0].ymin + rows[0].cnt;
  for (int r = 1; r < tb; ++r) {
    ybeg = min(ybeg, rows[r].ymin);
    yend = max(yend, rows[r].ymin + rows[r].cnt);
  }

  int acc[kRrcRows][4];
#pragma unroll
  for (int r = 0; r < kRrcRows; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 1 << 21;
  int built = -1;                               // first tap of the slab this thread holds

  for (int y0 = ybeg; y0 < yend; y0 += kRrcYChunk) {
    __syncthreads();                            // the previous chunk's vertical coefficients are consumed
    for (int e = threadIdx.x; e < kRrcRows * kRrcYChunk; e += nt) {
      const int r = e / kRrcYChunk, t = y0 + e % kRrcYChunk;
      int k = 0;
      if (r < tb && t >= rows[r].ymin && t < rows[r].ymin + rows[r].cnt)
        k = rrc_coef(rrc_tri(ay, rows[r].center, t), rows[r].ww);
      vtab[e] = k;
    }
    __syncthreads();
    if (xx >= OW) continue;
    const int y1 = min(y0 + kRrcYChunk, yend);
    for (int y = y0; y < y1; ++y) {
      const long long row = off + ((long long)(cy + y) * rw + cx + xmin) * C;
      int h[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
      for (int t0 = 0; t0 < xcnt; t0 += kRrcTaps) {
        const int te = min(kRrcTaps, xcnt - t0);
        if (t0 != built) {
          for (int t = 0; t < te; ++t) ktab[t * nt + xx] = rrc_coef(rrc_tri(ax, xc, xmin + t0 + t), xww);
          built = t0;
        }
        for (int t = 0; t < te; ++t) {
          const int k = ktab[t * nt + xx];
          const long long p = row + (long long)(t0 + t) * C;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < C) h[c] += (int)__ldg(regions + min(p + c, region_bytes - 1)) * k;
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) h[c] = rrc_clip8(h[c]);
#pragma unroll
      for (int r = 0; r < kRrcRows; ++r) {
        const int k = vtab[r * kRrcYChunk + (y - y0)];
        if (k != 0) {
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[r][c] += h[c] * k;
        }
      }
    }
  }

  // flip mirrors the resampled column; the tile holds the band's bytes in output-column order
  if (xx < OW) {
    const int j = flip ? OW - 1 - xx : xx;
#pragma unroll
    for (int r = 0; r < kRrcRows; ++r)
      if (r < tb)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < C) tile[((size_t)r * OW + j) * C + c] = (uint8_t)rrc_clip8(acc[r][c]);
  }
  __syncthreads();

  // mode 0: [N][OH][OW][Cpad];  mode 2: [N][OH/2+3][OW/2+3][Cpad], data at (+2, +2), channel (dy*2+dx)*C + c.
  // The first band also writes the top border rows, the last band the bottom one.
  const bool s2d = mode == 2;
  const int PH = s2d ? OH / 2 + 3 : OH, PW = s2d ? OW / 2 + 3 : OW, brd = s2d ? 2 : 0;
  const int r_lo = s2d ? (o0 == 0 ? 0 : o0 / 2 + brd) : o0;
  const int r_hi = s2d ? (o0 + tb == OH ? PH : (o0 + tb) / 2 + brd) : o0 + tb;
  const int total = (r_hi - r_lo) * PW;
  for (int p = threadIdx.x; p < total; p += nt) {
    const int pr = r_lo + p / PW, pc = p % PW;
    const int i = pr - brd, jj = pc - brd;
    const bool inside = !s2d || (i >= 0 && i < OH / 2 && jj >= 0 && jj < OW / 2);
    __nv_bfloat16* o = out + (((long long)n * PH + pr) * PW + pc) * Cpad;
    for (int c0 = 0; c0 < Cpad; c0 += 8) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int chn = c0 + e;
        const int sub = s2d ? chn / C : (chn < C ? 0 : 4), c = s2d ? chn - sub * C : chn;
        float v = 0.f;
        if (sub < 4 && inside) {
          const int ty = s2d ? 2 * i + (sub >> 1) : i, tx = s2d ? 2 * jj + (sub & 1) : jj;
          v = __ldg(lut + c * 256 + tile[((size_t)(ty - o0) * OW + tx) * C + c]);
        }
        f[e] = v;
      }
      uint4 u;
      u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
      u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
      *reinterpret_cast<uint4*>(o + c0) = u;
    }
  }
}

// ---- the ImageNet evaluation transform (the reference's scale_crop, preprocess.py:20-41, one crop): Resize(scale)
// -> CenterCrop(size) -> ToTensor -> Normalize ------------------------------------------------------------------------
// In Pillow's resample, output index xx of an in -> out resize depends on xx, in and out only.  So the centre crop of
// the resized image is the full-image axis rrc_axis(W, RW) evaluated at output indices left .. left + OW - 1, and
// likewise for rows: the resized image is never formed.  (Resizing the crop box instead, as the RRC kernel does, would
// differ in the last bits.)  Each image ships only its support region, the source pixels the window's taps touch; pixel
// (y, x) of the image is read at (y - y0, x - x0) of the region, clamped to the region and the buffer.  Output pixels
// outside the resized image -- a crop larger than the image, which CenterCrop pads -- take uint8 0.  Block shape,
// coefficient slab and vertical chunks are those of input_prep_rrc_kernel; one copy per image.
__global__ void __launch_bounds__(kRrcMaxOW) input_prep_scale_crop_kernel(
    const uint8_t* __restrict__ regions, long long region_bytes, const long long* __restrict__ index,
    const int* __restrict__ geom, int C, int OH, int OW, int Cpad, int mode, const float* __restrict__ lut,
    __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char sc_smem[];
  int* ktab = reinterpret_cast<int*>(sc_smem);                                   // [kRrcTaps][blockDim.x]
  uint8_t* tile = sc_smem + (size_t)kRrcTaps * blockDim.x * sizeof(int);         // [kRrcRows][OW][C]
  __shared__ RrcRow rows[kRrcRows];
  __shared__ int vtab[kRrcRows * kRrcYChunk];

  const int n = blockIdx.y;                     // image n
  const int o0 = blockIdx.x * kRrcRows;
  const int tb = min(kRrcRows, OH - o0);
  const int xx = threadIdx.x;
  const int nt = blockDim.x;

  // geom = {y0, x0, H, W, RH, RW, top, left}; sizes clamped like the RRC region, so any table values are bounded work
  const long long* ix = index + (long long)n * 3;
  const int* gm = geom + (long long)n * 8;
  const long long off = min(max(__ldg(ix + 0), 0LL), region_bytes - 1);
  const long long rh = min(max(__ldg(ix + 1), 1LL), 65535LL), rw = min(max(__ldg(ix + 2), 1LL), 65535LL);
  const long long ry0 = __ldg(gm + 0), rx0 = __ldg(gm + 1);
  const int H = min(max(__ldg(gm + 2), 1), 65535), W = min(max(__ldg(gm + 3), 1), 65535);
  const int RH = min(max(__ldg(gm + 4), 1), 65535), RW = min(max(__ldg(gm + 5), 1), 65535);
  const long long top = __ldg(gm + 6), left = __ldg(gm + 7);

  const RrcAxis ay = rrc_axis(H, RH), ax = rrc_axis(W, RW);
  if (xx < tb) {
    RrcRow r = {0.0, 0.0, 0, 0};                // a padded row: no taps
    const long long yy = top + o0 + xx;
    if (yy >= 0 && yy < RH) {
      rrc_bounds(ay, (int)yy, r.center, r.ymin, r.cnt);
      r.ww = rrc_sum(ay, r.center, r.ymin, r.cnt);
    }
    rows[xx] = r;
  }
  double xc = 0.0, xww = 0.0;
  int xmin = 0, xcnt = 0;                       // a padded column: no taps
  const long long xs = left + xx;
  if (xx < OW && xs >= 0 && xs < RW) {
    rrc_bounds(ax, (int)xs, xc, xmin, xcnt);
    xww = rrc_sum(ax, xc, xmin, xcnt);
  }
  __syncthreads();
  int ybeg = 0x7fffffff, yend = 0;
  for (int r = 0; r < tb; ++r)
    if (rows[r].cnt > 0) {
      ybeg = min(ybeg, rows[r].ymin);
      yend = max(yend, rows[r].ymin + rows[r].cnt);
    }

  int acc[kRrcRows][4];
#pragma unroll
  for (int r = 0; r < kRrcRows; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[r][c] = 1 << 21;
  int built = -1;                               // first tap of the slab this thread holds

  for (int yc = ybeg; yc < yend; yc += kRrcYChunk) {
    __syncthreads();                            // the previous chunk's vertical coefficients are consumed
    for (int e = threadIdx.x; e < kRrcRows * kRrcYChunk; e += nt) {
      const int r = e / kRrcYChunk, t = yc + e % kRrcYChunk;
      int k = 0;
      if (r < tb && t >= rows[r].ymin && t < rows[r].ymin + rows[r].cnt)
        k = rrc_coef(rrc_tri(ay, rows[r].center, t), rows[r].ww);
      vtab[e] = k;
    }
    __syncthreads();
    if (xx >= OW) continue;
    const int y1 = min(yc + kRrcYChunk, yend);
    for (int y = yc; y < y1; ++y) {
      const long long row = off + min(max(y - ry0, 0LL), rh - 1) * rw * C;
      int h[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
      for (int t0 = 0; t0 < xcnt; t0 += kRrcTaps) {
        const int te = min(kRrcTaps, xcnt - t0);
        if (t0 != built) {
          for (int t = 0; t < te; ++t) ktab[t * nt + xx] = rrc_coef(rrc_tri(ax, xc, xmin + t0 + t), xww);
          built = t0;
        }
        for (int t = 0; t < te; ++t) {
          const int k = ktab[t * nt + xx];
          const long long p = row + min(max(xmin + t0 + t - rx0, 0LL), rw - 1) * C;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < C) h[c] += (int)__ldg(regions + min(p + c, region_bytes - 1)) * k;
        }
      }
#pragma unroll
      for (int c = 0; c < 4; ++c) h[c] = rrc_clip8(h[c]);
#pragma unroll
      for (int r = 0; r < kRrcRows; ++r) {
        const int k = vtab[r * kRrcYChunk + (y - yc)];
        if (k != 0) {
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[r][c] += h[c] * k;
        }
      }
    }
  }

  // a row or column without taps keeps acc = 2^21, which rrc_clip8 maps to 0: CenterCrop's fill
  if (xx < OW) {
#pragma unroll
    for (int r = 0; r < kRrcRows; ++r)
      if (r < tb)
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < C) tile[((size_t)r * OW + xx) * C + c] = (uint8_t)rrc_clip8(acc[r][c]);
  }
  __syncthreads();

  // the store of input_prep_rrc_kernel, restated so that kernel's code stays as it is
  const bool s2d = mode == 2;
  const int PH = s2d ? OH / 2 + 3 : OH, PW = s2d ? OW / 2 + 3 : OW, brd = s2d ? 2 : 0;
  const int r_lo = s2d ? (o0 == 0 ? 0 : o0 / 2 + brd) : o0;
  const int r_hi = s2d ? (o0 + tb == OH ? PH : (o0 + tb) / 2 + brd) : o0 + tb;
  const int total = (r_hi - r_lo) * PW;
  for (int p = threadIdx.x; p < total; p += nt) {
    const int pr = r_lo + p / PW, pc = p % PW;
    const int i = pr - brd, jj = pc - brd;
    const bool inside = !s2d || (i >= 0 && i < OH / 2 && jj >= 0 && jj < OW / 2);
    __nv_bfloat16* o = out + (((long long)n * PH + pr) * PW + pc) * Cpad;
    for (int c0 = 0; c0 < Cpad; c0 += 8) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int chn = c0 + e;
        const int sub = s2d ? chn / C : (chn < C ? 0 : 4), c = s2d ? chn - sub * C : chn;
        float v = 0.f;
        if (sub < 4 && inside) {
          const int ty = s2d ? 2 * i + (sub >> 1) : i, tx = s2d ? 2 * jj + (sub & 1) : jj;
          v = __ldg(lut + c * 256 + tile[((size_t)(ty - o0) * OW + tx) * C + c]);
        }
        f[e] = v;
      }
      uint4 u;
      u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
      u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
      *reinterpret_cast<uint4*>(o + c0) = u;
    }
  }
}

// ---- the CIFAR Mix&Match transform (preprocess.py:44-54 with input_size != scale_size): RandomCrop(padding) ->
// Resize -> RandomHorizontalFlip -> ToTensor -> Normalize [-> Cutout], D copies per image ---------------------------
// Every copy resamples the same H x W window size to OH x OW, so the two coefficient tables depend on the launch only:
// one block owns one copy, builds both tables once in shared memory, stages the zero-padded crop window as uint8, runs
// the horizontal pass into a shared uint8 [H][OW][C] and lets each thread finish one output pixel (vertical pass, flip,
// LUT, Cutout, store).  Nothing passes through global memory between the passes, there is no workspace and the grid
// depends only on N*D: a captured CUDA graph replays with new images and draws.
constexpr int kAugRsThreads = 256;
constexpr int kAugRsMaxIn = 64;     // source side: the window and the intermediate stay in shared memory
constexpr int kAugRsMaxOut = 128;

// first tap, tap count and 22-bit coefficients of output index i of an in -> out resample; taps bounds the count
__device__ __forceinline__ void rrc_table(const RrcAxis& a, int i, int taps, int* first, int* count, int* coef) {
  double center;
  int lo, cnt;
  rrc_bounds(a, i, center, lo, cnt);
  cnt = min(cnt, taps);
  const double ww = rrc_sum(a, center, lo, cnt);
  first[i] = lo;
  count[i] = cnt;
  for (int t = 0; t < cnt; ++t) coef[i * taps + t] = rrc_coef(rrc_tri(a, center, lo + t), ww);
}

__global__ void __launch_bounds__(kAugRsThreads) input_prep_aug_resize_kernel(
    const uint8_t* __restrict__ x, int D, int C, int H, int W, int OH, int OW, int Cpad, int pad, int tx, int ty,
    const float* __restrict__ lut, const int16_t* __restrict__ params, int holes, __nv_bfloat16* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char aug_rs_smem[];
  int* xfirst = reinterpret_cast<int*>(aug_rs_smem);          // [OW]
  int* xcount = xfirst + OW;                                  // [OW]
  int* yfirst = xcount + OW;                                  // [OH]
  int* ycount = yfirst + OH;                                  // [OH]
  int* kx = ycount + OH;                                      // [OW][tx]
  int* ky = kx + OW * tx;                                     // [OH][ty]
  uint8_t* win = reinterpret_cast<uint8_t*>(ky + OH * ty);    // [H][W][C]   the padded crop window
  uint8_t* mid = win + H * W * C;                             // [H][OW][C]  after the horizontal pass

  const int n = blockIdx.x;                     // output row n: copy n % D of image n / D
  const int16_t* pr = params + (long long)n * (3 + 4 * holes);
  const int oy = __ldg(pr + 0) - pad, ox = __ldg(pr + 1) - pad;
  const bool flip = __ldg(pr + 2) != 0;

  const RrcAxis ax = rrc_axis(W, OW), ay = rrc_axis(H, OH);
  for (int i = threadIdx.x; i < OW + OH; i += kAugRsThreads) {
    if (i < OW) rrc_table(ax, i, tx, xfirst, xcount, kx);
    else rrc_table(ay, i - OW, ty, yfirst, ycount, ky);
  }
  // any draw values are safe: a source pixel is read only when it lies inside the image, else RandomCrop's fill 0
  const uint8_t* src = x + (long long)(n / D) * H * W * C;
  for (int e = threadIdx.x; e < H * W; e += kAugRsThreads) {
    const int sy = e / W + oy, sx = e % W + ox;
    const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
    for (int c = 0; c < C; ++c) win[e * C + c] = ok ? __ldg(src + (sy * W + sx) * C + c) : (uint8_t)0;
  }
  __syncthreads();

  for (int e = threadIdx.x; e < H * OW; e += kAugRsThreads) {
    const int r = e / OW, xx = e % OW;
    const int* k = kx + xx * tx;
    const uint8_t* p = win + (r * W + xfirst[xx]) * C;
    int h[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
    for (int t = 0; t < xcount[xx]; ++t)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < C) h[c] += (int)p[t * C + c] * k[t];
#pragma unroll
    for (int c = 0; c < 4; ++c)
      if (c < C) mid[e * C + c] = (uint8_t)rrc_clip8(h[c]);
  }
  __syncthreads();

  for (int e = threadIdx.x; e < OH * OW; e += kAugRsThreads) {
    const int yy = e / OW, xx = e % OW;
    const int* k = ky + yy * ty;
    const uint8_t* p = mid + (yfirst[yy] * OW + xx) * C;
    int v[4] = {1 << 21, 1 << 21, 1 << 21, 1 << 21};
    for (int t = 0; t < ycount[yy]; ++t)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (c < C) v[c] += (int)p[t * OW * C + c] * k[t];
    // the flip mirrors the resized picture; the Cutout boxes are in its (output) coordinates
    const int j = flip ? OW - 1 - xx : xx;
    bool cut = false;
    for (int hh = 0; hh < holes; ++hh) {
      const int16_t* b = pr + 3 + 4 * hh;
      cut |= yy >= __ldg(b + 0) && yy < __ldg(b + 1) && j >= __ldg(b + 2) && j < __ldg(b + 3);
    }
    float f[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      f[c] = 0.f;
      if (c < C) {
        f[c] = __ldg(lut + c * 256 + rrc_clip8(v[c]));
        if (cut) f[c] = __fmul_rn(f[c], 0.f);
      }
    }
    __nv_bfloat16* o = out + (((long long)n * OH + yy) * OW + j) * Cpad;
    uint4 u = {pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), 0u, 0u};
    for (int c0 = 0; c0 < Cpad; c0 += 8) {
      *reinterpret_cast<uint4*>(o + c0) = u;
      u = make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

// upper bound of the taps of one output index: hi - lo <= 2 * support + 1, and never more than the source
static int aug_rs_taps(int in, int out) {
  const int support = in > out ? (in + out - 1) / out : 1;
  const int taps = 2 * support + 1;
  return taps < in ? taps : in;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_input_prep_u8_aug_resize(const uint8_t* x_nhwc, int N, int D, int C, int H, int W, int OH, int OW,
                                             int Cpad, int pad, const float* lut, const int16_t* params, int holes,
                                             void* out, b200_stream_t stream) {
  B200_REQUIRE(x_nhwc && out && lut && params && N > 0 && D > 0 && C > 0 && C <= 4 && H > 0 && W > 0 && OH > 0 && OW > 0,
               B200_ERR_INVALID, "input_prep_u8_aug_resize: bad argument (C must be 1..4)");
  B200_REQUIRE(Cpad % 8 == 0 && Cpad >= C, B200_ERR_INVALID,
               "input_prep_u8_aug_resize: Cpad must be a multiple of 8 and >= C");
  B200_REQUIRE(pad >= 0 && holes >= 0 && holes <= 64, B200_ERR_INVALID,
               "input_prep_u8_aug_resize: pad=%d holes=%d out of range", pad, holes);
  B200_REQUIRE(H <= kAugRsMaxIn && W <= kAugRsMaxIn && OH <= kAugRsMaxOut && OW <= kAugRsMaxOut, B200_ERR_UNSUPPORTED,
               "input_prep_u8_aug_resize: %dx%d -> %dx%d above %d px sources or %d px outputs", H, W, OH, OW,
               kAugRsMaxIn, kAugRsMaxOut);
  B200_REQUIRE((long long)N * D <= 0x7fffffffLL, B200_ERR_UNSUPPORTED, "input_prep_u8_aug_resize: N*D too large");
  const int tx = aug_rs_taps(W, OW), ty = aug_rs_taps(H, OH);
  const size_t smem = (size_t)(2 * OW + 2 * OH + OW * tx + OH * ty) * sizeof(int) + (size_t)H * W * C + (size_t)H * OW * C;
  cudaError_t e = cudaFuncSetAttribute(input_prep_aug_resize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "input_prep_u8_aug_resize: smem attribute (%d bytes): %s", (int)smem,
               cudaGetErrorString(e));
  b200::launch(input_prep_aug_resize_kernel, N * D, kAugRsThreads, smem, (cudaStream_t)stream, x_nhwc, D, C, H, W, OH,
               OW, Cpad, pad, tx, ty, lut, params, holes, (__nv_bfloat16*)out);
  B200_CHECK_LAUNCH("input_prep_aug_resize_kernel");
  return B200_OK;
}

extern "C" int b200_input_prep_u8_rrc(const uint8_t* regions, long long region_bytes, const long long* index,
                                      const int* draws, int B, int D, int C, int OH, int OW, int Cpad, int mode,
                                      const float* lut, void* out, b200_stream_t stream) {
  B200_REQUIRE(regions && index && draws && lut && out && region_bytes > 0 && B > 0 && D > 0 && C > 0 && C <= 4 &&
                   OH > 0 && OW > 0,
               B200_ERR_INVALID, "input_prep_u8_rrc: bad argument (C must be 1..4)");
  B200_REQUIRE(OW <= kRrcMaxOW, B200_ERR_UNSUPPORTED, "input_prep_u8_rrc: OW=%d above %d", OW, kRrcMaxOW);
  B200_REQUIRE((long long)B * D <= 65535LL, B200_ERR_UNSUPPORTED, "input_prep_u8_rrc: B*D=%lld above 65535",
               (long long)B * D);
  B200_REQUIRE(Cpad % 8 == 0, B200_ERR_INVALID, "input_prep_u8_rrc: Cpad=%d must be a multiple of 8", Cpad);
  if (mode == 0) {
    B200_REQUIRE(Cpad >= C, B200_ERR_INVALID, "input_prep_u8_rrc: Cpad < C");
  } else if (mode == 2) {
    B200_REQUIRE(OH % 2 == 0 && OW % 2 == 0 && Cpad >= 4 * C, B200_ERR_UNSUPPORTED,
                 "input_prep_u8_rrc: space-to-depth needs even OH, OW and Cpad >= 4C");
  } else {
    B200_REQUIRE(false, B200_ERR_UNSUPPORTED, "input_prep_u8_rrc: mode %d (0 or 2 only)", mode);
  }
  const int threads = (OW + 31) / 32 * 32;
  const size_t smem = (size_t)kRrcTaps * threads * sizeof(int) + (size_t)kRrcRows * OW * C;
  const dim3 grid((OH + kRrcRows - 1) / kRrcRows, B * D);
  cudaError_t e = cudaFuncSetAttribute(input_prep_rrc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "input_prep_u8_rrc: smem attribute (%d bytes): %s", (int)smem,
               cudaGetErrorString(e));
  b200::launch(input_prep_rrc_kernel, grid, threads, smem, (cudaStream_t)stream, regions, region_bytes, index, draws,
               D, C, OH, OW, Cpad, mode, lut, (__nv_bfloat16*)out);
  B200_CHECK_LAUNCH("input_prep_rrc_kernel");
  return B200_OK;
}

extern "C" int b200_input_prep_u8_scale_crop(const uint8_t* regions, long long region_bytes, const long long* index,
                                             const int* geom, int B, int C, int OH, int OW, int Cpad, int mode,
                                             const float* lut, void* out, b200_stream_t stream) {
  B200_REQUIRE(regions && index && geom && lut && out && region_bytes > 0 && B > 0 && C > 0 && C <= 4 && OH > 0 &&
                   OW > 0,
               B200_ERR_INVALID, "input_prep_u8_scale_crop: bad argument (C must be 1..4)");
  B200_REQUIRE(OW <= kRrcMaxOW, B200_ERR_UNSUPPORTED, "input_prep_u8_scale_crop: OW=%d above %d", OW, kRrcMaxOW);
  B200_REQUIRE(B <= 65535, B200_ERR_UNSUPPORTED, "input_prep_u8_scale_crop: B=%d above 65535", B);
  B200_REQUIRE(Cpad % 8 == 0, B200_ERR_INVALID, "input_prep_u8_scale_crop: Cpad=%d must be a multiple of 8", Cpad);
  if (mode == 0) {
    B200_REQUIRE(Cpad >= C, B200_ERR_INVALID, "input_prep_u8_scale_crop: Cpad < C");
  } else if (mode == 2) {
    B200_REQUIRE(OH % 2 == 0 && OW % 2 == 0 && Cpad >= 4 * C, B200_ERR_UNSUPPORTED,
                 "input_prep_u8_scale_crop: space-to-depth needs even OH, OW and Cpad >= 4C");
  } else {
    B200_REQUIRE(false, B200_ERR_UNSUPPORTED, "input_prep_u8_scale_crop: mode %d (0 or 2 only)", mode);
  }
  const int threads = (OW + 31) / 32 * 32;
  const size_t smem = (size_t)kRrcTaps * threads * sizeof(int) + (size_t)kRrcRows * OW * C;
  const dim3 grid((OH + kRrcRows - 1) / kRrcRows, B);
  cudaError_t e = cudaFuncSetAttribute(input_prep_scale_crop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem);
  B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "input_prep_u8_scale_crop: smem attribute (%d bytes): %s", (int)smem,
               cudaGetErrorString(e));
  b200::launch(input_prep_scale_crop_kernel, grid, threads, smem, (cudaStream_t)stream, regions, region_bytes, index,
               geom, C, OH, OW, Cpad, mode, lut, (__nv_bfloat16*)out);
  B200_CHECK_LAUNCH("input_prep_scale_crop_kernel");
  return B200_OK;
}
