// Layout / precision transforms around the tensor-core kernels:
//  - network input NCHW fp32 -> NHWC bf16 (channel padded) or space-to-depth NHWC bf16 for the 7x7/s2 stem
//    (replaces inputs.to(device, dtype), trainer.py:116-117, plus the relayout cuDNN does internally)
//  - weight relayouts: [K][T][C] -> [C][T][K] for dgrad, 7x7 stem <-> 4x4 space-to-depth form
//  - fp32 -> bf16 cast of flat arrays
#include "common.cuh"
#include "host.h"

namespace b200 {

// Optional input mixing (MixUp / CutMix of the reference's utils/mixup.py:19-26,57-90, applied at trainer.py:119-135).
// MIX is a template parameter so that the plain instantiation compiles to exactly the code it had without mixing.
//   MIX == 1 (MixUp):  v = lambda * x[n] + (1 - lambda) * x[perm[n]], two fp32 products and one fp32 sum (no FMA
//                      contraction: the reference's torch expression, bit for bit), then the single bf16 rounding.
//   MIX == 2 (CutMix): pixel (r, c) of sample n comes from sample perm[n] inside the box [r0, r1) x [c0, c1), else
//                      from n; in the space-to-depth layouts every one of the four sub-pixels decides on its own.
// The parameter block lives in device memory so that a captured CUDA graph reads each step's values.
constexpr int kMixNone = 0, kMixUp = 1, kMixCut = 2;

template <int MIX>
__device__ __forceinline__ float mix_pick(float a, float b, float lam) {
  return MIX == kMixUp ? __fadd_rn(__fmul_rn(lam, a), __fmul_rn(__fsub_rn(1.f, lam), b)) : a;
}

__device__ __forceinline__ bool in_box(const b200_mix_params& p, int r, int c) {
  return r >= p.r0 && r < p.r1 && c >= p.c0 && c < p.c1;
}

// source image of the element at pixel (r, c): x[n], or x[perm[n]] where CutMix pastes its box
template <int MIX, typename T>
__device__ __forceinline__ const T* mix_src(const T* xi, const T* xm, const b200_mix_params& p, int r, int c) {
  return (MIX == kMixCut && in_box(p, r, c)) ? xm : xi;
}

template <int MIX>
__global__ void __launch_bounds__(256) input_prep_kernel(const float* __restrict__ x, int N, int C, int H, int W,
                                                         int Cpad, int mode, __nv_bfloat16* __restrict__ out,
                                                         const long long* __restrict__ perm,
                                                         const b200_mix_params* __restrict__ mixp) {
  b200_mix_params mp = {};
  if (MIX != kMixNone) mp = *mixp;
  // one thread per output pixel; Cpad is a multiple of 8
  const int brd = mode == 2 ? 2 : 0;                       // low border of the padded space-to-depth layout
  const int OH = mode == 0 ? H : H / 2 + (mode == 2 ? 3 : 0), OW = mode == 0 ? W : W / 2 + (mode == 2 ? 3 : 0);
  const long long total = (long long)N * OH * OW;
  const long long plane = (long long)H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % OW) - brd;
    const int i = (int)((idx / OW) % OH) - brd;
    const int n = (int)(idx / ((long long)OW * OH));
    __nv_bfloat16* o = out + idx * Cpad;
    const bool inside = mode != 2 || (i >= 0 && j >= 0 && i < H / 2 && j < W / 2);
    const float* xi = x + (long long)n * C * plane;
    const float* xm = MIX != kMixNone ? x + __ldg(perm + n) * C * plane : xi;
    for (int c0 = 0; c0 < Cpad; c0 += 8) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int ch = c0 + e;
        float val = 0.f;
        if (mode == 0) {
          if (ch < C) {
            if (MIX == kMixNone) {
              val = __ldg(xi + (long long)ch * plane + (long long)i * W + j);
            } else {
              const long long off = (long long)ch * plane + (long long)i * W + j;
              val = __ldg(mix_src<MIX>(xi, xm, mp, i, j) + off);
              if (MIX == kMixUp) val = mix_pick<MIX>(val, __ldg(xm + off), mp.lam);
            }
          }
        } else {
          const int sub = ch / C, c = ch - sub * C;  // sub = dy*2+dx
          if (sub < 4 && inside) {
            const int dy = sub >> 1, dx = sub & 1;
            if (MIX == kMixNone) {
              val = __ldg(xi + (long long)c * plane + (long long)(2 * i + dy) * W + (2 * j + dx));
            } else {
              const long long off = (long long)c * plane + (long long)(2 * i + dy) * W + (2 * j + dx);
              val = __ldg(mix_src<MIX>(xi, xm, mp, 2 * i + dy, 2 * j + dx) + off);
              if (MIX == kMixUp) val = mix_pick<MIX>(val, __ldg(xm + off), mp.lam);
            }
          }
        }
        f[e] = val;
      }
      uint4 u;
      u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
      u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
      *reinterpret_cast<uint4*>(o + c0) = u;
    }
  }
}

// uint8 NHWC images (what a decoder produces) -> the same bf16 layouts, normalised on the fly:
// value = u8 * scale[c] + bias[c]  (scale = 1 / (255 * std), bias = -mean / std: ToTensor + Normalize of the reference's
// preprocess.py:20-24).  4x fewer host->device bytes than the fp32 NCHW batch and no separate normalisation pass.
struct U8Norm { float scale[4], bias[4]; };

// Batch augmentation (AUG, mode 0 only): output row n of N = B*D rows is copy n % D of image n / D after the
// reference's RandomCrop(padding) + RandomHorizontalFlip + ToTensor + Normalize + Cutout (preprocess.py:44-54,185-227).
// params[n] = {oy, ox, flip, y1, y2, x1, x2, ...} (int16, holes boxes); lut[c][u] = Normalize(ToTensor(u)) in fp32, as
// torchvision computes it; a cut element is v * 0 (the reference multiplies by its mask: a signed zero).  Any values in
// params are memory-safe: a source pixel is read only when it lies inside image n / D, else the pad value 0 is used.
struct U8Aug { const int16_t* params; const float* lut; int D, pad, holes; };

template <int MIX, bool AUG = false>
__global__ void __launch_bounds__(256) input_prep_u8_kernel(const uint8_t* __restrict__ x, int N, int C, int H, int W,
                                                            int Cpad, int mode, U8Norm nm,
                                                            __nv_bfloat16* __restrict__ out,
                                                            const long long* __restrict__ perm,
                                                            const b200_mix_params* __restrict__ mixp, U8Aug ag) {
  static_assert(!AUG || MIX == kMixNone, "batch augmentation is not combined with mixing");
  b200_mix_params mp = {};
  if (MIX != kMixNone) mp = *mixp;
  const int brd = mode == 2 ? 2 : 0;
  const int OH = mode == 0 ? H : H / 2 + (mode == 2 ? 3 : 0), OW = mode == 0 ? W : W / 2 + (mode == 2 ? 3 : 0);
  const long long total = (long long)N * OH * OW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % OW) - brd;
    const int i = (int)((idx / OW) % OH) - brd;
    const int n = (int)(idx / ((long long)OW * OH));
    __nv_bfloat16* o = out + idx * Cpad;
    if (AUG) {
      const int16_t* pr = ag.params + (long long)n * (3 + 4 * ag.holes);
      const int cs = __ldg(pr + 2) != 0 ? W - 1 - j : j;
      const int sy = i + __ldg(pr + 0) - ag.pad, sx = cs + __ldg(pr + 1) - ag.pad;
      const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
      bool cut = false;
      for (int h = 0; h < ag.holes; ++h) {
        const int16_t* b = pr + 3 + 4 * h;
        cut |= i >= __ldg(b + 0) && i < __ldg(b + 1) && j >= __ldg(b + 2) && j < __ldg(b + 3);
      }
      const uint8_t* src = x + ((long long)(n / ag.D) * H * W + (ok ? (long long)sy * W + sx : 0)) * C;
      for (int c0 = 0; c0 < Cpad; c0 += 8) {
        float f[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int ch = c0 + e;
          float val = 0.f;
          if (ch < C) {
            val = __ldg(ag.lut + ch * 256 + (ok ? __ldg(src + ch) : 0));
            if (cut) val = __fmul_rn(val, 0.f);
          }
          f[e] = val;
        }
        uint4 u;
        u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
        u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
        *reinterpret_cast<uint4*>(o + c0) = u;
      }
      continue;
    }
    const bool inside = mode != 2 || (i >= 0 && j >= 0 && i < H / 2 && j < W / 2);
    const uint8_t* xi = x + (long long)n * H * W * C;
    const uint8_t* xm = MIX != kMixNone ? x + __ldg(perm + n) * H * W * C : xi;
    for (int c0 = 0; c0 < Cpad; c0 += 8) {
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int ch = c0 + e;
        float val = 0.f;
        // each source is normalised on its own (the fp32 batch the reference mixes), then mixed
        if (mode == 0) {
          if (ch < C) {
            if (MIX == kMixNone) {
              val = fmaf((float)__ldg(xi + ((long long)i * W + j) * C + ch), nm.scale[ch], nm.bias[ch]);
            } else {
              const long long off = ((long long)i * W + j) * C + ch;
              val = fmaf((float)__ldg(mix_src<MIX>(xi, xm, mp, i, j) + off), nm.scale[ch], nm.bias[ch]);
              if (MIX == kMixUp)
                val = mix_pick<MIX>(val, fmaf((float)__ldg(xm + off), nm.scale[ch], nm.bias[ch]), mp.lam);
            }
          }
        } else {
          const int sub = ch / C, c = ch - sub * C;  // sub = dy*2+dx
          if (sub < 4 && inside) {
            const int dy = sub >> 1, dx = sub & 1;
            if (MIX == kMixNone) {
              val = fmaf((float)__ldg(xi + ((long long)(2 * i + dy) * W + (2 * j + dx)) * C + c), nm.scale[c], nm.bias[c]);
            } else {
              const long long off = ((long long)(2 * i + dy) * W + (2 * j + dx)) * C + c;
              val = fmaf((float)__ldg(mix_src<MIX>(xi, xm, mp, 2 * i + dy, 2 * j + dx) + off), nm.scale[c], nm.bias[c]);
              if (MIX == kMixUp)
                val = mix_pick<MIX>(val, fmaf((float)__ldg(xm + off), nm.scale[c], nm.bias[c]), mp.lam);
            }
          }
        }
        f[e] = val;
      }
      uint4 u;
      u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
      u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
      *reinterpret_cast<uint4*>(o + c0) = u;
    }
  }
}

// bf16 [K][T][C] -> [C][T][K]; one 32x32 tile per block, blockIdx.z = tap
__global__ void __launch_bounds__(256) weight_transpose_kernel(const __nv_bfloat16* __restrict__ src,
                                                               __nv_bfloat16* __restrict__ dst, int K, int T, int C) {
  __shared__ __nv_bfloat16 tile[32][33];
  const int t = blockIdx.z;
  const int c0 = blockIdx.x * 32, k0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int r = ty; r < 32; r += 8) {
    const int k = k0 + r, c = c0 + tx;
    tile[r][tx] = (k < K && c < C) ? src[((long long)k * T + t) * C + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, k = k0 + tx;
    if (c < C && k < K) dst[((long long)c * T + t) * K + k] = tile[tx][r];
  }
}

// multi-tensor version: one launch transposes every conv weight of the network (53 launches -> 1 per step).
// jobs[j] = {src_off, dst_off, K, T, C, tile_start} in elements of the two arenas; a block owns one 32x32 tile and
// finds its job by binary search over tile_start.
__global__ void __launch_bounds__(256) weight_transpose_batched_kernel(const __nv_bfloat16* __restrict__ src_base,
                                                                       __nv_bfloat16* __restrict__ dst_base,
                                                                       const int* __restrict__ jobs, int njobs) {
  __shared__ __nv_bfloat16 tile[32][33];
  int lo = 0, hi = njobs - 1;
  const int g = blockIdx.x;
  while (lo < hi) {   // last job with tile_start <= g
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(jobs + mid * 6 + 5) <= g) lo = mid; else hi = mid - 1;
  }
  const int* jb = jobs + lo * 6;
  const __nv_bfloat16* src = src_base + __ldg(jb + 0);
  __nv_bfloat16* dst = dst_base + __ldg(jb + 1);
  const int K = __ldg(jb + 2), T = __ldg(jb + 3), C = __ldg(jb + 4);
  const int local = g - __ldg(jb + 5);
  const int tiles_c = (C + 31) >> 5, tiles_k = (K + 31) >> 5;
  const int t = local / (tiles_c * tiles_k);
  const int rem = local - t * tiles_c * tiles_k;
  const int k0 = (rem / tiles_c) * 32, c0 = (rem % tiles_c) * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const int k = k0 + r, c = c0 + tx;
    tile[r][tx] = (k < K && c < C) ? src[((long long)k * T + t) * C + c] : __float2bfloat16(0.f);
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int c = c0 + r, k = k0 + tx;
    if (c < C && k < K) dst[((long long)c * T + t) * K + k] = tile[tx][r];
  }
}

// stem: w fp32 [K][7][7][C] -> bf16 [K][16][Cpad], tap (ah,aw) in 4x4, channel (bh*2+bw)*C + c,
// r = 2*ah + bh - 1, s = 2*aw + bw - 1 (out-of-range -> 0)
__global__ void stem_w_to_s2d_kernel(const float* __restrict__ w, int K, int C, int Cpad,
                                     __nv_bfloat16* __restrict__ out) {
  const int total = K * 16 * Cpad;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int ch = idx % Cpad;
    const int tap = (idx / Cpad) % 16;
    const int k = idx / (Cpad * 16);
    const int ah = tap >> 2, aw = tap & 3;
    float val = 0.f;
    const int sub = ch / C, c = ch - sub * C;
    if (sub < 4) {
      const int r = 2 * ah + (sub >> 1) - 1, s = 2 * aw + (sub & 1) - 1;
      if (r >= 0 && r < 7 && s >= 0 && s < 7) val = w[(((long long)k * 7 + r) * 7 + s) * C + c];
    }
    out[idx] = __float2bfloat16(val);
  }
}
// reverse gather for the gradient: dw[K][7][7][C] += dw_s2d[K][16][Cpad]
__global__ void stem_wgrad_from_s2d_kernel(const float* __restrict__ dws, int K, int C, int Cpad,
                                           float* __restrict__ dw) {
  const int total = K * 49 * C;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int c = idx % C;
    const int s = (idx / C) % 7;
    const int r = (idx / (C * 7)) % 7;
    const int k = idx / (C * 49);
    const int ah = (r + 1) >> 1, bh = (r + 1) & 1, aw = (s + 1) >> 1, bw = (s + 1) & 1;
    dw[idx] += dws[((long long)k * 16 + ah * 4 + aw) * Cpad + (bh * 2 + bw) * C + c];
  }
}

__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ src,
                                                            __nv_bfloat16* __restrict__ dst, long long n) {
  const long long n4 = n >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 f = __ldg(reinterpret_cast<const float4*>(src) + i);
    uint2 u;
    u.x = pack_bf16x2(f.x, f.y);
    u.y = pack_bf16x2(f.z, f.w);
    reinterpret_cast<uint2*>(dst)[i] = u;
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = __float2bfloat16(src[i]);
}

static inline int grid_cap(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace b200

using namespace b200;

static int input_prep_impl(const float* x, int N, int C, int H, int W, int Cpad, int mode, const long long* perm,
                           const b200_mix_params* params, int kind, void* out, b200_stream_t stream) {
  B200_REQUIRE(x && out && N > 0 && C > 0 && H > 0 && W > 0, B200_ERR_INVALID, "input_prep: bad argument");
  B200_REQUIRE(Cpad % 8 == 0, B200_ERR_UNSUPPORTED, "input_prep: Cpad=%d must be a multiple of 8", Cpad);
  if (mode == 0) {
    B200_REQUIRE(Cpad >= C, B200_ERR_INVALID, "input_prep: Cpad < C");
  } else if (mode == 1 || mode == 2) {
    B200_REQUIRE(H % 2 == 0 && W % 2 == 0 && Cpad >= 4 * C, B200_ERR_UNSUPPORTED,
                 "input_prep: space-to-depth needs even H,W and Cpad >= 4C");
  } else {
    B200_REQUIRE(false, B200_ERR_INVALID, "input_prep: unknown mode %d", mode);
  }
  B200_REQUIRE(kind >= B200_MIX_NONE && kind <= B200_MIX_CUTMIX, B200_ERR_INVALID, "input_prep: unknown mix kind %d", kind);
  B200_REQUIRE(kind == B200_MIX_NONE || (perm && params), B200_ERR_INVALID, "input_prep: mixing needs perm and params");
  const long long total = (long long)N * (mode == 0 ? (long long)H * W : (long long)(H / 2 + (mode == 2 ? 3 : 0)) * (W / 2 + (mode == 2 ? 3 : 0)));
  const int grid = grid_cap(total, 256);
  if (kind == B200_MIX_MIXUP)
    b200::launch(input_prep_kernel<kMixUp>, grid, 256, 0, (cudaStream_t)stream, x, N, C, H, W, Cpad, mode,
                 (__nv_bfloat16*)out, perm, params);
  else if (kind == B200_MIX_CUTMIX)
    b200::launch(input_prep_kernel<kMixCut>, grid, 256, 0, (cudaStream_t)stream, x, N, C, H, W, Cpad, mode,
                 (__nv_bfloat16*)out, perm, params);
  else
    b200::launch(input_prep_kernel<kMixNone>, grid, 256, 0, (cudaStream_t)stream, x, N, C, H, W, Cpad, mode,
                 (__nv_bfloat16*)out, (const long long*)nullptr, (const b200_mix_params*)nullptr);
  B200_CHECK_LAUNCH("input_prep_kernel");
  return B200_OK;
}

static int input_prep_u8_impl(const uint8_t* x_nhwc, int N, int C, int H, int W, int Cpad, int mode,
                              const float* scale_host, const float* bias_host, const long long* perm,
                              const b200_mix_params* params, int kind, void* out, b200_stream_t stream) {
  B200_REQUIRE(x_nhwc && out && scale_host && bias_host && N > 0 && C > 0 && C <= 4 && H > 0 && W > 0,
               B200_ERR_INVALID, "input_prep_u8: bad argument (C must be 1..4)");
  B200_REQUIRE(Cpad % 8 == 0 && Cpad >= C, B200_ERR_INVALID, "input_prep_u8: Cpad must be a multiple of 8 and >= C");
  B200_REQUIRE(mode >= 0 && mode <= 2, B200_ERR_INVALID, "input_prep_u8: unknown mode %d", mode);
  if (mode != 0)
    B200_REQUIRE(H % 2 == 0 && W % 2 == 0 && 4 * C <= Cpad, B200_ERR_UNSUPPORTED,
                 "input_prep_u8: space-to-depth needs even H, W and 4*C <= Cpad");
  B200_REQUIRE(kind >= B200_MIX_NONE && kind <= B200_MIX_CUTMIX, B200_ERR_INVALID, "input_prep_u8: unknown mix kind %d",
               kind);
  B200_REQUIRE(kind == B200_MIX_NONE || (perm && params), B200_ERR_INVALID, "input_prep_u8: mixing needs perm and params");
  U8Norm nm;
  for (int c = 0; c < 4; ++c) { nm.scale[c] = c < C ? scale_host[c] : 0.f; nm.bias[c] = c < C ? bias_host[c] : 0.f; }
  const int OH = mode == 0 ? H : H / 2 + (mode == 2 ? 3 : 0), OW = mode == 0 ? W : W / 2 + (mode == 2 ? 3 : 0);
  const long long total = (long long)N * OH * OW;
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  if (kind == B200_MIX_MIXUP)
    b200::launch(input_prep_u8_kernel<kMixUp>, (int)blocks, 256, 0, (cudaStream_t)stream, x_nhwc, N, C, H, W, Cpad,
                 mode, nm, (__nv_bfloat16*)out, perm, params, U8Aug{});
  else if (kind == B200_MIX_CUTMIX)
    b200::launch(input_prep_u8_kernel<kMixCut>, (int)blocks, 256, 0, (cudaStream_t)stream, x_nhwc, N, C, H, W, Cpad,
                 mode, nm, (__nv_bfloat16*)out, perm, params, U8Aug{});
  else
    b200::launch(input_prep_u8_kernel<kMixNone>, (int)blocks, 256, 0, (cudaStream_t)stream, x_nhwc, N, C, H, W, Cpad,
                 mode, nm, (__nv_bfloat16*)out, (const long long*)nullptr, (const b200_mix_params*)nullptr, U8Aug{});
  B200_CHECK_LAUNCH("input_prep_u8_kernel");
  return B200_OK;
}

extern "C" int b200_input_prep_u8_aug(const uint8_t* x_nhwc, int N, int D, int C, int H, int W, int Cpad, int pad,
                                      const float* lut, const int16_t* params, int holes, void* out,
                                      b200_stream_t stream) {
  B200_REQUIRE(x_nhwc && out && lut && params && N > 0 && D > 0 && C > 0 && C <= 4 && H > 0 && W > 0,
               B200_ERR_INVALID, "input_prep_u8_aug: bad argument (C must be 1..4)");
  B200_REQUIRE(Cpad % 8 == 0 && Cpad >= C, B200_ERR_INVALID, "input_prep_u8_aug: Cpad must be a multiple of 8 and >= C");
  B200_REQUIRE(pad >= 0 && holes >= 0 && holes <= 64, B200_ERR_INVALID, "input_prep_u8_aug: pad=%d holes=%d out of range",
               pad, holes);
  B200_REQUIRE((long long)N * D <= 0x7fffffffLL, B200_ERR_UNSUPPORTED, "input_prep_u8_aug: N*D too large");
  const U8Norm nm = {};
  const long long total = (long long)N * D * H * W;
  b200::launch(input_prep_u8_kernel<kMixNone, true>, grid_cap(total, 256), 256, 0, (cudaStream_t)stream, x_nhwc,
               N * D, C, H, W, Cpad, 0, nm, (__nv_bfloat16*)out, (const long long*)nullptr,
               (const b200_mix_params*)nullptr, U8Aug{params, lut, D, pad, holes});
  B200_CHECK_LAUNCH("input_prep_u8_aug_kernel");
  return B200_OK;
}

extern "C" int b200_input_prep(const float* x, int N, int C, int H, int W, int Cpad, int mode, void* out,
                               b200_stream_t stream) {
  return input_prep_impl(x, N, C, H, W, Cpad, mode, nullptr, nullptr, B200_MIX_NONE, out, stream);
}

extern "C" int b200_input_prep_mix(const float* x, int N, int C, int H, int W, int Cpad, int mode, const long long* perm,
                                   const b200_mix_params* params, int kind, void* out, b200_stream_t stream) {
  return input_prep_impl(x, N, C, H, W, Cpad, mode, perm, params, kind, out, stream);
}

extern "C" int b200_input_prep_u8(const uint8_t* x_nhwc, int N, int C, int H, int W, int Cpad, int mode,
                                  const float* scale_host, const float* bias_host, void* out, b200_stream_t stream) {
  return input_prep_u8_impl(x_nhwc, N, C, H, W, Cpad, mode, scale_host, bias_host, nullptr, nullptr, B200_MIX_NONE, out,
                            stream);
}

extern "C" int b200_input_prep_u8_mix(const uint8_t* x_nhwc, int N, int C, int H, int W, int Cpad, int mode,
                                      const float* scale_host, const float* bias_host, const long long* perm,
                                      const b200_mix_params* params, int kind, void* out, b200_stream_t stream) {
  return input_prep_u8_impl(x_nhwc, N, C, H, W, Cpad, mode, scale_host, bias_host, perm, params, kind, out, stream);
}

extern "C" int b200_weight_transpose(const void* src, void* dst, int K, int T, int C, b200_stream_t stream) {
  B200_REQUIRE(src && dst && K > 0 && T > 0 && C > 0, B200_ERR_INVALID, "weight_transpose: bad argument");
  dim3 grid((C + 31) / 32, (K + 31) / 32, T);
  b200::launch(weight_transpose_kernel, grid, 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)src, (__nv_bfloat16*)dst, K, T,
                                                                C);
  B200_CHECK_LAUNCH("weight_transpose_kernel");
  return B200_OK;
}

extern "C" int b200_weight_transpose_batched(const void* src_base, void* dst_base, const int* jobs, int njobs,
                                             int total_tiles, b200_stream_t stream) {
  B200_REQUIRE(src_base && dst_base && jobs && njobs > 0 && total_tiles > 0, B200_ERR_INVALID,
               "weight_transpose_batched: bad argument");
  b200::launch(weight_transpose_batched_kernel, total_tiles, 256, 0, (cudaStream_t)stream,
      (const __nv_bfloat16*)src_base, (__nv_bfloat16*)dst_base, jobs, njobs);
  B200_CHECK_LAUNCH("weight_transpose_batched_kernel");
  return B200_OK;
}

extern "C" int b200_stem_weight_to_s2d(const float* w, int K, int C, int Cpad, void* w_s2d, b200_stream_t stream) {
  B200_REQUIRE(w && w_s2d && K > 0 && C > 0 && Cpad >= 4 * C, B200_ERR_INVALID, "stem_weight_to_s2d: bad argument");
  b200::launch(stem_w_to_s2d_kernel, (K * 16 * Cpad + 255) / 256, 256, 0, (cudaStream_t)stream, w, K, C, Cpad,
                                                                                    (__nv_bfloat16*)w_s2d);
  B200_CHECK_LAUNCH("stem_w_to_s2d_kernel");
  return B200_OK;
}

extern "C" int b200_stem_wgrad_from_s2d(const float* dw_s2d, int K, int C, int Cpad, float* dw, b200_stream_t stream) {
  B200_REQUIRE(dw_s2d && dw && K > 0 && C > 0 && Cpad >= 4 * C, B200_ERR_INVALID, "stem_wgrad_from_s2d: bad argument");
  b200::launch(stem_wgrad_from_s2d_kernel, (K * 49 * C + 255) / 256, 256, 0, (cudaStream_t)stream, dw_s2d, K, C, Cpad, dw);
  B200_CHECK_LAUNCH("stem_wgrad_from_s2d_kernel");
  return B200_OK;
}

extern "C" int b200_cast_f32_to_bf16(const float* src, void* dst, long long n, b200_stream_t stream) {
  B200_REQUIRE(src && dst && n >= 0, B200_ERR_INVALID, "cast_f32_to_bf16: bad argument");
  if (n == 0) return B200_OK;
  b200::launch(cast_f32_bf16_kernel, grid_cap((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream, src, (__nv_bfloat16*)dst, n);
  B200_CHECK_LAUNCH("cast_f32_bf16_kernel");
  return B200_OK;
}

// ---- grouped convolution support (ResNeXt, nn.Conv2d(groups=32), models/resnext.py:10-16) -------------------------
// A grouped convolution with C == K is block diagonal at ANY granularity that is a multiple of the group width: output
// channels [W*b, W*b+W) only read input channels of the same window.  The tensor-core kernels run it as K/W independent
// W-wide diagonal blocks ("window" mode of the conv entry points, W = 64 for fprop/dgrad, 128 for the k-tile of wgrad),
// so the weight operand is packed per window:
//   pack      : w_g fp32 [K][T][C/g] -> bf16 [K][T][W],   out[k][t][cl] = w_g[k][t][c - first(k)] if channel
//               c = W*(k/W) + cl lies in the group of k, else 0                                   (fprop operand)
//   transposed: bf16 [C][T][W],  out[c][t][kl] = the same weight seen from input channel c, k = W*(c/W) + kl (dgrad operand)
//   unpack    : dw_g[k][t][cl] += dw_win[k][t][first(k) + cl - W*(k/W)]   from the windowed fp32 gradient [K][T][W]
// W == C is the dense block-diagonal expansion, for any C and K (ResNeXt's C != K stage entries): window origin 0,
// operands [K][T][C] (fprop) and [C][T][K] (dgrad), unpack from a dense [K][T][C] gradient.
namespace b200 {
__global__ void __launch_bounds__(256) group_pack_kernel(const float* __restrict__ wg, int K, int T, int C, int groups,
                                                         int Wd, int transpose, __nv_bfloat16* __restrict__ out) {
  const int cg = C / groups, kg = K / groups;
  const bool dense = Wd == C;
  const int rows = transpose ? C : K;
  const int width = (transpose && dense) ? K : Wd;   // row length of the operand
  const long long total = (long long)rows * T * width;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int l = (int)(idx % width);
    const int t = (int)((idx / width) % T);
    const int row = (int)(idx / ((long long)width * T));
    int k, c;
    if (transpose) { c = row; k = dense ? l : (c / Wd) * Wd + l; } else { k = row; c = dense ? l : (k / Wd) * Wd + l; }
    float v = 0.f;
    if (k < K && c < C) {
      const int grp = k / kg;
      if (c / cg == grp) v = wg[((long long)k * T + t) * cg + (c - grp * cg)];
    }
    out[idx] = __float2bfloat16(v);
  }
}
__global__ void __launch_bounds__(256) group_unpack_kernel(const float* __restrict__ dw_win, int K, int T, int C,
                                                           int groups, int Wd, float* __restrict__ dwg) {
  const int cg = C / groups, kg = K / groups;
  const long long total = (long long)K * T * cg;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int cl = (int)(idx % cg);
    const int t = (int)((idx / cg) % T);
    const int k = (int)(idx / ((long long)cg * T));
    const int c = (k / kg) * cg + cl;
    dwg[idx] += dw_win[((long long)k * T + t) * Wd + (Wd == C ? c : c - (k / Wd) * Wd)];
  }
}
}  // namespace b200

extern "C" int b200_group_weight_pack(const float* w_grouped, int K, int T, int C, int groups, int window, int transpose,
                                      void* out_bf16, b200_stream_t stream) {
  B200_REQUIRE(w_grouped && out_bf16 && K > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0 && K % groups == 0,
               B200_ERR_INVALID, "group_weight_pack: bad argument");
  B200_REQUIRE(window > 0 && window % (C / groups) == 0 && window % (K / groups) == 0 && (window == C || (C == K && C % window == 0)),
               B200_ERR_UNSUPPORTED, "group_weight_pack: window %d must be a multiple of the group width and divide C == K",
               window);
  const long long total = (long long)(transpose ? C : K) * T * ((transpose && window == C) ? K : window);
  b200::launch(b200::group_pack_kernel, b200::grid_cap(total, 256), 256, 0, (cudaStream_t)stream,
      w_grouped, K, T, C, groups, window, transpose, (__nv_bfloat16*)out_bf16);
  B200_CHECK_LAUNCH("group_pack_kernel");
  return B200_OK;
}

extern "C" int b200_group_wgrad_unpack(const float* dw_win, int K, int T, int C, int groups, int window, float* dw_grouped,
                                       b200_stream_t stream) {
  B200_REQUIRE(dw_win && dw_grouped && K > 0 && T > 0 && C > 0 && groups > 0 && C % groups == 0 && K % groups == 0,
               B200_ERR_INVALID, "group_wgrad_unpack: bad argument");
  B200_REQUIRE(window > 0 && window % (C / groups) == 0 && window % (K / groups) == 0 && (window == C || (C == K && C % window == 0)),
               B200_ERR_UNSUPPORTED, "group_wgrad_unpack: window %d must be a multiple of the group width and divide C == K",
               window);
  const long long total = (long long)K * T * (C / groups);
  b200::launch(b200::group_unpack_kernel, b200::grid_cap(total, 256), 256, 0, (cudaStream_t)stream, dw_win, K, T, C, groups, window,
                                                                                       dw_grouped);
  B200_CHECK_LAUNCH("group_unpack_kernel");
  return B200_OK;
}
