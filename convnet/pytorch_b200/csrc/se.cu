// Squeeze-and-excitation on the residual branch (reference models/modules/se.py:6-25, used by resnet_se / resnext_se,
// models/resnet.py:112-113,159-160,434-436):   r' = r * sigmoid(W2 relu(W1 mean_hw(r) + b1) + b2).
// The two tiny linear layers run on the wgmma 1x1-conv kernels; this file holds the HBM-bound NHWC bf16 passes
// around them (pool, scale, and the two backward passes) plus a generic elementwise activation backward.
//   forward : se_pool (read r) -> [MLP] -> se_scale_fwd (read r, write r')
//   backward: se_bwd_reduce (read g, r: dlogit = sigma' * sum_hw g*r) -> [MLP backward] ->
//             se_bwd_dx (read g, write dr = g * sigma + dmean / HW)
#include "common.cuh"
#include "host.h"

namespace b200 {

__device__ __forceinline__ void se_ld8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void se_st8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + __expf(-x)); }

// One block per (image, 64-channel slab): 8 channel vectors x 32 row lanes; rows strided by 32, smem tree at the end.
// MODE 0: out[n][c] = mean_hw a          (bf16)            -- squeeze
// MODE 1: out[n][c] = sigma'(logit) * sum_hw a * b  (bf16) -- gradient of the gate's pre-activation
template <int MODE>
__global__ void __launch_bounds__(256) se_reduce_kernel(const __nv_bfloat16* __restrict__ a,
                                                        const __nv_bfloat16* __restrict__ b,
                                                        const float* __restrict__ logit, int HW, int C,
                                                        __nv_bfloat16* __restrict__ out) {
  __shared__ float red[32][65];
  const int n = blockIdx.x, slab = blockIdx.y;
  const int v = threadIdx.x & 7, lane = threadIdx.x >> 3;      // 8 vectors of 8 channels, 32 row lanes
  const int c0 = slab * 64 + v * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c0 < C) {
    const long long base = (long long)n * HW * C + c0;
    for (int r = lane; r < HW; r += 32) {
      float fa[8];
      se_ld8(a + base + (long long)r * C, fa);
      if (MODE == 1) {
        float fb[8];
        se_ld8(b + base + (long long)r * C, fb);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = fmaf(fa[j], fb[j], acc[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += fa[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[lane][v * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = slab * 64 + threadIdx.x;
    if (c < C) {
      float s = 0.f;
#pragma unroll 8
      for (int l = 0; l < 32; ++l) s += red[l][threadIdx.x];
      if (MODE == 0) {
        s *= 1.f / (float)HW;
      } else {
        const float sg = sigmoidf(logit[(long long)n * C + c]);
        s *= sg * (1.f - sg);
      }
      out[(long long)n * C + c] = __float2bfloat16(s);
    }
  }
}

// MODE 0: out = r * sigma(logit[n][c])                       (forward gate)
// MODE 1: out = g * sigma(logit[n][c]) + dmean[n][c] / HW    (gradient w.r.t. r)
template <int MODE>
__global__ void __launch_bounds__(256) se_scale_kernel(const __nv_bfloat16* __restrict__ x,
                                                       const float* __restrict__ logit,
                                                       const __nv_bfloat16* __restrict__ dmean, long long total_vec,
                                                       int HW, int C, __nv_bfloat16* __restrict__ out) {
  const int cv = C >> 3;
  const float inv = 1.f / (float)HW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total_vec;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % cv);
    const long long pix = idx / cv;
    const int n = (int)(pix / HW);
    float f[8], m[8];
    se_ld8(x + pix * C + v * 8, f);
    const float4 l0 = *reinterpret_cast<const float4*>(logit + (long long)n * C + v * 8);
    const float4 l1 = *reinterpret_cast<const float4*>(logit + (long long)n * C + v * 8 + 4);
    m[0] = sigmoidf(l0.x); m[1] = sigmoidf(l0.y); m[2] = sigmoidf(l0.z); m[3] = sigmoidf(l0.w);
    m[4] = sigmoidf(l1.x); m[5] = sigmoidf(l1.y); m[6] = sigmoidf(l1.z); m[7] = sigmoidf(l1.w);
    if (MODE == 1) {
      float d[8];
      se_ld8(dmean + (long long)n * C + v * 8, d);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaf(f[j], m[j], d[j] * inv);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] *= m[j];
    }
    se_st8(out + pix * C + v * 8, f);
  }
}

// dx = dy * act'(y) for y = act(.) (ReLU / ReLU6), elementwise on bf16 vectors of 8
__global__ void __launch_bounds__(256) act_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                                      const __nv_bfloat16* __restrict__ y, long long nvec, int act,
                                                      __nv_bfloat16* __restrict__ dx) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float g[8], f[8];
    se_ld8(dy + i * 8, g);
    se_ld8(y + i * 8, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool pass = act == B200_ACT_RELU ? f[j] > 0.f : (act == B200_ACT_RELU6 ? (f[j] > 0.f && f[j] < 6.f) : true);
      g[j] = pass ? g[j] : 0.f;
    }
    se_st8(dx + i * 8, g);
  }
}

static inline int se_grid(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace b200

using namespace b200;

#define SE_CHECK_SHAPE(name)                                                                                   \
  B200_REQUIRE(N > 0 && HW > 0 && C > 0 && C % 8 == 0, B200_ERR_UNSUPPORTED, name ": N, HW > 0 and C %% 8 == 0 needed " \
               "(N=%d HW=%d C=%d)", N, HW, C)

extern "C" int b200_se_pool(const void* r, int N, int HW, int C, void* mean_bf16, b200_stream_t stream) {
  B200_REQUIRE(r && mean_bf16, B200_ERR_INVALID, "se_pool: null pointer");
  SE_CHECK_SHAPE("se_pool");
  dim3 grid(N, (C + 63) / 64);
  b200::launch(se_reduce_kernel<0>, grid, 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)r, nullptr, nullptr, HW, C,
                                                             (__nv_bfloat16*)mean_bf16);
  B200_CHECK_LAUNCH("se_reduce_kernel<0>");
  return B200_OK;
}

extern "C" int b200_se_scale_fwd(const void* r, const float* logit, int N, int HW, int C, void* out, b200_stream_t stream) {
  B200_REQUIRE(r && logit && out, B200_ERR_INVALID, "se_scale_fwd: null pointer");
  SE_CHECK_SHAPE("se_scale_fwd");
  const long long total = (long long)N * HW * (C / 8);
  b200::launch(se_scale_kernel<0>, se_grid(total, 256), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)r, logit, nullptr, total,
                                                                           HW, C, (__nv_bfloat16*)out);
  B200_CHECK_LAUNCH("se_scale_kernel<0>");
  return B200_OK;
}

extern "C" int b200_se_bwd_reduce(const void* g, const void* r, const float* logit, int N, int HW, int C,
                                  void* dlogit_bf16, b200_stream_t stream) {
  B200_REQUIRE(g && r && logit && dlogit_bf16, B200_ERR_INVALID, "se_bwd_reduce: null pointer");
  SE_CHECK_SHAPE("se_bwd_reduce");
  dim3 grid(N, (C + 63) / 64);
  b200::launch(se_reduce_kernel<1>, grid, 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)g, (const __nv_bfloat16*)r, logit, HW,
                                                             C, (__nv_bfloat16*)dlogit_bf16);
  B200_CHECK_LAUNCH("se_reduce_kernel<1>");
  return B200_OK;
}

extern "C" int b200_se_bwd_dx(const void* g, const float* logit, const void* dmean_bf16, int N, int HW, int C, void* dr,
                              b200_stream_t stream) {
  B200_REQUIRE(g && logit && dmean_bf16 && dr, B200_ERR_INVALID, "se_bwd_dx: null pointer");
  SE_CHECK_SHAPE("se_bwd_dx");
  const long long total = (long long)N * HW * (C / 8);
  b200::launch(se_scale_kernel<1>, se_grid(total, 256), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)g, logit,
                                                                           (const __nv_bfloat16*)dmean_bf16, total, HW, C,
                                                                           (__nv_bfloat16*)dr);
  B200_CHECK_LAUNCH("se_scale_kernel<1>");
  return B200_OK;
}

extern "C" int b200_act_bwd(const void* dy, const void* y, long long n, int act, void* dx, b200_stream_t stream) {
  B200_REQUIRE(dy && y && dx && n > 0 && n % 8 == 0, B200_ERR_INVALID, "act_bwd: bad argument (n %% 8 == 0 needed)");
  b200::launch(act_bwd_kernel, se_grid(n / 8, 256), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)dy, (const __nv_bfloat16*)y,
                                                                       n / 8, act, (__nv_bfloat16*)dx);
  B200_CHECK_LAUNCH("act_bwd_kernel");
  return B200_OK;
}
