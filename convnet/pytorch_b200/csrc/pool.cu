// Pooling for NHWC bf16: 3x3/s2/p1 max pool (argmax kept as one byte per output element so backward
// is a deterministic gather) and global average pool.  HBM-bound, 128-bit vectorised.
// Replaces nn.MaxPool2d(3,2,1) (models/resnet.py:230) and nn.AdaptiveAvgPool2d(1)
// (models/resnet.py:241,341; models/mobilenet_v2.py:124) forward and backward.
#include "common.cuh"
#include "host.h"
#include <math_constants.h>

namespace b200 {

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// AFFINE: the pooled tensor is act(x * scale[c] + shift[c]) rounded to bf16 -- BatchNorm apply + ReLU + max pool of the
// ImageNet stem in one pass (models/resnet.py:226-230), bit-identical to bn_apply followed by the plain pool, without
// writing and re-reading the [N, 112, 112, 64] activation
template <bool AFFINE>
__global__ void __launch_bounds__(256) maxpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, int N, int H, int W,
                                                          int C, int OH, int OW, const float* __restrict__ scale,
                                                          const float* __restrict__ shift, int act,
                                                          __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ amax) {
  const int cv = C >> 3;
  // 32-bit index arithmetic (the host checks N*H*W*C/8 < 2^31): 64-bit div/mod cost more than the loads
  const unsigned total = (unsigned)N * OH * OW * cv;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int v = (int)(idx % (unsigned)cv);
    unsigned pix = idx / (unsigned)cv;
    const int q = (int)(pix % (unsigned)OW); pix /= (unsigned)OW;
    const int p = (int)(pix % (unsigned)OH);
    const int n = (int)(pix / (unsigned)OH);
    float best[8];
    int bidx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { best[i] = -CUDART_INF_F; bidx[i] = 0; }
    float sc[8], sh[8];
    if (AFFINE) {
#pragma unroll
      for (int i = 0; i < 8; i += 4) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(scale + v * 8 + i));
        const float4 b = __ldg(reinterpret_cast<const float4*>(shift + v * 8 + i));
        sc[i] = a.x; sc[i + 1] = a.y; sc[i + 2] = a.z; sc[i + 3] = a.w;
        sh[i] = b.x; sh[i + 1] = b.y; sh[i + 2] = b.z; sh[i + 3] = b.w;
      }
    }
    bool first = true;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int h = 2 * p - 1 + r;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int w = 2 * q - 1 + s;
        if (w < 0 || w >= W) continue;
        float f[8];
        ld8(x + (((long long)n * H + h) * W + w) * C + v * 8, f);
        if (AFFINE) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float a = fmaf(f[i], sc[i], sh[i]);
            if (act == B200_ACT_RELU) a = fmaxf(a, 0.f);
            else if (act == B200_ACT_RELU6) a = fminf(fmaxf(a, 0.f), 6.f);
            f[i] = __bfloat162float(__float2bfloat16(a));     // the value bn_apply would have stored
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          // first occurrence wins on ties (strict >), NaN propagates, like ATen's max_pool2d
          if (first || f[i] > best[i] || f[i] != f[i]) { best[i] = f[i]; bidx[i] = r * 3 + s; }
        }
        first = false;
      }
    }
    const long long o = (((long long)n * OH + p) * OW + q) * C + v * 8;
    st8(y + o, best);
    if (amax != nullptr) {
      uint2 pk;
      pk.x = bidx[0] | (bidx[1] << 8) | (bidx[2] << 16) | (bidx[3] << 24);
      pk.y = bidx[4] | (bidx[5] << 8) | (bidx[6] << 16) | (bidx[7] << 24);
      *reinterpret_cast<uint2*>(amax + o) = pk;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Sliding-window backward: the pooled gradient rows stay in registers -- 2 loads instead of 8 per input-gradient
// vector, no 64-bit index arithmetic.  The kernel is bound by load requests in flight, like the BatchNorm ones.
struct PoolSlide {
  int N, H, W, C, OH, OW;
  int TP;                 // row pairs per work item
};
__device__ __forceinline__ uint4 pool_ldg(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// backward: a thread owns one INPUT column (n, w, v) and walks the row pairs (2j, 2j + 1); pooled rows j and j + 1 are
// the only ones whose windows contain them.  Column slots: even w lies in window q = w/2 only (local column 1), odd w
// in q = (w+1)/2 (local column 0) and q = (w-1)/2 (local column 2).
__global__ void __launch_bounds__(128) maxpool_bwd_slide_kernel(const __nv_bfloat16* __restrict__ dy,
                                                                const uint8_t* __restrict__ amax, const PoolSlide g,
                                                                __nv_bfloat16* __restrict__ dx) {
  const unsigned cv = (unsigned)g.C >> 3;
  const int J = (g.H + 1) >> 1;
  const unsigned chunks = (unsigned)(J + g.TP - 1) / (unsigned)g.TP;
  const unsigned total = (unsigned)g.N * chunks * (unsigned)g.W * cv;
  const unsigned step = gridDim.x * blockDim.x;
  const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
  const uint2 none2 = make_uint2(0xffffffffu, 0xffffffffu);   // argmax byte 255 never matches
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += step) {
    const unsigned v = idx % cv;
    unsigned t = idx / cv;
    const int wc = (int)(t % (unsigned)g.W); t /= (unsigned)g.W;
    const int ch = (int)(t % chunks);
    const int n = (int)(t / chunks);
    const bool odd = wc & 1;
    const int qa = odd ? (wc + 1) >> 1 : wc >> 1, sa = odd ? 0 : 1;
    const int qb = (wc - 1) >> 1, sb = 2;
    const bool oka = qa < g.OW, okb = odd && qb >= 0 && qb < g.OW;
    const size_t pn = (size_t)n * g.OH * g.OW;
    auto load_row = [&](int p, uint4& ga, uint2& ma, uint4& gb, uint2& mb) {
      ga = zero4; gb = zero4; ma = none2; mb = none2;
      if (p < 0 || p >= g.OH) return;
      const size_t r = (pn + (size_t)p * g.OW) * g.C + v * 8;
      if (oka) { ga = pool_ldg(dy + r + (size_t)qa * g.C); ma = __ldg(reinterpret_cast<const uint2*>(amax + r + (size_t)qa * g.C)); }
      if (okb) { gb = pool_ldg(dy + r + (size_t)qb * g.C); mb = __ldg(reinterpret_cast<const uint2*>(amax + r + (size_t)qb * g.C)); }
    };
    auto add_if = [](const uint4& gr, const uint2& mk, int want, float (&acc)[8]) {
      const uint32_t gw[4] = {gr.x, gr.y, gr.z, gr.w};
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int b = (i < 4 ? (mk.x >> (8 * i)) : (mk.y >> (8 * (i - 4)))) & 0xff;
        const float2 g2 = unpack_bf16x2(gw[i >> 1]);
        if (b == want) acc[i] += (i & 1) ? g2.y : g2.x;
      }
    };
    const int j0 = ch * g.TP, j1 = min(J, j0 + g.TP);
    uint4 cga, cgb, nga, ngb;
    uint2 cma, cmb, nma, nmb;
    load_row(j0, cga, cma, cgb, cmb);
    __nv_bfloat16* xo = dx + (((size_t)n * g.H + 2 * j0) * g.W + wc) * g.C + v * 8;
    for (int j = j0; j < j1; ++j) {
      load_row(j + 1, nga, nma, ngb, nmb);
      float e[8], o[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) { e[i] = 0.f; o[i] = 0.f; }
      // accumulation order = window order (p, q) ascending (fp32 sums)
      if (odd) {
        add_if(cgb, cmb, 3 + sb, e); add_if(cga, cma, 3 + sa, e);        // row 2j    : local row 1 of pooled row j
        add_if(cgb, cmb, 6 + sb, o); add_if(cga, cma, 6 + sa, o);        // row 2j + 1: local row 2 of pooled row j
        add_if(ngb, nmb, 0 + sb, o); add_if(nga, nma, 0 + sa, o);        //             local row 0 of pooled row j + 1
      } else {
        add_if(cga, cma, 3 + sa, e);
        add_if(cga, cma, 6 + sa, o);
        add_if(nga, nma, 0 + sa, o);
      }
      st8(xo, e);
      if (2 * j + 1 < g.H) st8(xo + (size_t)g.W * g.C, o);
      xo += 2 * (size_t)g.W * g.C;
      cga = nga; cgb = ngb; cma = nma; cmb = nmb;
    }
  }
}

static inline PoolSlide pool_slide_geom(int N, int H, int W, int C, int OH, int OW, int rows) {
  PoolSlide g;
  g.N = N; g.H = H; g.W = W; g.C = C; g.OH = OH; g.OW = OW;
  g.TP = rows < 14 ? rows : 14;       // 112 rows -> 56 row pairs: four chunks of 14
  return g;
}
static inline int pool_slide_grid(long long items, int cv) {
  long long b = (items + 127) / 128;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  b = (b + cv - 1) / cv * cv;
  return (int)b;
}

__global__ void __launch_bounds__(256) avgpool_fwd_kernel(const __nv_bfloat16* __restrict__ x, int N, int HW, int C,
                                                          __nv_bfloat16* __restrict__ y) {
  const int cv = C >> 3;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * cv) return;
  const int n = idx / cv, v = idx - n * cv;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const __nv_bfloat16* base = x + (long long)n * HW * C + v * 8;
  for (int i = 0; i < HW; ++i) {
    float f[8];
    ld8(base + (long long)i * C, f);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += f[j];
  }
  const float inv = 1.f / (float)HW;
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] *= inv;
  st8(y + (long long)n * C + v * 8, acc);
}

__global__ void __launch_bounds__(256) avgpool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, int N, int HW, int C,
                                                          __nv_bfloat16* __restrict__ dx) {
  const int cv = C >> 3;
  const long long total = (long long)N * HW * cv;
  const float inv = 1.f / (float)HW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % cv);
    const long long pix = idx / cv;
    const int n = (int)(pix / HW);
    float g[8];
    ld8(dy + (long long)n * C + v * 8, g);
#pragma unroll
    for (int j = 0; j < 8; ++j) g[j] *= inv;
    st8(dx + pix * C + v * 8, g);
  }
}

static inline int grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_maxpool3x3s2_fwd(const void* x, int N, int H, int W, int C, void* y, uint8_t* argmax,
                                     b200_stream_t stream) {
  B200_REQUIRE(x && y && N > 0 && H > 0 && W > 0, B200_ERR_INVALID, "maxpool_fwd: bad argument");
  B200_REQUIRE(C % 8 == 0, B200_ERR_UNSUPPORTED, "maxpool_fwd: C=%d must be a multiple of 8", C);
  B200_REQUIRE((long long)N * H * W * (C / 8) < (1LL << 31), B200_ERR_UNSUPPORTED, "maxpool_fwd: tensor too large");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const long long total = (long long)N * OH * OW * (C / 8);
  b200::launch(maxpool_fwd_kernel<false>, grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, N, H,
               W, C, OH, OW, nullptr, nullptr, 0, (__nv_bfloat16*)y, argmax);
  B200_CHECK_LAUNCH("maxpool_fwd_kernel");
  return B200_OK;
}

extern "C" int b200_bn_apply_maxpool3x3s2(const void* z, int N, int H, int W, int C, const float* scale,
                                          const float* shift, int act, void* y, uint8_t* argmax, b200_stream_t stream) {
  B200_REQUIRE(z && y && scale && shift && N > 0 && H > 0 && W > 0, B200_ERR_INVALID, "bn_apply_maxpool: bad argument");
  B200_REQUIRE(C % 8 == 0, B200_ERR_UNSUPPORTED, "bn_apply_maxpool: C=%d must be a multiple of 8", C);
  B200_REQUIRE((long long)N * H * W * (C / 8) < (1LL << 31), B200_ERR_UNSUPPORTED, "bn_apply_maxpool: tensor too large");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const long long total = (long long)N * OH * OW * (C / 8);
  b200::launch(maxpool_fwd_kernel<true>, grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)z, N, H,
               W, C, OH, OW, scale, shift, act, (__nv_bfloat16*)y, argmax);
  B200_CHECK_LAUNCH("maxpool_fwd_kernel<affine>");
  return B200_OK;
}

extern "C" int b200_maxpool3x3s2_bwd(const void* dy, const uint8_t* argmax, int N, int H, int W, int C, void* dx,
                                     b200_stream_t stream) {
  B200_REQUIRE(dy && argmax && dx && N > 0, B200_ERR_INVALID, "maxpool_bwd: bad argument");
  B200_REQUIRE(C % 8 == 0, B200_ERR_UNSUPPORTED, "maxpool_bwd: C=%d must be a multiple of 8", C);
  B200_REQUIRE((long long)N * H * W * (C / 8) < (1LL << 31), B200_ERR_UNSUPPORTED, "maxpool_bwd: tensor too large");
  const int OH = (H + 2 - 3) / 2 + 1, OW = (W + 2 - 3) / 2 + 1;
  const int J = (H + 1) / 2;
  const PoolSlide g = pool_slide_geom(N, H, W, C, OH, OW, J);
  const long long items = (long long)N * ((J + g.TP - 1) / g.TP) * W * (C / 8);
  b200::launch(maxpool_bwd_slide_kernel, pool_slide_grid(items, C / 8), 128, 0, (cudaStream_t)stream,
               (const __nv_bfloat16*)dy, argmax, g, (__nv_bfloat16*)dx);
  B200_CHECK_LAUNCH("maxpool_bwd_slide_kernel");
  return B200_OK;
}

extern "C" int b200_avgpool_fwd(const void* x, int N, int HW, int C, void* y, b200_stream_t stream) {
  B200_REQUIRE(x && y && N > 0 && HW > 0, B200_ERR_INVALID, "avgpool_fwd: bad argument");
  B200_REQUIRE(C % 8 == 0, B200_ERR_UNSUPPORTED, "avgpool_fwd: C=%d must be a multiple of 8", C);
  const int total = N * (C / 8);
  b200::launch(avgpool_fwd_kernel, (total + 255) / 256, 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)x, N, HW, C,
                                                                          (__nv_bfloat16*)y);
  B200_CHECK_LAUNCH("avgpool_fwd_kernel");
  return B200_OK;
}

extern "C" int b200_avgpool_bwd(const void* dy, int N, int HW, int C, void* dx, b200_stream_t stream) {
  B200_REQUIRE(dy && dx && N > 0 && HW > 0, B200_ERR_INVALID, "avgpool_bwd: bad argument");
  B200_REQUIRE(C % 8 == 0, B200_ERR_UNSUPPORTED, "avgpool_bwd: C=%d must be a multiple of 8", C);
  const long long total = (long long)N * HW * (C / 8);
  b200::launch(avgpool_bwd_kernel, grid_for(total, 256), 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)dy, N, HW, C,
                                                                           (__nv_bfloat16*)dx);
  B200_CHECK_LAUNCH("avgpool_bwd_kernel");
  return B200_OK;
}
