// Fused softmax cross-entropy forward + backward (one block per sample) and the bias-gradient column
// sum.  Replaces utils/cross_entropy.py:14-67 of the reference: F.cross_entropy when smooth_eps == 0
// (:20-24) and the label-smoothing formula loss = -((1-eps-eps/C)*lsm[target] + (eps/C)*sum(lsm)) (:48-52),
// reduction='mean'; and the soft-target loss of MixUp / CutMix (utils/mixup.py:37-45 with :53-54 of cross_entropy.py).
#include "common.cuh"
#include "host.h"
#include <math_constants.h>

namespace b200 {

constexpr int kCeThreads = 256;

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float other = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, other) : v + other;
  }
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  float r = sh[0];
  for (int i = 1; i < kCeThreads / 32; ++i) r = is_max ? fmaxf(r, sh[i]) : r + sh[i];
  return r;
}

// MIX: soft target q = lam*onehot(t) + (1-lam)*onehot(t2) with t2 = target[perm[b]] (MixUp / CutMix); eps is 0 then.
// A template parameter, so that the plain instantiation keeps its code.
template <bool MIX>
__global__ void __launch_bounds__(kCeThreads) softmax_ce_kernel(const float* __restrict__ logits,
                                                                const long long* __restrict__ target, int B,
                                                                int classes, int ld, float eps, float grad_scale,
                                                                const float* __restrict__ grad_scale_dev,
                                                                float* __restrict__ row_loss,
                                                                __nv_bfloat16* __restrict__ dlogits,
                                                                const long long* __restrict__ perm,
                                                                const float* __restrict__ lam_dev) {
  // row_loss layout: [0, B) per-sample loss, [B, 2B) number of classes scoring strictly above the target class
  // (rank of the target: top-1 <=> 0, top-5 <=> < 5 -- utils/meters.py:59-72 of the reference, ties aside)
  __shared__ float sh[kCeThreads / 32];
  const int b = blockIdx.x;
  const float* row = logits + (long long)b * ld;
  float mx = -CUDART_INF_F;
  for (int c = threadIdx.x; c < classes; c += kCeThreads) mx = fmaxf(mx, row[c]);
  mx = block_reduce(mx, true, sh);
  float se = 0.f, sx = 0.f;
  for (int c = threadIdx.x; c < classes; c += kCeThreads) {
    const float x = row[c];
    se += expf(x - mx);
    sx += x;
  }
  se = block_reduce(se, false, sh);
  sx = block_reduce(sx, false, sh);
  const float lse = mx + logf(se);
  const int t = (int)target[b];
  const float eps_sum = eps / (float)classes;
  const float eps_nll = 1.f - eps_sum - eps;
  const int t2 = MIX ? (int)target[perm[b]] : t;
  const float lam = MIX ? __ldg(lam_dev) : 1.f, oml = 1.f - lam;
  if (row_loss != nullptr) {
    const float xt = row[t];
    float above = 0.f;
    for (int c = threadIdx.x; c < classes; c += kCeThreads) above += (row[c] > xt) ? 1.f : 0.f;
    above = block_reduce(above, false, sh);
    if (threadIdx.x == 0) {
      // sum_c lsm[c] = sx - classes*lse
      if (MIX)
        row_loss[b] = -(lam * (xt - lse) + oml * (row[t2] - lse));
      else
        row_loss[b] = -(eps_nll * (xt - lse) + eps_sum * (sx - (float)classes * lse));
      row_loss[B + b] = above;
    }
  }
  if (dlogits != nullptr) {
    const float gs = grad_scale * (grad_scale_dev != nullptr ? __ldg(grad_scale_dev) : 1.f) / (float)B;
    // d/dx_c of li: (eps_nll + classes*eps_sum) * softmax_c - eps_nll*[c==t] - eps_sum
    const float wsm = MIX ? lam + oml : eps_nll + (float)classes * eps_sum;
    for (int c = threadIdx.x; c < classes; c += kCeThreads) {
      const float sm = expf(row[c] - lse);
      float g;
      if (MIX)
        g = wsm * sm - (c == t ? lam : 0.f) - (c == t2 ? oml : 0.f);
      else
        g = wsm * sm - eps_sum - (c == t ? eps_nll : 0.f);
      dlogits[(long long)b * ld + c] = __float2bfloat16(g * gs);
    }
    for (int c = classes + threadIdx.x; c < ld; c += kCeThreads) dlogits[(long long)b * ld + c] = __float2bfloat16(0.f);
  }
}

// loss[0] = mean_b row_loss[b], loss[1] / loss[2] = top-1 / top-5 precision in percent: one block, fixed summation
// order (bit-reproducible, no atomics, no pre-zeroed output)
__global__ void __launch_bounds__(kCeThreads) ce_mean_kernel(const float* __restrict__ row_loss, int B,
                                                             float* __restrict__ loss) {
  __shared__ float sh[kCeThreads / 32];
  float s = 0.f, t1 = 0.f, t5 = 0.f;
  for (int b = threadIdx.x; b < B; b += kCeThreads) {
    s += row_loss[b];
    const float above = row_loss[B + b];
    t1 += above < 0.5f ? 1.f : 0.f;
    t5 += above < 4.5f ? 1.f : 0.f;
  }
  s = block_reduce(s, false, sh);
  t1 = block_reduce(t1, false, sh);
  t5 = block_reduce(t5, false, sh);
  if (threadIdx.x == 0) {
    loss[0] = s / (float)B;
    loss[1] = 100.f * t1 / (float)B;
    loss[2] = 100.f * t5 / (float)B;
  }
}

__global__ void __launch_bounds__(256) colsum_bf16_kernel(const __nv_bfloat16* __restrict__ m, int B, int K,
                                                          float* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += __bfloat162float(m[(long long)b * K + k]);
  out[k] += s;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_softmax_ce(const float* logits, const long long* target, int B, int classes, int ld,
                               float smooth_eps, float grad_scale, const float* grad_scale_dev, float* loss,
                               float* row_loss, void* dlogits_bf16, b200_stream_t stream) {
  B200_REQUIRE(logits && target && B > 0 && classes > 0 && ld >= classes, B200_ERR_INVALID,
               "softmax_ce: bad argument");
  B200_REQUIRE((loss == nullptr) == (row_loss == nullptr), B200_ERR_INVALID,
               "softmax_ce: loss and row_loss must be given together");
  B200_REQUIRE(loss != nullptr || dlogits_bf16 != nullptr, B200_ERR_INVALID, "softmax_ce: nothing to compute");
  b200::launch(softmax_ce_kernel<false>, B, kCeThreads, 0, (cudaStream_t)stream, logits, target, B, classes, ld, smooth_eps,
               grad_scale, grad_scale_dev, row_loss, (__nv_bfloat16*)dlogits_bf16, (const long long*)nullptr,
               (const float*)nullptr);
  B200_CHECK_LAUNCH("softmax_ce_kernel");
  if (loss != nullptr) {
    b200::launch(ce_mean_kernel, 1, kCeThreads, 0, (cudaStream_t)stream, row_loss, B, loss);
    B200_CHECK_LAUNCH("ce_mean_kernel");
  }
  return B200_OK;
}

extern "C" int b200_softmax_ce_mix(const float* logits, const long long* target, const long long* perm,
                                   const float* lam_dev, int B, int classes, int ld, float grad_scale,
                                   const float* grad_scale_dev, float* loss, float* row_loss, void* dlogits_bf16,
                                   b200_stream_t stream) {
  B200_REQUIRE(logits && target && perm && lam_dev && B > 0 && classes > 0 && ld >= classes, B200_ERR_INVALID,
               "softmax_ce_mix: bad argument");
  B200_REQUIRE((loss == nullptr) == (row_loss == nullptr), B200_ERR_INVALID,
               "softmax_ce_mix: loss and row_loss must be given together");
  B200_REQUIRE(loss != nullptr || dlogits_bf16 != nullptr, B200_ERR_INVALID, "softmax_ce_mix: nothing to compute");
  b200::launch(softmax_ce_kernel<true>, B, kCeThreads, 0, (cudaStream_t)stream, logits, target, B, classes, ld, 0.f,
               grad_scale, grad_scale_dev, row_loss, (__nv_bfloat16*)dlogits_bf16, perm, lam_dev);
  B200_CHECK_LAUNCH("softmax_ce_kernel");
  if (loss != nullptr) {
    b200::launch(ce_mean_kernel, 1, kCeThreads, 0, (cudaStream_t)stream, row_loss, B, loss);
    B200_CHECK_LAUNCH("ce_mean_kernel");
  }
  return B200_OK;
}

extern "C" int b200_colsum_bf16(const void* m, int B, int K, float* out, b200_stream_t stream) {
  B200_REQUIRE(m && out && B > 0 && K > 0, B200_ERR_INVALID, "colsum_bf16: bad argument");
  b200::launch(colsum_bf16_kernel, (K + 255) / 256, 256, 0, (cudaStream_t)stream, (const __nv_bfloat16*)m, B, K, out);
  B200_CHECK_LAUNCH("colsum_bf16_kernel");
  return B200_OK;
}
