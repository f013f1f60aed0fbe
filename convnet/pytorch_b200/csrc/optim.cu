// Fused multi-tensor SGD over flat parameter arenas, plus the global gradient-norm machinery.
// One pass (20 B/param + 2 B bf16 shadow) replaces the reference's chain of per-tensor kernels:
//   loss-scale division          trainer.py:165-169
//   WeightDecay.pre_step         utils/regularization.py:127-131   (g += wd * p on the decayed set)
//   torch.optim.SGD.step         utils/optim.py:254-264            (m = mu*m + (1-damp)*g ; p -= lr*m)
//   fp32 master -> low precision utils/optim.py:43-47,263-264
// and clip_grad_norm_ / GradSmooth (trainer.py:171-172, utils/regularization.py:198-224) run on the
// device without the reference's per-tensor .item() host synchronisations.
#include "common.cuh"
#include "host.h"

namespace b200 {

__global__ void __launch_bounds__(256) fused_sgd_kernel(float* __restrict__ p32, const float* __restrict__ g32,
                                                        float* __restrict__ m32, __nv_bfloat16* __restrict__ p16,
                                                        long long n, long long wd_count, float lr, float momentum,
                                                        float dampening, float wd, float inv_scale,
                                                        const float* __restrict__ clip_coef, int first_step) {
  const float gs = inv_scale * (clip_coef != nullptr ? __ldg(clip_coef) : 1.f);
  const long long n4 = n >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 p = reinterpret_cast<float4*>(p32)[i];
    const float4 g4 = __ldg(reinterpret_cast<const float4*>(g32) + i);
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!first_step && momentum != 0.f) m = reinterpret_cast<float4*>(m32)[i];
    float pv[4] = {p.x, p.y, p.z, p.w}, gv[4] = {g4.x, g4.y, g4.z, g4.w}, mv[4] = {m.x, m.y, m.z, m.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float g = gv[e] * gs;
      if (i * 4 + e < wd_count) g = fmaf(wd, pv[e], g);
      float step = g;
      if (momentum != 0.f) {
        mv[e] = first_step ? g : fmaf(momentum, mv[e], (1.f - dampening) * g);
        step = mv[e];
      }
      pv[e] = fmaf(-lr, step, pv[e]);
    }
    reinterpret_cast<float4*>(p32)[i] = make_float4(pv[0], pv[1], pv[2], pv[3]);
    if (momentum != 0.f) reinterpret_cast<float4*>(m32)[i] = make_float4(mv[0], mv[1], mv[2], mv[3]);
    if (p16 != nullptr) {
      uint2 u;
      u.x = pack_bf16x2(pv[0], pv[1]);
      u.y = pack_bf16x2(pv[2], pv[3]);
      reinterpret_cast<uint2*>(p16)[i] = u;
    }
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float g = g32[i] * gs;
    float p = p32[i];
    if (i < wd_count) g = fmaf(wd, p, g);
    float step = g;
    if (momentum != 0.f) {
      const float m = first_step ? g : fmaf(momentum, m32[i], (1.f - dampening) * g);
      m32[i] = m;
      step = m;
    }
    p = fmaf(-lr, step, p);
    p32[i] = p;
    if (p16 != nullptr) p16[i] = __float2bfloat16(p);
  }
}

constexpr int kSumsqBlocks = 592;
__global__ void __launch_bounds__(256) sumsq_partial_kernel(const float* __restrict__ g, long long n,
                                                            float* __restrict__ partial) {
  __shared__ float sh[8];
  float acc = 0.f;
  const long long n4 = n >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(g) + i);
    acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    acc += g[i] * g[i];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += sh[i];
    partial[blockIdx.x] = s;
  }
}
__global__ void sumsq_final_kernel(const float* __restrict__ partial, int nb, float* out) {
  __shared__ double sh[8];
  double acc = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) acc += (double)partial[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += sh[i];
    *out = (float)s;
  }
}

__global__ void grad_coef_kernel(const float* sumsq, float inv_scale, int mode, float max_norm, float momentum,
                                 float* state, float* coef_out, float* norm_out) {
  const float norm = sqrtf(*sumsq) * inv_scale;
  float coef = 1.f;
  if (mode == 0) {
    // torch.nn.utils.clip_grad_norm_: coef = max_norm / (norm + 1e-6), clamped to 1
    coef = fminf(max_norm / (norm + 1e-6f), 1.f);
  } else {
    // GradSmooth.pre_step (utils/regularization.py:207-219)
    if (state[1] == 0.f) {
      state[0] = norm;
      state[1] = 1.f;
    } else {
      state[0] = momentum * state[0] + (1.f - momentum) * norm;
      coef = state[0] / (norm + 1e-6f);
    }
  }
  *coef_out = coef;
  if (norm_out) *norm_out = norm;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_fused_sgd(float* p32, float* g32, float* m32, void* p16, long long n, long long wd_count,
                              float lr, float momentum, float dampening, float weight_decay, float inv_scale,
                              const float* clip_coef_dev, int first_step, int zero_grad, b200_stream_t stream) {
  B200_REQUIRE(p32 && g32 && n >= 0 && (m32 || momentum == 0.f), B200_ERR_INVALID, "fused_sgd: bad argument");
  if (n == 0) return B200_OK;
  long long blocks = ((n + 3) / 4 + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  b200::launch(fused_sgd_kernel, (int)blocks, 256, 0, (cudaStream_t)stream, p32, (const float*)g32, m32, (__nv_bfloat16*)p16, n,
               wd_count, lr, momentum, dampening, weight_decay, inv_scale, clip_coef_dev, first_step);
  B200_CHECK_LAUNCH("fused_sgd_kernel");
  if (zero_grad) {
    // the next step's zero_grad(): a memset node behind the update.  Clearing the gradient inside the kernel (a 16-byte
    // store to the line just loaded) was measured 4.5x SLOWER than the whole update (440 vs 98 us on 25.6 M parameters;
    // tools/sgd_bench.py); kernel + memset is 116 us.
    cudaError_t e = cudaMemsetAsync(g32, 0, (size_t)n * sizeof(float), (cudaStream_t)stream);
    B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "fused_sgd: memset of the gradient arena failed: %s", cudaGetErrorString(e));
  }
  return B200_OK;
}

extern "C" int b200_sumsq(const float* g, long long n, float* out, float* workspace, b200_stream_t stream) {
  B200_REQUIRE(g && out && workspace && n > 0, B200_ERR_INVALID, "sumsq: bad argument");
  long long blocks = ((n + 3) / 4 + 255) / 256;
  if (blocks > kSumsqBlocks) blocks = kSumsqBlocks;
  b200::launch(sumsq_partial_kernel, (int)blocks, 256, 0, (cudaStream_t)stream, g, n, workspace);
  B200_CHECK_LAUNCH("sumsq_partial_kernel");
  b200::launch(sumsq_final_kernel, 1, 256, 0, (cudaStream_t)stream, workspace, (int)blocks, out);
  B200_CHECK_LAUNCH("sumsq_final_kernel");
  return B200_OK;
}

extern "C" int b200_grad_coef(const float* sumsq, float inv_scale, int mode, float max_norm, float momentum,
                              float* state, float* coef_out, float* norm_out, b200_stream_t stream) {
  B200_REQUIRE(sumsq && coef_out && (mode == 0 || state), B200_ERR_INVALID, "grad_coef: bad argument");
  b200::launch(grad_coef_kernel, 1, 1, 0, (cudaStream_t)stream, sumsq, inv_scale, mode, max_norm, momentum, state, coef_out,
                                                     norm_out);
  B200_CHECK_LAUNCH("grad_coef_kernel");
  return B200_OK;
}
