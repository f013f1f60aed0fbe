// Batch-norm statistics / apply / backward for NHWC bf16 activations: HBM-bound, 128-bit vectorised,
// ReLU/ReLU6 and the residual add fused.  Replaces nn.BatchNorm2d (+ nn.ReLU, + `out += residual`) of the
// reference (models/resnet.py:88-91,115-116,128-134,162-163; models/mobilenet_v2.py:50-63), train and eval.
//
// Thread mapping shared by all kernels: a block owns a contiguous range of rows (pixels); thread t is
// (row_in_iter = t / cv, vec = t % cv) with cv = C/8 channel vectors, so every iteration of a block touches
// one contiguous span of memory and per-channel coefficients are loaded once per thread.
//
// Forward statistics normally come from the convolution epilogue (fp64 atomics into 16 replica rows of the
// workspace, finished by bn_finalize_kernel); bn_stats_kernel is the stand-alone version for outputs the conv kernel
// cannot cover (single kernel: the last block, elected by a ticket counter, finalises and re-zeroes the
// accumulators).  The backward reduction writes one partial row per block and a second tiny kernel sums them in a
// fixed order (no atomics: same-address fp64 atomics at the end of ~600 blocks cost more than the extra launch).
// The workspace must be zero before first use and must not be shared by concurrent streams.
#include "bn_common.cuh"

namespace b200 {

static inline int reduce_blocks(long long M, int C, const RowMap& rm, int resident_per_sm = 6) {
  long long iters = (M + rm.rows_per_iter - 1) / rm.rows_per_iter;
  long long want = (iters + 7) / 8;          // >= 8 row-iterations per block
  long long cap = 1200000LL / (2 * C);       // bound the number of fp64 atomics (blocks * 2C)
  if (cap < sm_count()) cap = sm_count();
  // one full wave of fat blocks, no tail wave
  if (cap > resident_per_sm * sm_count()) cap = resident_per_sm * sm_count();
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  return (int)want;
}
// Block partials -> fp64 global accumulators; returns true in the LAST block of the grid (after a grid-wide
// happens-before: every other block's atomics are visible).
__device__ __forceinline__ bool accumulate_and_elect(float (&acc)[16], int cv, int rows_per_iter, int C,
                                                     double* accum, unsigned* ticket) {
  __shared__ float red[kBnThreads][17];
  __shared__ bool is_last;
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 16; ++i) red[t][i] = acc[i];
  __syncthreads();
  for (int o = t; o < 2 * C; o += kBnThreads) {
    const int stat = o / C;
    const int c = o - stat * C;
    const int v = c >> 3, e = c & 7;
    float s = 0.f;
    for (int r = 0; r < rows_per_iter; ++r) s += red[r * cv + v][stat * 8 + e];
    atomicAdd(accum + (blockIdx.x % kReplicas) * 2 * C + o, (double)s);
  }
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (is_last) __threadfence();
  return is_last;
}

// ---- forward statistics -------------------------------------------------------------------------
__global__ void __launch_bounds__(kBnThreads) bn_stats_kernel(
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter,
    const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum, float* running_mean,
    float* running_var, long long* num_batches_tracked, float* mean, float* invstd, float* scale, float* shift,
    double* accum, unsigned* ticket) {
  const int t = threadIdx.x;
  const bool active = t < rows_per_iter * cv;
  const int r0 = t / cv, v = t - r0 * cv;
  const long long rows_per_block = (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  float acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;
  if (active) {
    long long r = row_begin + r0;
    for (; r + 7LL * rows_per_iter < row_end; r += 8LL * rows_per_iter) {
      uint4 raw[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        raw[u] = *reinterpret_cast<const uint4*>(z + (r + (long long)u * rows_per_iter) * C + v * 8);
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        float f[8];
        unpack8(raw[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) { acc[i] += f[i]; acc[8 + i] += f[i] * f[i]; }
      }
    }
    for (; r < row_end; r += rows_per_iter) {
      float f[8];
      load8(z + r * C + v * 8, f);
#pragma unroll
      for (int i = 0; i < 8; ++i) { acc[i] += f[i]; acc[8 + i] += f[i] * f[i]; }
    }
  }
  if (!accumulate_and_elect(acc, cv, rows_per_iter, C, accum, ticket)) return;
  // ---- last block: finalise ----
  float f = momentum;
  if (momentum < 0.f) {  // cumulative moving average (momentum=None): factor 1/(num_batches_tracked+1)
    const long long nbt = num_batches_tracked ? *num_batches_tracked : 0;
    f = 1.f / (float)(nbt + 1);
  }
  for (int c = t; c < C; c += kBnThreads) {
    double s1 = 0.0, s2 = 0.0;
    for (int rep = 0; rep < kReplicas; ++rep) {
      s1 += __ldcg(accum + rep * 2 * C + c);
      s2 += __ldcg(accum + rep * 2 * C + C + c);
      accum[rep * 2 * C + c] = 0.0;
      accum[rep * 2 * C + C + c] = 0.0;
    }
    const double mu = s1 / (double)M;
    double var = s2 / (double)M - mu * mu;
    if (var < 0.0) var = 0.0;
    const float istd = (float)(1.0 / sqrt(var + (double)eps));
    mean[c] = (float)mu;
    invstd[c] = istd;
    const float g = gamma ? gamma[c] : 1.f, bt = beta ? beta[c] : 0.f;
    const float sc = g * istd;
    scale[c] = sc;
    shift[c] = bt - (float)mu * sc;
    if (running_mean != nullptr && running_var != nullptr) {
      const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
      running_mean[c] = (1.f - f) * running_mean[c] + f * (float)mu;
      running_var[c] = (1.f - f) * running_var[c] + f * (float)unbiased;
    }
  }
  __syncthreads();
  if (t == 0) {
    *ticket = 0u;
    if (num_batches_tracked != nullptr && running_mean != nullptr) *num_batches_tracked += 1;
  }
}

// finalisation of statistics accumulated elsewhere (conv epilogue): same math as the last block of bn_stats_kernel
__global__ void __launch_bounds__(kBnThreads) bn_finalize_kernel(
    long long M, int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
    float* running_mean, float* running_var, long long* num_batches_tracked, float* mean, float* invstd, float* scale,
    float* shift, double* accum) {
  // 16 lanes per channel, one per accumulator replica (a serial loop over the replicas was a chain of L2 round
  // trips in a kernel that sits on the critical path between the convolution and the BN apply)
  static_assert(kReplicas == 16, "lane mapping below assumes 16 replicas");
  const int rep = threadIdx.x & 15;
  const int c = blockIdx.x * (kBnThreads / 16) + (threadIdx.x >> 4);
  float f = momentum;
  if (momentum < 0.f) {
    const long long nbt = num_batches_tracked ? *num_batches_tracked : 0;
    f = 1.f / (float)(nbt + 1);
  }
  double s1 = 0.0, s2 = 0.0;
  if (c < C) {
    s1 = accum[rep * 2 * C + c];
    s2 = accum[rep * 2 * C + C + c];
    accum[rep * 2 * C + c] = 0.0;
    accum[rep * 2 * C + C + c] = 0.0;
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if (c < C && rep == 0) {
    const double mu = s1 / (double)M;
    double var = s2 / (double)M - mu * mu;
    if (var < 0.0) var = 0.0;
    const float istd = (float)(1.0 / sqrt(var + (double)eps));
    mean[c] = (float)mu;
    invstd[c] = istd;
    const float g = gamma ? gamma[c] : 1.f, bt = beta ? beta[c] : 0.f;
    const float sc = g * istd;
    scale[c] = sc;
    shift[c] = bt - (float)mu * sc;
    if (running_mean != nullptr && running_var != nullptr) {
      const double unbiased = M > 1 ? var * (double)M / (double)(M - 1) : var;
      running_mean[c] = (1.f - f) * running_mean[c] + f * (float)mu;
      running_var[c] = (1.f - f) * running_var[c] + f * (float)unbiased;
    }
  }
  // with a fixed momentum nobody reads the counter, so it can be bumped here; the cumulative mode (momentum < 0)
  // reads it in every block above and gets a separate, stream-ordered bump kernel instead
  if (momentum >= 0.f && blockIdx.x == 0 && threadIdx.x == 0 && num_batches_tracked != nullptr && running_mean != nullptr)
    *num_batches_tracked += 1;
}
__global__ void bn_bump_kernel(long long* nbt) {
  *nbt += 1;
}

__global__ void bn_eval_coeffs_kernel(int C, const float* gamma, const float* beta, const float* rm, const float* rv,
                                      float eps, float* scale, float* shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float istd = rsqrtf(rv[c] + eps);
  const float sc = (gamma ? gamma[c] : 1.f) * istd;
  scale[c] = sc;
  shift[c] = (beta ? beta[c] : 0.f) - rm[c] * sc;
}

// ---- forward apply ------------------------------------------------------------------------------
template <int MODE>  // 0: none, 1: + residual, 2: + (z2*scale2+shift2)
__global__ void __launch_bounds__(kBnThreads) bn_apply_kernel(
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter,
    const float* __restrict__ scale, const float* __restrict__ shift, const __nv_bfloat16* __restrict__ res,
    const float* __restrict__ scale2, const float* __restrict__ shift2, int act, __nv_bfloat16* __restrict__ y,
    uint8_t* __restrict__ act_mask) {
  const int t = threadIdx.x;
  if (t >= rows_per_iter * cv) return;
  const int r0 = t / cv, v = t - r0 * cv;
  const long long rows_per_block = (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  float sc[8], sh[8], sc2[8], sh2[8];
  loadf8(scale + v * 8, sc);
  loadf8(shift + v * 8, sh);
  if (MODE == 2) { loadf8(scale2 + v * 8, sc2); loadf8(shift2 + v * 8, sh2); }
  for (long long r = row_begin + r0; r < row_end; r += 2LL * rows_per_iter) {
    const long long ra = r, rb = r + rows_per_iter;
    const bool hb = rb < row_end;
    float fa[8], fb[8], ga[8], gb[8];
    uint32_t ma = 0, mb = 0;
    load8(z + ra * C + v * 8, fa);
    if (hb) load8(z + rb * C + v * 8, fb);
    if (MODE != 0) {
      load8(res + ra * C + v * 8, ga);
      if (hb) load8(res + rb * C + v * 8, gb);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float a = fa[i] * sc[i] + sh[i];
      float b = hb ? fb[i] * sc[i] + sh[i] : 0.f;
      if (MODE == 1) { a += ga[i]; if (hb) b += gb[i]; }
      if (MODE == 2) { a += ga[i] * sc2[i] + sh2[i]; if (hb) b += gb[i] * sc2[i] + sh2[i]; }
      ma |= static_cast<uint32_t>(act_mask_value(a, act)) << i;
      mb |= static_cast<uint32_t>(act_mask_value(b, act)) << i;
      if (act == B200_ACT_RELU) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
      if (act == B200_ACT_RELU6) { a = fminf(fmaxf(a, 0.f), 6.f); b = fminf(fmaxf(b, 0.f), 6.f); }
      fa[i] = a; fb[i] = b;
    }
    store8(y + ra * C + v * 8, fa);
    if (hb) store8(y + rb * C + v * 8, fb);
    if (act_mask != nullptr) {   // one byte per (row, 8-channel vector): bit i = act'(.) of channel v*8+i
      act_mask[mask_byte_index(ra, cv, v)] = static_cast<uint8_t>(ma);
      if (hb) act_mask[mask_byte_index(rb, cv, v)] = static_cast<uint8_t>(mb);
    }
  }
}

// ---- backward kernels (bodies in bn_common.cuh) --------------------------------------------------
// backward reduce: dbeta = sum g, dgamma = sum g * xhat
// SRC: activation argument 0 recomputed from z, 1 = y, 2 = mask bits
template <int VEC, int ROWS, int MINB, int SRC>
__global__ void __launch_bounds__(kBnThreads, MINB) bn_bwd_reduce_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ amask,
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter, int act,
    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
    const float* __restrict__ beta, float* __restrict__ partial) {
  bn_bwd_reduce_body<VEC, ROWS, SRC>(dy, y, amask, z, M, C, cv, rows_per_iter, act, mean, invstd, gamma, beta,
                                     partial, 1.f);
}

// second stage: sums[o] = sum over blocks of partial[b][o]  (o in [0, 2C): dgamma then dbeta); a block of 256
// threads owns 4 outputs x 64 interleaved block groups (every load independent: the kernel is pure latency),
// fp64 across the groups.
__global__ void __launch_bounds__(kBnThreads) bn_bwd_reduce_final_kernel(const float* __restrict__ partial, int nblocks,
                                                                          int C, float* __restrict__ sums,
                                                                          float* dgamma_acc, float* dbeta_acc) {
  __shared__ double red[64][5];
  const int lane_o = threadIdx.x & 3, grp = threadIdx.x >> 2;
  const int o = blockIdx.x * 4 + lane_o;
  double acc = 0.0;
  if (o < 2 * C) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int b = grp;
    for (; b + 192 < nblocks; b += 256) {
      a0 += __ldcg(partial + (size_t)b * 2 * C + o);
      a1 += __ldcg(partial + (size_t)(b + 64) * 2 * C + o);
      a2 += __ldcg(partial + (size_t)(b + 128) * 2 * C + o);
      a3 += __ldcg(partial + (size_t)(b + 192) * 2 * C + o);
    }
    for (; b < nblocks; b += 64) a0 += __ldcg(partial + (size_t)b * 2 * C + o);
    acc = (double)a0 + (double)a1 + (double)a2 + (double)a3;
  }
  red[grp][lane_o] = acc;
  __syncthreads();
  if (grp == 0 && o < 2 * C) {
    double tot = 0.0;
#pragma unroll 8
    for (int g = 0; g < 64; ++g) tot += red[g][lane_o];
    const float f = (float)tot;
    sums[o] = f;
    if (o < C) { if (dgamma_acc) dgamma_acc[o] += f; }
    else if (dbeta_acc) dbeta_acc[o - C] += f;
  }
}
void launch_bwd_reduce_final(const float* partial, int nblocks, int C, float* sums, float* dgamma_acc,
                             float* dbeta_acc, cudaStream_t stream) {
  b200::launch(bn_bwd_reduce_final_kernel, (2 * C + 3) / 4, kBnThreads, 0, stream, partial, nblocks, C, sums, dgamma_acc,
                                                                           dbeta_acc);
}

// ---- backward dx --------------------------------------------------------------------------------
template <int VEC, int ROWS, int MINB, int SRC>   // SRC as in bn_bwd_reduce_kernel
__global__ void __launch_bounds__(kBnThreads, MINB) bn_bwd_dx_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ amask,
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter, int act,
    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
    const float* __restrict__ beta, const float* __restrict__ sums, __nv_bfloat16* __restrict__ dz,
    __nv_bfloat16* __restrict__ g_out) {
  bn_bwd_dx_body<VEC, ROWS, SRC>(dy, y, amask, z, M, C, cv, rows_per_iter, act, mean, invstd, gamma, beta, sums, dz,
                                 g_out, 1.f);
}

static inline double* ws_accum(float* ws) { return reinterpret_cast<double*>(ws); }
static inline unsigned* ws_ticket(float* ws) { return reinterpret_cast<unsigned*>(ws + kReplicas * 2 * kBnMaxC * 2); }

}  // namespace b200

using namespace b200;

extern "C" size_t b200_bn_workspace_floats(int C) { (void)C; return (size_t)kWsFloats; }
// rows padded to a multiple of 8: the backward kernels read whole row-quad words (two of them with 8 rows in flight)
extern "C" size_t b200_bn_act_mask_bytes(long long M, int C) { return (size_t)((M + 7) / 8 * 8) * (size_t)(C / 8); }

extern "C" int b200_bn_stats(const void* z, long long M, int C, const float* gamma, const float* beta, float eps,
                             float momentum, float* running_mean, float* running_var, long long* nbt, float* mean,
                             float* invstd, float* scale, float* shift, float* workspace, b200_stream_t stream_) {
  int rc = check_c(C, "bn_stats");
  if (rc) return rc;
  B200_REQUIRE(z && mean && invstd && scale && shift && workspace && M > 0, B200_ERR_INVALID, "bn_stats: bad argument");
  B200_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, B200_ERR_INVALID, "bn_stats: workspace misaligned");
  const RowMap rm = make_rowmap(C);
  b200::launch(bn_stats_kernel, reduce_blocks(M, C, rm), kBnThreads, 0, (cudaStream_t)stream_,
      (const __nv_bfloat16*)z, M, C, rm.cv, rm.rows_per_iter, gamma, beta, eps, momentum, running_mean, running_var,
      nbt, mean, invstd, scale, shift, ws_accum(workspace), ws_ticket(workspace));
  B200_CHECK_LAUNCH("bn_stats_kernel");
  return B200_OK;
}

extern "C" int b200_bn_finalize(long long M, int C, const float* gamma, const float* beta, float eps, float momentum,
                                float* running_mean, float* running_var, long long* nbt, float* mean, float* invstd,
                                float* scale, float* shift, float* workspace, b200_stream_t stream_) {
  int rc = check_c(C, "bn_finalize");
  if (rc) return rc;
  B200_REQUIRE(mean && invstd && scale && shift && workspace && M > 0, B200_ERR_INVALID, "bn_finalize: bad argument");
  cudaStream_t stream = (cudaStream_t)stream_;
  // NOTE: momentum < 0 reads *nbt before the bump below (same stream => ordered)
  b200::launch(bn_finalize_kernel, (C + 15) / 16, kBnThreads, 0, stream,
      M, C, gamma, beta, eps, momentum, running_mean, running_var, nbt, mean, invstd, scale, shift, ws_accum(workspace));
  B200_CHECK_LAUNCH("bn_finalize_kernel");
  if (momentum < 0.f && nbt != nullptr && running_mean != nullptr) {
    b200::launch(bn_bump_kernel, 1, 1, 0, stream, nbt);
    B200_CHECK_LAUNCH("bn_bump_kernel");
  }
  return B200_OK;
}

extern "C" int b200_bn_eval_coeffs(int C, const float* gamma, const float* beta, const float* running_mean,
                                   const float* running_var, float eps, float* scale, float* shift,
                                   b200_stream_t stream_) {
  B200_REQUIRE(C > 0 && running_mean && running_var && scale && shift, B200_ERR_INVALID, "bn_eval_coeffs: bad argument");
  b200::launch(bn_eval_coeffs_kernel, (C + 127) / 128, 128, 0, (cudaStream_t)stream_, C, gamma, beta, running_mean, running_var,
                                                                         eps, scale, shift);
  B200_CHECK_LAUNCH("bn_eval_coeffs_kernel");
  return B200_OK;
}

extern "C" int b200_bn_apply(const void* z, long long M, int C, const float* scale, const float* shift,
                             const void* residual, const void* z2, const float* scale2, const float* shift2, int act,
                             void* y, uint8_t* act_mask, b200_stream_t stream_) {
  int rc = check_c(C, "bn_apply");
  if (rc) return rc;
  B200_REQUIRE(z && scale && shift && y && M > 0, B200_ERR_INVALID, "bn_apply: bad argument");
  B200_REQUIRE(!(residual && z2), B200_ERR_INVALID, "bn_apply: residual and z2 are exclusive");
  B200_REQUIRE(!z2 || (scale2 && shift2), B200_ERR_INVALID, "bn_apply: z2 needs scale2/shift2");
  cudaStream_t stream = (cudaStream_t)stream_;
  const RowMap rm = make_rowmap(C);
  const int blocks = stream_blocks(M, rm);
  const __nv_bfloat16* zz = (const __nv_bfloat16*)z;
  __nv_bfloat16* yy = (__nv_bfloat16*)y;
  if (residual)
    b200::launch(bn_apply_kernel<1>, blocks, kBnThreads, 0, stream, zz, M, C, rm.cv, rm.rows_per_iter, scale, shift,
                                                         (const __nv_bfloat16*)residual, nullptr, nullptr, act, yy, act_mask);
  else if (z2)
    b200::launch(bn_apply_kernel<2>, blocks, kBnThreads, 0, stream, zz, M, C, rm.cv, rm.rows_per_iter, scale, shift,
                                                         (const __nv_bfloat16*)z2, scale2, shift2, act, yy, act_mask);
  else
    b200::launch(bn_apply_kernel<0>, blocks, kBnThreads, 0, stream, zz, M, C, rm.cv, rm.rows_per_iter, scale, shift, nullptr,
                                                         nullptr, nullptr, act, yy, act_mask);
  B200_CHECK_LAUNCH("bn_apply_kernel");
  return B200_OK;
}

// Launch shape of the backward kernels (VEC channels per thread, ROWS rows in flight per thread, MINB resident blocks
// per SM): (4, 4, 4) up to C = 1024, (8, 2, 3) above.
extern "C" int b200_bn_bwd_reduce(const void* dy, const void* y, const uint8_t* act_mask, const void* z, long long M,
                                  int C, int act,
                                  const float* mean, const float* invstd, const float* gamma, const float* beta,
                                  float* sums, float* dgamma_acc, float* dbeta_acc, float* workspace,
                                  b200_stream_t stream_) {
  int rc = check_c(C, "bn_bwd_reduce");
  if (rc) return rc;
  B200_REQUIRE(dy && z && mean && invstd && sums && workspace && M > 0, B200_ERR_INVALID, "bn_bwd_reduce: bad argument");
  // activation-argument source: 2 = mask bits, 1 = y, 0 = recomputed from z (or no activation)
  const int src = (act == B200_ACT_NONE) ? 0 : (act_mask != nullptr ? 2 : (y != nullptr ? 1 : 0));
#define B200_RED_ARGS(VEC)                                                                                     \
  (const __nv_bfloat16*)dy, (const __nv_bfloat16*)y, act_mask, (const __nv_bfloat16*)z, M, C, rm.cv,           \
      rm.rows_per_iter, act, mean, invstd, gamma, beta, partial
#define B200_LAUNCH_RED(VEC, ROWS, MINB)                                                                       \
  do {                                                                                                         \
    const RowMap rm = make_rowmap_v<VEC>(C);                                                                   \
    blocks = partial_blocks(M, rm, MINB);                                                                      \
    if (src == 2)                                                                                              \
      b200::launch(bn_bwd_reduce_kernel<VEC, ROWS, MINB, 2>, blocks, kBnThreads, 0, stream, B200_RED_ARGS(VEC));         \
    else if (src == 1)                                                                                         \
      b200::launch(bn_bwd_reduce_kernel<VEC, ROWS, MINB, 1>, blocks, kBnThreads, 0, stream, B200_RED_ARGS(VEC));         \
    else                                                                                                       \
      b200::launch(bn_bwd_reduce_kernel<VEC, ROWS, MINB, 0>, blocks, kBnThreads, 0, stream, B200_RED_ARGS(VEC));         \
  } while (0)
  cudaStream_t stream = (cudaStream_t)stream_;
  float* partial = workspace + kAccumFloats;
  int blocks = 0;
  if (C > 1024)
    B200_LAUNCH_RED(8, 2, 3);
  else
    B200_LAUNCH_RED(4, 4, 4);
#undef B200_LAUNCH_RED
#undef B200_RED_ARGS
  B200_CHECK_LAUNCH("bn_bwd_reduce_kernel");
  launch_bwd_reduce_final(partial, blocks, C, sums, dgamma_acc, dbeta_acc, stream);
  B200_CHECK_LAUNCH("bn_bwd_reduce_final_kernel");
  return B200_OK;
}

extern "C" int b200_bn_bwd_dx(const void* dy, const void* y, const uint8_t* act_mask, const void* z, long long M, int C,
                              int act,
                              const float* mean, const float* invstd, const float* gamma, const float* beta,
                              const float* sums, void* dz, void* g_out, b200_stream_t stream_) {
  int rc = check_c(C, "bn_bwd_dx");
  if (rc) return rc;
  B200_REQUIRE(dy && z && mean && invstd && sums && dz && M > 0, B200_ERR_INVALID, "bn_bwd_dx: bad argument");
  const int src = (act == B200_ACT_NONE) ? 0 : (act_mask != nullptr ? 2 : (y != nullptr ? 1 : 0));
#define B200_DX_ARGS(VEC)                                                                                    \
  (const __nv_bfloat16*)dy, (const __nv_bfloat16*)y, act_mask, (const __nv_bfloat16*)z, M, C, rm.cv,         \
      rm.rows_per_iter, act, mean, invstd, gamma, beta, sums, (__nv_bfloat16*)dz, (__nv_bfloat16*)g_out
#define B200_LAUNCH_DX(VEC, ROWS, MINB)                                                                      \
  do {                                                                                                       \
    const RowMap rm = make_rowmap_v<VEC>(C);                                                                 \
    const int blocks = stream_blocks(M, rm);                                                                 \
    if (src == 2)                                                                                            \
      b200::launch(bn_bwd_dx_kernel<VEC, ROWS, MINB, 2>, blocks, kBnThreads, 0, (cudaStream_t)stream_, B200_DX_ARGS(VEC)); \
    else if (src == 1)                                                                                       \
      b200::launch(bn_bwd_dx_kernel<VEC, ROWS, MINB, 1>, blocks, kBnThreads, 0, (cudaStream_t)stream_, B200_DX_ARGS(VEC)); \
    else                                                                                                     \
      b200::launch(bn_bwd_dx_kernel<VEC, ROWS, MINB, 0>, blocks, kBnThreads, 0, (cudaStream_t)stream_, B200_DX_ARGS(VEC)); \
  } while (0)
  if (C > 1024)
    B200_LAUNCH_DX(8, 2, 3);
  else
    B200_LAUNCH_DX(4, 4, 4);
#undef B200_LAUNCH_DX
#undef B200_DX_ARGS
  B200_CHECK_LAUNCH("bn_bwd_dx_kernel");
  return B200_OK;
}
