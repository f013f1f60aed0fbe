// L1 batch normalization ("Norm matters", Hoffer et al. 2018) for NHWC bf16 activations: the statistics, eval
// coefficients and input-gradient kernels that differ from the variance BatchNorm of bn.cu.  Replaces the reference's
// L1BatchNorm2d (models/modules/lp_norm.py:238-291), selected by resnet(bn_norm='L1').  Per channel, with M rows:
//   mu = mean(z),  L = mean|z - mu|,  s = 1 / (L * sqrt(pi/2) + eps),  y = (z - mu) * s * gamma + beta.
// The apply and the backward reduction are bn.cu's: b200_bn_apply takes scale/shift, and b200_bn_bwd_reduce called
// with invstd = s returns sums = {sum g*(z-mu)*s, sum g} (= dgamma, dbeta).  Only the input gradient differs:
//   dz = gamma*s*(g - sum g/M) - gamma*s^2*sqrt(pi/2) * (sum g*(z-mu)/M) * (sign(z-mu) - S/M),  S = sum sign(z-mu)
// with sign(0) = 0, as torch's abs backward.
//
// Statistics take two reads of z: one for mu, one for sum|z-mu| and S.  Each read writes one partial row per block
// into the BN workspace (after the fp64 accumulators, which stay untouched and zero), and a second kernel sums the
// rows in a fixed order in fp64: no atomics, so repeated calls are bitwise identical.
#include "bn_common.cuh"

namespace b200 {

constexpr float kL1Fix = 1.2533141373155003f;   // sqrt(pi/2): E|x - mu| = sigma * sqrt(2/pi) for a normal x
constexpr double kL1FixD = 1.2533141373155003;

// ---- statistics, first stage: per-block partial row ---------------------------------------------------
// PASS 0: partial[b][c] = sum z.  PASS 1: partial[b][c] = sum |z - mu|, partial[b][C + c] = sum sign(z - mu).
template <int PASS>
__global__ void __launch_bounds__(kBnThreads) bn_l1_partial_kernel(const __nv_bfloat16* __restrict__ z, long long M,
                                                                   int C, int cv, int rows_per_iter,
                                                                   const float* __restrict__ mean,
                                                                   float* __restrict__ partial) {
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
    float mu[8];
    if (PASS == 1) loadf8(mean + v * 8, mu);
    long long r = row_begin + r0;
    for (; r < row_end; r += 4LL * rows_per_iter) {
      uint4 raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long rr = r + (long long)u * rows_per_iter;
        if (rr < row_end) raw[u] = ld_stream(z + rr * C + v * 8);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (r + (long long)u * rows_per_iter >= row_end) continue;
        float f[8];
        unpack8(raw[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (PASS == 0) {
            acc[i] += f[i];
          } else {
            const float d = f[i] - mu[i];
            acc[i] += fabsf(d);
            acc[8 + i] += (d > 0.f ? 1.f : 0.f) - (d < 0.f ? 1.f : 0.f);
          }
        }
      }
    }
  }
  __shared__ float red[kBnThreads][17];
#pragma unroll
  for (int i = 0; i < 16; ++i) red[t][i] = acc[i];
  __syncthreads();
  const int nout = PASS == 0 ? C : 2 * C;
  float* dst = partial + (size_t)blockIdx.x * 2 * C;
  for (int o = t; o < nout; o += kBnThreads) {
    const int stat = o / C;
    const int c = o - stat * C;
    const int vv = c >> 3, e = c & 7;
    float s = 0.f;
    for (int r = 0; r < rows_per_iter; ++r) s += red[r * cv + vv][stat * 8 + e];
    dst[o] = s;
  }
}

// ---- statistics, second stage: fixed-order fp64 sum of the partial rows, then the per-channel results ----------
// A block owns 4 channels x 64 interleaved block groups.  PASS 0 writes mean.  PASS 1 writes invstd = s, the sign sum
// S, scale/shift (the fp32 expressions of bn.cu's finalisation, so that bn_apply and the activation mask recomputed
// from z in the backward kernels agree bit for bit) and updates the running buffers with the reference's convention:
// running = running * momentum + batch * (1 - momentum), running_var holding s.
template <int PASS>
__global__ void __launch_bounds__(kBnThreads) bn_l1_final_kernel(
    const float* __restrict__ partial, int nblocks, long long M, int C, const float* __restrict__ gamma,
    const float* __restrict__ beta, float eps, float momentum, float* running_mean, float* running_var, float* mean,
    float* invstd, float* sign_sum, float* scale, float* shift) {
  __shared__ double red[64][4][2];
  const int lane_c = threadIdx.x & 3, grp = threadIdx.x >> 2;
  const int c = blockIdx.x * 4 + lane_c;
  double a0 = 0.0, a1 = 0.0;
  if (c < C) {
    for (int b = grp; b < nblocks; b += 64) {
      a0 += (double)__ldcg(partial + (size_t)b * 2 * C + c);
      if (PASS == 1) a1 += (double)__ldcg(partial + (size_t)b * 2 * C + C + c);
    }
  }
  red[grp][lane_c][0] = a0;
  red[grp][lane_c][1] = a1;
  __syncthreads();
  if (grp != 0 || c >= C) return;
  double s0 = 0.0, s1 = 0.0;
  for (int g = 0; g < 64; ++g) {
    s0 += red[g][lane_c][0];
    s1 += red[g][lane_c][1];
  }
  if (PASS == 0) {
    mean[c] = (float)(s0 / (double)M);
    return;
  }
  const float mu = mean[c];
  // explicit roundings (no fused multiply-add): the value is reproducible from the sums on any IEEE fp64 host
  const float istd = (float)(1.0 / __dadd_rn(__dmul_rn(s0 / (double)M, kL1FixD), (double)eps));
  invstd[c] = istd;
  sign_sum[c] = (float)s1;
  const float g = gamma ? gamma[c] : 1.f, bt = beta ? beta[c] : 0.f;
  const float sc = g * istd;
  scale[c] = sc;
  shift[c] = bt - mu * sc;
  if (running_mean != nullptr && running_var != nullptr) {
    const float keep = 1.f - momentum;
    running_mean[c] = __fadd_rn(__fmul_rn(running_mean[c], momentum), __fmul_rn(mu, keep));
    running_var[c] = __fadd_rn(__fmul_rn(running_var[c], momentum), __fmul_rn(istd, keep));
  }
}

// eval mode: y = (z - running_mean) * running_var * gamma + beta (running_var holds the scale s)
__global__ void bn_l1_eval_coeffs_kernel(int C, const float* gamma, const float* beta, const float* rm, const float* rv,
                                         float* scale, float* shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float sc = (gamma ? gamma[c] : 1.f) * rv[c];
  scale[c] = sc;
  shift[c] = (beta ? beta[c] : 0.f) - rm[c] * sc;
}

// ---- backward dx: dz = A*g + B*sign(z - mean) + Cc ------------------------------------------------------------
// Thread mapping, launch shapes, activation sources (SRC 0: recomputed from z, 1: y, 2: mask bits) and the +0
// selection of masked gradients are those of bn.cu's bn_bwd_dx_kernel.  sums = {sum g*(z-mu)*s, sum g} from
// b200_bn_bwd_reduce with invstd = s:  A = gamma*s, B = -A*sqrt(pi/2)*sums[0]/M, Cc = -A*sums[1]/M - B*S/M.
template <int VEC, int ROWS, int MINB, int SRC>
__global__ void __launch_bounds__(kBnThreads, MINB) bn_l1_bwd_dx_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ amask,
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter, int act,
    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ sign_sum,
    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ sums,
    __nv_bfloat16* __restrict__ dz, __nv_bfloat16* __restrict__ g_out) {
  const int t = threadIdx.x;
  if (t >= rows_per_iter * cv) return;
  const int r0 = t / cv, v = t - r0 * cv;
  const long long rows_per_block = SRC == 2 ? (((M + gridDim.x - 1) / gridDim.x + 7) & ~7LL) : (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  constexpr long long kRowStep = SRC == 2 ? 1 : 0;
  float A[VEC], B[VEC], Cc[VEC], sh[VEC], mu[VEC];
  {
    float is[VEC], dg[VEC], dbt[VEC], ss[VEC];
    loadfv<VEC>(mean + v * VEC, mu);
    loadfv<VEC>(invstd + v * VEC, is);
    loadfv<VEC>(sign_sum + v * VEC, ss);
    if (gamma) loadfv<VEC>(gamma + v * VEC, A);
    if (beta) loadfv<VEC>(beta + v * VEC, sh);
    loadfv<VEC>(sums + v * VEC, dg);
    loadfv<VEC>(sums + C + v * VEC, dbt);
    const float invM = 1.f / (float)M;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float gm = gamma ? A[i] : 1.f;
      A[i] = gm * is[i];
      B[i] = -A[i] * kL1Fix * dg[i] * invM;
      Cc[i] = -A[i] * dbt[i] * invM - B[i] * ss[i] * invM;
      sh[i] = (beta ? sh[i] : 0.f) - mu[i] * A[i];
    }
  }
  const long long col = (long long)v * VEC;
  const long long rstep = kRowStep ? 1 : rows_per_iter;
  for (long long r = row_begin + (kRowStep ? (long long)r0 * ROWS : r0); r < row_end;
       r += (long long)ROWS * rows_per_iter) {
    RawVec<VEC> rd[ROWS], rz[ROWS], ry[ROWS];
    unsigned long long rm = 0;
    bool ok[ROWS];
    if (SRC == 2) rm = mask_rows<ROWS>(amask, r, C >> 3, (int)(col >> 3)) >> (col & 7 & ~(VEC - 1));
#pragma unroll
    for (int u = 0; u < ROWS; ++u) {
      const long long rr = r + (long long)u * rstep;
      ok[u] = rr < row_end;
      if (ok[u]) {
        rd[u] = ldv(dy + rr * C + col, (RawVec<VEC>*)nullptr);
        rz[u] = ldv(z + rr * C + col, (RawVec<VEC>*)nullptr);
        if (SRC == 1) ry[u] = ldv(y + rr * C + col, (RawVec<VEC>*)nullptr);
      }
    }
#pragma unroll
    for (int u = 0; u < ROWS; ++u) {
      if (!ok[u]) continue;
      const long long rr = r + (long long)u * rstep;
      float da[VEC], za[VEC], ya[VEC];
      unpackv(rd[u], da);
      unpackv(rz[u], za);
      if (SRC == 1) unpackv(ry[u], ya);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        float g = da[i];
        if (SRC == 2) g = ((rm >> (8 * u + i)) & 1ull) ? g : 0.f;
        else if (act != B200_ACT_NONE && act_mask(SRC == 1 ? ya[i] : fmaf(za[i], A[i], sh[i]), act) == 0.f) g = 0.f;
        const float d = za[i] - mu[i];
        const float sgn = (d > 0.f ? 1.f : 0.f) - (d < 0.f ? 1.f : 0.f);
        da[i] = g;
        za[i] = A[i] * g + B[i] * sgn + Cc[i];
      }
      storev(dz + rr * C + col, za);
      if (g_out) storev(g_out + rr * C + col, da);
    }
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_bn_l1_stats(const void* z, long long M, int C, const float* gamma, const float* beta, float eps,
                                float momentum, float* running_mean, float* running_var, float* mean, float* invstd,
                                float* sign_sum, float* scale, float* shift, float* workspace, b200_stream_t stream_) {
  int rc = check_c(C, "bn_l1_stats");
  if (rc) return rc;
  B200_REQUIRE(z && mean && invstd && sign_sum && scale && shift && workspace && M > 0, B200_ERR_INVALID,
               "bn_l1_stats: bad argument");
  B200_REQUIRE(momentum >= 0.f && momentum <= 1.f, B200_ERR_INVALID, "bn_l1_stats: momentum %g outside [0, 1]",
               (double)momentum);
  cudaStream_t stream = (cudaStream_t)stream_;
  const RowMap rm = make_rowmap(C);
  const int blocks = partial_blocks(M, rm, 6);
  float* partial = workspace + kAccumFloats;
  const int fin = (C + 3) / 4;
  const __nv_bfloat16* zz = (const __nv_bfloat16*)z;
  b200::launch(bn_l1_partial_kernel<0>, blocks, kBnThreads, 0, stream, zz, M, C, rm.cv, rm.rows_per_iter,
               (const float*)nullptr, partial);
  B200_CHECK_LAUNCH("bn_l1_partial_kernel<0>");
  b200::launch(bn_l1_final_kernel<0>, fin, kBnThreads, 0, stream, (const float*)partial, blocks, M, C, gamma, beta, eps,
               momentum, running_mean, running_var, mean, invstd, sign_sum, scale, shift);
  B200_CHECK_LAUNCH("bn_l1_final_kernel<0>");
  b200::launch(bn_l1_partial_kernel<1>, blocks, kBnThreads, 0, stream, zz, M, C, rm.cv, rm.rows_per_iter,
               (const float*)mean, partial);
  B200_CHECK_LAUNCH("bn_l1_partial_kernel<1>");
  b200::launch(bn_l1_final_kernel<1>, fin, kBnThreads, 0, stream, (const float*)partial, blocks, M, C, gamma, beta, eps,
               momentum, running_mean, running_var, mean, invstd, sign_sum, scale, shift);
  B200_CHECK_LAUNCH("bn_l1_final_kernel<1>");
  return B200_OK;
}

extern "C" int b200_bn_l1_eval_coeffs(int C, const float* gamma, const float* beta, const float* running_mean,
                                      const float* running_var, float* scale, float* shift, b200_stream_t stream_) {
  B200_REQUIRE(C > 0 && running_mean && running_var && scale && shift, B200_ERR_INVALID,
               "bn_l1_eval_coeffs: bad argument");
  b200::launch(bn_l1_eval_coeffs_kernel, (C + 127) / 128, 128, 0, (cudaStream_t)stream_, C, gamma, beta, running_mean,
               running_var, scale, shift);
  B200_CHECK_LAUNCH("bn_l1_eval_coeffs_kernel");
  return B200_OK;
}

// launch shapes as b200_bn_bwd_dx: (VEC 4, ROWS 4, MINB 4) up to C = 1024, (8, 2, 3) above
extern "C" int b200_bn_l1_bwd_dx(const void* dy, const void* y, const uint8_t* act_mask, const void* z, long long M,
                                 int C, int act, const float* mean, const float* invstd, const float* sign_sum,
                                 const float* gamma, const float* beta, const float* sums, void* dz, void* g_out,
                                 b200_stream_t stream_) {
  int rc = check_c(C, "bn_l1_bwd_dx");
  if (rc) return rc;
  B200_REQUIRE(dy && z && mean && invstd && sign_sum && sums && dz && M > 0, B200_ERR_INVALID,
               "bn_l1_bwd_dx: bad argument");
  const int src = (act == B200_ACT_NONE) ? 0 : (act_mask != nullptr ? 2 : (y != nullptr ? 1 : 0));
#define B200_DX_ARGS(VEC)                                                                                    \
  (const __nv_bfloat16*)dy, (const __nv_bfloat16*)y, act_mask, (const __nv_bfloat16*)z, M, C, rm.cv,         \
      rm.rows_per_iter, act, mean, invstd, sign_sum, gamma, beta, sums, (__nv_bfloat16*)dz, (__nv_bfloat16*)g_out
#define B200_LAUNCH_DX(VEC, ROWS, MINB)                                                                      \
  do {                                                                                                       \
    const RowMap rm = make_rowmap_v<VEC>(C);                                                                 \
    const int blocks = stream_blocks(M, rm);                                                                 \
    if (src == 2)                                                                                            \
      b200::launch(bn_l1_bwd_dx_kernel<VEC, ROWS, MINB, 2>, blocks, kBnThreads, 0, (cudaStream_t)stream_,    \
                   B200_DX_ARGS(VEC));                                                                       \
    else if (src == 1)                                                                                       \
      b200::launch(bn_l1_bwd_dx_kernel<VEC, ROWS, MINB, 1>, blocks, kBnThreads, 0, (cudaStream_t)stream_,    \
                   B200_DX_ARGS(VEC));                                                                       \
    else                                                                                                     \
      b200::launch(bn_l1_bwd_dx_kernel<VEC, ROWS, MINB, 0>, blocks, kBnThreads, 0, (cudaStream_t)stream_,    \
                   B200_DX_ARGS(VEC));                                                                       \
  } while (0)
  if (C > 1024)
    B200_LAUNCH_DX(8, 2, 3);
  else
    B200_LAUNCH_DX(4, 4, 4);
#undef B200_LAUNCH_DX
#undef B200_DX_ARGS
  B200_CHECK_LAUNCH("bn_l1_bwd_dx_kernel");
  return B200_OK;
}
