// Dropout inside residual blocks: dropout(relu(bn(z))) fused into the BatchNorm apply and backward.  Replaces the
// reference's nn.Dropout between relu(bn1(conv1(x))) and conv2 of a CIFAR BasicBlock (models/resnet.py:81-118).
//
// Random stream (a pure function of key, layer and element; tests/test_dropout_cpu.py restates it in numpy):
//   Philox4x32-10 (Salmon et al., SC'11) with key {k0, k1} = low / high word of a 64-bit value the caller draws per
//   training step.  The 8-channel vector g = (row*C + c) / 8 of dropout layer `layer` uses counter
//   {g & 0xffffffff, g >> 32, layer, 0}; its element j takes the 16-bit uniform u_j = (w[j>>1] >> 16*(j&1)) & 0xffff of
//   the output words w and is kept iff u_j < T, T = round((1 - p) * 65536).  One Philox call covers 8 elements.
//
// Forward: y = keep && pre > 0 ? bf16(pre * c) : +0 with pre = z*scale + shift (bn_apply's fused multiply-add) and
// c = fp32(1/(1-p)); the same bit goes to the row-quad activation mask, so the backward never regenerates the stream.
// Backward: g = bit ? dy * c : +0, then the ordinary BN backward (bodies shared with bn.cu through bn_common.cuh).
#include "bn_common.cuh"

namespace b200 {

__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t lo0 = 0xD2511F53u * ctr.x, hi0 = __umulhi(0xD2511F53u, ctr.x);
    const uint32_t lo1 = 0xCD9E8D57u * ctr.z, hi1 = __umulhi(0xCD9E8D57u, ctr.z);
    ctr = make_uint4(hi1 ^ ctr.y ^ k0, lo1, hi0 ^ ctr.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return ctr;
}

// y and mask byte of one 8-channel vector of row `row`
__device__ __forceinline__ uint32_t apply_dropout8(const uint4& raw, const float (&sc)[8], const float (&sh)[8],
                                                   long long vec, uint32_t k0, uint32_t k1, int layer, uint32_t T,
                                                   float c, float (&out)[8]) {
  float f[8];
  unpack8(raw, f);
  const uint4 w4 = philox4x32_10(make_uint4((uint32_t)vec, (uint32_t)((unsigned long long)vec >> 32), (uint32_t)layer, 0u),
                                 k0, k1);
  const uint32_t w[4] = {w4.x, w4.y, w4.z, w4.w};
  uint32_t bits = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float pre = fmaf(f[i], sc[i], sh[i]);
    const bool keep = ((w[i >> 1] >> (16 * (i & 1))) & 0xffffu) < T;
    const bool bit = keep && pre > 0.f;
    out[i] = bit ? pre * c : 0.f;
    bits |= static_cast<uint32_t>(bit) << i;
  }
  return bits;
}

__global__ void __launch_bounds__(kBnThreads) bn_apply_dropout_kernel(
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter,
    const float* __restrict__ scale, const float* __restrict__ shift, const unsigned long long* __restrict__ key,
    int layer, uint32_t T, float c, __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ act_mask) {
  const int t = threadIdx.x;
  if (t >= rows_per_iter * cv) return;
  const int r0 = t / cv, v = t - r0 * cv;
  const long long rows_per_block = (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  const unsigned long long k = __ldg(key);
  const uint32_t k0 = (uint32_t)k, k1 = (uint32_t)(k >> 32);
  float sc[8], sh[8];
  loadf8(scale + v * 8, sc);
  loadf8(shift + v * 8, sh);
  for (long long r = row_begin + r0; r < row_end; r += 2LL * rows_per_iter) {
    const long long ra = r, rb = r + rows_per_iter;
    const bool hb = rb < row_end;
    uint4 za = ld_stream(z + ra * C + v * 8), zb;
    if (hb) zb = ld_stream(z + rb * C + v * 8);
    float fa[8], fb[8];
    const uint32_t ma = apply_dropout8(za, sc, sh, ra * cv + v, k0, k1, layer, T, c, fa);
    store8(y + ra * C + v * 8, fa);
    act_mask[mask_byte_index(ra, cv, v)] = static_cast<uint8_t>(ma);
    if (hb) {
      const uint32_t mb = apply_dropout8(zb, sc, sh, rb * cv + v, k0, k1, layer, T, c, fb);
      store8(y + rb * C + v * 8, fb);
      act_mask[mask_byte_index(rb, cv, v)] = static_cast<uint8_t>(mb);
    }
  }
}

template <int VEC, int ROWS, int MINB>
__global__ void __launch_bounds__(kBnThreads, MINB) bn_bwd_reduce_dropout_kernel(
    const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ amask, const __nv_bfloat16* __restrict__ z,
    long long M, int C, int cv, int rows_per_iter, float c, const float* __restrict__ mean,
    const float* __restrict__ invstd, float* __restrict__ partial) {
  bn_bwd_reduce_body<VEC, ROWS, 3>(dy, nullptr, amask, z, M, C, cv, rows_per_iter, B200_ACT_RELU, mean, invstd, nullptr,
                                   nullptr, partial, c);
}

template <int VEC, int ROWS, int MINB>
__global__ void __launch_bounds__(kBnThreads, MINB) bn_bwd_dx_dropout_kernel(
    const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ amask, const __nv_bfloat16* __restrict__ z,
    long long M, int C, int cv, int rows_per_iter, float c, const float* __restrict__ mean,
    const float* __restrict__ invstd, const float* __restrict__ gamma, const float* __restrict__ sums,
    __nv_bfloat16* __restrict__ dz) {
  bn_bwd_dx_body<VEC, ROWS, 3>(dy, nullptr, amask, z, M, C, cv, rows_per_iter, B200_ACT_RELU, mean, invstd, gamma,
                               nullptr, sums, dz, nullptr, c);
}

}  // namespace b200

using namespace b200;

extern "C" int b200_bn_apply_dropout(const void* z, long long M, int C, const float* scale, const float* shift,
                                     const uint64_t* key, int layer, unsigned T, float c, void* y, uint8_t* act_mask,
                                     b200_stream_t stream_) {
  int rc = check_c(C, "bn_apply_dropout");
  if (rc) return rc;
  B200_REQUIRE(z && scale && shift && key && y && act_mask && M > 0, B200_ERR_INVALID, "bn_apply_dropout: bad argument");
  B200_REQUIRE(layer >= 0 && T <= 65536u, B200_ERR_INVALID, "bn_apply_dropout: layer=%d T=%u out of range", layer, T);
  const RowMap rm = make_rowmap(C);
  b200::launch(bn_apply_dropout_kernel, stream_blocks(M, rm), kBnThreads, 0, (cudaStream_t)stream_,
               (const __nv_bfloat16*)z, M, C, rm.cv, rm.rows_per_iter, scale, shift,
               (const unsigned long long*)key, layer, (uint32_t)T, c, (__nv_bfloat16*)y, act_mask);
  B200_CHECK_LAUNCH("bn_apply_dropout_kernel");
  return B200_OK;
}

// launch shapes (VEC, ROWS, MINB) as b200_bn_bwd_reduce / b200_bn_bwd_dx: (4, 4, 4) up to C = 1024, (8, 2, 3) above
extern "C" int b200_bn_bwd_reduce_dropout(const void* dy, const uint8_t* act_mask, const void* z, long long M, int C,
                                          float c, const float* mean, const float* invstd, float* sums,
                                          float* dgamma_acc, float* dbeta_acc, float* workspace,
                                          b200_stream_t stream_) {
  int rc = check_c(C, "bn_bwd_reduce_dropout");
  if (rc) return rc;
  B200_REQUIRE(dy && act_mask && z && mean && invstd && sums && workspace && M > 0, B200_ERR_INVALID,
               "bn_bwd_reduce_dropout: bad argument");
  cudaStream_t stream = (cudaStream_t)stream_;
  float* partial = workspace + kAccumFloats;
  int blocks = 0;
#define B200_LAUNCH_RED(VEC, ROWS, MINB)                                                                       \
  do {                                                                                                         \
    const RowMap rm = make_rowmap_v<VEC>(C);                                                                   \
    blocks = partial_blocks(M, rm, MINB);                                                                      \
    b200::launch(bn_bwd_reduce_dropout_kernel<VEC, ROWS, MINB>, blocks, kBnThreads, 0, stream,                 \
                 (const __nv_bfloat16*)dy, act_mask, (const __nv_bfloat16*)z, M, C, rm.cv, rm.rows_per_iter, c, \
                 mean, invstd, partial);                                                                       \
  } while (0)
  if (C > 1024)
    B200_LAUNCH_RED(8, 2, 3);
  else
    B200_LAUNCH_RED(4, 4, 4);
#undef B200_LAUNCH_RED
  B200_CHECK_LAUNCH("bn_bwd_reduce_dropout_kernel");
  launch_bwd_reduce_final(partial, blocks, C, sums, dgamma_acc, dbeta_acc, stream);
  B200_CHECK_LAUNCH("bn_bwd_reduce_final_kernel");
  return B200_OK;
}

extern "C" int b200_bn_bwd_dx_dropout(const void* dy, const uint8_t* act_mask, const void* z, long long M, int C,
                                      float c, const float* mean, const float* invstd, const float* gamma,
                                      const float* sums, void* dz, b200_stream_t stream_) {
  int rc = check_c(C, "bn_bwd_dx_dropout");
  if (rc) return rc;
  B200_REQUIRE(dy && act_mask && z && mean && invstd && sums && dz && M > 0, B200_ERR_INVALID,
               "bn_bwd_dx_dropout: bad argument");
#define B200_LAUNCH_DX(VEC, ROWS, MINB)                                                                        \
  do {                                                                                                         \
    const RowMap rm = make_rowmap_v<VEC>(C);                                                                   \
    b200::launch(bn_bwd_dx_dropout_kernel<VEC, ROWS, MINB>, stream_blocks(M, rm), kBnThreads, 0,               \
                 (cudaStream_t)stream_, (const __nv_bfloat16*)dy, act_mask, (const __nv_bfloat16*)z, M, C, rm.cv, \
                 rm.rows_per_iter, c, mean, invstd, gamma, sums, (__nv_bfloat16*)dz);                          \
  } while (0)
  if (C > 1024)
    B200_LAUNCH_DX(8, 2, 3);
  else
    B200_LAUNCH_DX(4, 4, 4);
#undef B200_LAUNCH_DX
  B200_CHECK_LAUNCH("bn_bwd_dx_dropout_kernel");
  return B200_OK;
}
