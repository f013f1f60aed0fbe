// Shared by the BatchNorm kernels (bn.cu), the L1 BatchNorm kernels (bn_l1.cu) and the dropout kernels (dropout.cu):
// the BN workspace layout, the row/vector thread mapping, grid sizing, the vectorised bf16 load/store and
// activation-mask helpers, and the bodies of the backward reduction and input-gradient kernels.
#pragma once
#include "common.cuh"
#include "host.h"

namespace b200 {

constexpr int kBnThreads = 256;
constexpr int kBnMaxC = 2048;
constexpr int kBnMaxBlocks = 1184;  // 8 per SM on 148 SMs
constexpr int kAccumFloats = kReplicas * 2 * kBnMaxC * 2 + 64;  // replicas x 2*C doubles + ticket counter
constexpr int kMaxPartialBlocks = 6 * 148;                         // backward reduce: per-block partial rows
constexpr int kWsFloats = kAccumFloats + kMaxPartialBlocks * 2 * kBnMaxC;

struct RowMap {
  int cv, rows_per_iter;
};
static inline RowMap make_rowmap(int C) {
  RowMap m;
  m.cv = C / 8;
  m.rows_per_iter = kBnThreads / m.cv;
  return m;
}
// backward reduce (two-stage, no atomics): one resident wave of fat blocks, each at least 4 row-iterations
static inline int partial_blocks(long long M, const RowMap& rm, int resident_per_sm) {
  long long iters = (M + rm.rows_per_iter - 1) / rm.rows_per_iter;
  long long want = (iters + 3) / 4;
  long long cap = (long long)resident_per_sm * sm_count();
  if (cap > kMaxPartialBlocks) cap = kMaxPartialBlocks;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  return (int)want;
}
static inline int stream_blocks(long long M, const RowMap& rm) {
  long long iters = (M + rm.rows_per_iter - 1) / rm.rows_per_iter;
  long long blocks = (iters + 15) / 16;
  if (blocks < 1) blocks = 1;
  if (blocks > 4 * kBnMaxBlocks) blocks = 4 * kBnMaxBlocks;
  return (int)blocks;
}

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
// streaming 128-bit load: read-only path, no L1 allocation (every byte is touched once per kernel)
__device__ __forceinline__ uint4 ld_stream(const __nv_bfloat16* p) {
  uint4 u;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
  return u;
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void loadf8(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
// 1 where the activation passes the gradient, evaluated on the PRE-activation value (same test as act_mask on y)
__device__ __forceinline__ int act_mask_value(float pre, int act) {
  if (act == B200_ACT_RELU) return pre > 0.f ? 1 : 0;
  if (act == B200_ACT_RELU6) return (pre > 0.f && pre < 6.f) ? 1 : 0;
  return 1;
}
__device__ __forceinline__ float act_mask(float v, int act) {
  if (act == B200_ACT_RELU) return v > 0.f ? 1.f : 0.f;
  if (act == B200_ACT_RELU6) return (v > 0.f && v < 6.f) ? 1.f : 0.f;
  return 1.f;
}

// Activation-mask layout ("row quads"): the bytes of rows 4q..4q+3 for one 8-channel vector form ONE 32-bit word,
// word index q * (C/8) + v8.  A backward thread that owns ROWS consecutive rows fetches their masks with a single
// 16/32-bit load -- with a plain [row][C/8] byte layout every row cost its own load instruction, and the kernels are
// bound by requests in flight, not by bytes (that version was slower than re-reading the bf16 output).
__device__ __forceinline__ long long mask_byte_index(long long row, int cv8, int v8) {
  return (((row >> 2) * cv8 + v8) << 2) + (row & 3);
}
// mask bytes of rows [row0, row0 + ROWS) (row0 % ROWS == 0, ROWS in {2, 4, 8}) for vector v8: byte u = row row0 + u
template <int ROWS>
__device__ __forceinline__ unsigned long long mask_rows(const uint8_t* __restrict__ amask, long long row0, int cv8,
                                                        int v8) {
  const uint8_t* p = amask + mask_byte_index(row0, cv8, v8);
  if (ROWS == 2) return __ldg(reinterpret_cast<const unsigned short*>(p));
  if (ROWS == 4) return __ldg(reinterpret_cast<const unsigned int*>(p));
  const unsigned long long lo = __ldg(reinterpret_cast<const unsigned int*>(p));
  const unsigned long long hi = __ldg(reinterpret_cast<const unsigned int*>(p + 4LL * cv8));
  return lo | (hi << 32);
}

// ---- backward helpers: VEC (4 or 8) channels per thread ----------------------------------------------
template <int VEC> struct RawVec;
template <> struct RawVec<4> { uint2 u; };
template <> struct RawVec<8> { uint4 u; };
__device__ __forceinline__ RawVec<4> ldv(const __nv_bfloat16* p, RawVec<4>*) {
  RawVec<4> r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.u.x), "=r"(r.u.y) : "l"(p));
  return r;
}
__device__ __forceinline__ RawVec<8> ldv(const __nv_bfloat16* p, RawVec<8>*) {
  RawVec<8> r;
  r.u = ld_stream(p);
  return r;
}
__device__ __forceinline__ void unpackv(const RawVec<4>& r, float (&f)[4]) {
  const float2 a = unpack_bf16x2(r.u.x), b = unpack_bf16x2(r.u.y);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}
__device__ __forceinline__ void unpackv(const RawVec<8>& r, float (&f)[8]) { unpack8(r.u, f); }
__device__ __forceinline__ void storev(__nv_bfloat16* p, const float (&f)[4]) {
  uint2 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  *reinterpret_cast<uint2*>(p) = u;
}
__device__ __forceinline__ void storev(__nv_bfloat16* p, const float (&f)[8]) { store8(p, f); }
template <int VEC>
__device__ __forceinline__ void loadfv(const float* p, float (&f)[VEC]) {
#pragma unroll
  for (int i = 0; i < VEC; i += 4) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p + i));
    f[i] = a.x; f[i + 1] = a.y; f[i + 2] = a.z; f[i + 3] = a.w;
  }
}

template <int VEC>
static inline RowMap make_rowmap_v(int C) {
  RowMap m;
  m.cv = C / VEC;
  m.rows_per_iter = kBnThreads / m.cv;
  return m;
}

static int check_c(int C, const char* who) {
  B200_REQUIRE(C > 0 && C % 8 == 0 && C <= kBnMaxC, B200_ERR_UNSUPPORTED,
               "%s: C=%d must be a multiple of 8 and <= %d", who, C, kBnMaxC);
  return B200_OK;
}

// ---- backward kernel bodies ---------------------------------------------------------------------
// Thread mapping: VEC channels per thread (VEC=4: 64-bit accesses, half the per-channel coefficient registers of
// VEC=8, which is what keeps these 2-read(+1-write) streams at the occupancy of bn_apply; VEC=8 only for C > 1024).
// g = dy where act'(.) passes, else +0 (selected, not multiplied: dy * 0 would give -0 for negative dy, unlike the
// mask-bit source and torch's threshold backward), where the activation argument is y when given, else recomputed as
// z*scale+shift (bit-identical to the forward's fused multiply-add).
// SRC: activation argument 0 recomputed from z, 1 = y, 2 = mask bits, 3 = mask bits of dropout(relu(.)) -- the kept
// gradient is dy * dscale (the dropout scale), read by dropout.cu only.

// backward reduce: dbeta = sum g, dgamma = sum g * xhat; one partial row of 2C floats per block
template <int VEC, int ROWS, int SRC>
__device__ __forceinline__ void bn_bwd_reduce_body(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ amask,
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter, int act,
    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
    const float* __restrict__ beta, float* __restrict__ partial, float dscale) {
  constexpr bool kBits = SRC >= 2;
  const int t = threadIdx.x;
  const bool active = t < rows_per_iter * cv;
  const int r0 = t / cv, v = t - r0 * cv;
  // mask words: a thread owns ROWS CONSECUTIVE rows (one mask load); block ranges are multiples of 8 rows
  const long long rows_per_block = kBits ? (((M + gridDim.x - 1) / gridDim.x + 7) & ~7LL) : (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  constexpr long long kRowStep = kBits ? 1 : 0;          // distance between a thread's rows: 1 or rows_per_iter
  float acc[2 * VEC];
#pragma unroll
  for (int i = 0; i < 2 * VEC; ++i) acc[i] = 0.f;
  if (active) {
    float mu[VEC], sc[VEC], sh[VEC];
    loadfv<VEC>(mean + v * VEC, mu);
    if (SRC == 0 && act != B200_ACT_NONE) {
      float is[VEC];
      loadfv<VEC>(invstd + v * VEC, is);
      if (gamma) loadfv<VEC>(gamma + v * VEC, sc);
      if (beta) loadfv<VEC>(beta + v * VEC, sh);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        sc[i] = (gamma ? sc[i] : 1.f) * is[i];
        sh[i] = (beta ? sh[i] : 0.f) - mu[i] * sc[i];
      }
    }
    const long long col = (long long)v * VEC;
    const long long rstep = kRowStep ? 1 : rows_per_iter;
    for (long long r = row_begin + (kRowStep ? (long long)r0 * ROWS : r0); r < row_end;
         r += (long long)ROWS * rows_per_iter) {
      RawVec<VEC> rd[ROWS], rz[ROWS], ry[ROWS];
      unsigned long long rm = 0;
      bool ok[ROWS];
      if (kBits) rm = mask_rows<ROWS>(amask, r, C >> 3, (int)(col >> 3)) >> (col & 7 & ~(VEC - 1));
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
        float da[VEC], za[VEC], ya[VEC];
        unpackv(rd[u], da);
        unpackv(rz[u], za);
        if (SRC == 1) unpackv(ry[u], ya);
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          float g = da[i];
          if (kBits) g = ((rm >> (8 * u + i)) & 1ull) ? (SRC == 3 ? g * dscale : g) : 0.f;
          else if (act != B200_ACT_NONE && act_mask(SRC == 1 ? ya[i] : fmaf(za[i], sc[i], sh[i]), act) == 0.f) g = 0.f;
          acc[i] = fmaf(g, za[i] - mu[i], acc[i]);   // the 1/std factor is applied once per channel below
          acc[VEC + i] += g;
        }
      }
    }
    float is[VEC];
    loadfv<VEC>(invstd + v * VEC, is);
#pragma unroll
    for (int i = 0; i < VEC; ++i) acc[i] *= is[i];
  }
  // block partial: fold the rows_per_iter row groups in shared memory, one coalesced row of 2C floats per block
  __shared__ float red[kBnThreads][2 * VEC + 1];
#pragma unroll
  for (int i = 0; i < 2 * VEC; ++i) red[t][i] = acc[i];
  __syncthreads();
  float* dst = partial + (size_t)blockIdx.x * 2 * C;
  for (int o = t; o < 2 * C; o += kBnThreads) {
    const int stat = o / C;
    const int c = o - stat * C;
    const int vv = c / VEC, e = c - vv * VEC;
    float sacc = 0.f;
    for (int r = 0; r < rows_per_iter; ++r) sacc += red[r * cv + vv][stat * VEC + e];
    dst[o] = sacc;
  }
}

// backward dx: dz = A*g + B*z + Cc (g_out: optionally also g)
template <int VEC, int ROWS, int SRC>
__device__ __forceinline__ void bn_bwd_dx_body(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ amask,
    const __nv_bfloat16* __restrict__ z, long long M, int C, int cv, int rows_per_iter, int act,
    const float* __restrict__ mean, const float* __restrict__ invstd, const float* __restrict__ gamma,
    const float* __restrict__ beta, const float* __restrict__ sums, __nv_bfloat16* __restrict__ dz,
    __nv_bfloat16* __restrict__ g_out, float dscale) {
  constexpr bool kBits = SRC >= 2;
  const int t = threadIdx.x;
  if (t >= rows_per_iter * cv) return;
  const int r0 = t / cv, v = t - r0 * cv;
  const long long rows_per_block = kBits ? (((M + gridDim.x - 1) / gridDim.x + 7) & ~7LL) : (M + gridDim.x - 1) / gridDim.x;
  const long long row_begin = blockIdx.x * rows_per_block;
  const long long row_end = min(M, row_begin + rows_per_block);
  constexpr long long kRowStep = kBits ? 1 : 0;          // as in bn_bwd_reduce_body
  // dz = A*g + B*z + Cc  with A = gamma*istd, B = -gamma*istd^2*dgamma/M, Cc = -A*dbeta/M - B*mean;
  // the activation argument recomputed from z is z*A + sh
  float A[VEC], B[VEC], Cc[VEC], sh[VEC];
  {
    float mu[VEC], is[VEC], dg[VEC], dbt[VEC];
    loadfv<VEC>(mean + v * VEC, mu);
    loadfv<VEC>(invstd + v * VEC, is);
    if (gamma) loadfv<VEC>(gamma + v * VEC, A);
    if (beta) loadfv<VEC>(beta + v * VEC, sh);
    loadfv<VEC>(sums + v * VEC, dg);
    loadfv<VEC>(sums + C + v * VEC, dbt);
    const float invM = 1.f / (float)M;
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float gm = gamma ? A[i] : 1.f;
      A[i] = gm * is[i];
      B[i] = -gm * is[i] * is[i] * dg[i] * invM;
      Cc[i] = -A[i] * dbt[i] * invM - B[i] * mu[i];
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
    if (kBits) rm = mask_rows<ROWS>(amask, r, C >> 3, (int)(col >> 3)) >> (col & 7 & ~(VEC - 1));
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
        if (kBits) g = ((rm >> (8 * u + i)) & 1ull) ? (SRC == 3 ? g * dscale : g) : 0.f;
        else if (act != B200_ACT_NONE && act_mask(SRC == 1 ? ya[i] : fmaf(za[i], A[i], sh[i]), act) == 0.f) g = 0.f;
        da[i] = g;
        za[i] = A[i] * g + B[i] * za[i] + Cc[i];
      }
      storev(dz + rr * C + col, za);
      if (g_out) storev(g_out + rr * C + col, da);
    }
  }
}

// second stage of the backward reduction (bn_bwd_reduce_final_kernel, bn.cu): sums = the fixed-order sum of the
// partial rows, accumulated into dgamma_acc / dbeta_acc when given
void launch_bwd_reduce_final(const float* partial, int nblocks, int C, float* sums, float* dgamma_acc,
                             float* dbeta_acc, cudaStream_t stream);

}  // namespace b200
