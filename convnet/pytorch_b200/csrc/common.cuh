// Shared device helpers for the sm_90a kernels: mbarrier, TMA, wgmma wrappers.
// Everything here is inline PTX for compute_90a; nothing is borrowed from a library.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "wgmma.cuh"
#include "../../../include/b200conv.h"

#ifndef B200_WAIT_TIMEOUT_NS
#define B200_WAIT_TIMEOUT_NS 4000000000ull  // 4 s
#endif

namespace b200 {

// The convolution kernels: two consumer warpgroups + a producer warpgroup (only warp 8 works: registers are allocated
// per warpgroup in wgmma kernels, so 288 threads would cost as much as 384), 128 accumulator rows per tile.
constexpr int kThreads = 384;
constexpr int kTileM = 128;
// BN workspace accumulators: [kReplicas][2][C] fp64 rows (sum, sum of squares).  A block adds into replica
// blockIdx.x % kReplicas, which spreads same-address fp64 atomics over 16 lines.
constexpr int kReplicas = 16;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile(
      "{\n\t.reg .b64 st;\n\t"
      "mbarrier.arrive.shared::cta.b64 st, [%0];\n\t}"
      ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile(
      "{\n\t.reg .b64 st;\n\t"
      "mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}"
      ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Kept out of line: a trap instruction inlined after setmaxnreg makes ptxas allocate that code within the launch-bounds
// register cap (168 for 384 threads) instead of the reallocated count, and the consumers spill.
static __device__ __noinline__ void wait_timeout_trap() { __trap(); }
// Bounded wait: a protocol bug becomes a trap (launch failure) after B200_WAIT_TIMEOUT_NS instead of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0xFFu) == 0u && global_timer_ns() - t0 > B200_WAIT_TIMEOUT_NS) wait_timeout_trap();
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// tiled loads (global -> shared), completion on mbarrier
__device__ __forceinline__ void tma_load_2d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const void* tmap, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col load of a rank-4 NHWC tensor: coords {c, w, h, n} of the first base pixel, filter offsets {w, h}
__device__ __forceinline__ void tma_load_im2col_4d(const void* tmap, uint64_t* bar, void* dst,
                                                   int c, int w, int h, int n, uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)),
        "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

// tiled store (shared -> global), bulk-group completion
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------- wgmma
// Warpgroup MMA (sm_90a): a warpgroup (4 consecutive warps, the first a multiple of 4) issues wgmma.mma_async with both
// operands in shared memory; the fp32 accumulators live in the issuing threads' registers (wgmma.cuh).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Register reallocation of the 384-thread wgmma kernels (one producer warpgroup, two consumer warpgroups, 168 registers
// per thread at launch): the producer, which only issues TMA, drops to 56 (the weight-gradient producer keeps its
// per-box coordinate tables in registers) and the consumers grow to 224 (56 * 128 + 2 * 224 * 128 <= 65536).  Every
// warp of a warpgroup must execute the call, before any of them exits.
constexpr uint32_t kProducerRegs = 56, kConsumerRegs = 224;
__device__ __forceinline__ void producer_setmaxnreg() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
}
__device__ __forceinline__ void consumer_setmaxnreg() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
}
// Orders ordinary register accesses of the accumulators against the asynchronous MMAs that write them.
template <int SZ>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[SZ]) {
#pragma unroll
  for (int i = 0; i < SZ; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of wgmma.
//  start address [0,14) (>>4), leading byte offset [16,30) (>>4), stride byte offset [32,46) (>>4),
//  layout type [62,64): 0 none, 1 = 128B swizzle, 2 = 64B, 3 = 32B.  The swizzle is a function of the absolute
//  shared-memory address, so a descriptor may be advanced by any multiple of 16 bytes into a TMA-written buffer.
//  K-major: SBO = distance between 8-row groups (LBO unused with a swizzle).
//  MN-major: LBO = distance between swizzle-width column blocks along M/N, SBO = distance between 8-row groups along K.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t layout_type) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr >> 4) & 0x3FFF);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(layout_type & 3) << 62;
  return d;
}
__device__ __host__ __forceinline__ uint32_t layout_type_for_row_bytes(uint32_t row_bytes) {
  return row_bytes == 128 ? 1u : (row_bytes == 64 ? 2u : 3u);
}
// Accumulator fragment of m64nNk16 for thread t of the warpgroup: element i sits at row 16 * (t / 32) + (t % 32) / 4
// + 8 * ((i / 2) % 2), column 8 * (i / 4) + 2 * (t % 4) + i % 2.

// ---------------------------------------------------------------- misc
__device__ __forceinline__ float apply_act(float v, int act) {
  return act == B200_ACT_RELU ? fmaxf(v, 0.f) : (act == B200_ACT_RELU6 ? fminf(fmaxf(v, 0.f), 6.f) : v);
}
// consumer warp: its MMAs are done reading a ring slot whose empty barrier counts one arrival per consumer warp
__device__ __forceinline__ void release_stage(uint64_t* empty_bar, int lane) {
  __syncwarp();
  if (lane == 0) mbar_arrive(empty_bar);
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
// Byte offset of element (row, c) in a convolution epilogue's bf16 staging tile: 64-channel boxes `pitch` bytes apart,
// each [rows][128 B] in the 128B swizzle of the TMA store that writes it out.
__device__ __forceinline__ uint32_t staged_offset(int row, int c, uint32_t pitch) {
  return (c >> 6) * pitch + row * 128 + ((((c & 63) >> 3) ^ (row & 7)) << 4) + (c & 7) * 2;
}
// Adds one thread's (sum, sum of squares) of output channel n0 + col into this block's replica row of the BN workspace.
__device__ __forceinline__ void flush_bn_stats(double* stats, int C, int n0, int col, float s1, float s2) {
  double* dst = stats + (blockIdx.x % kReplicas) * 2 * C + n0 + col;
  atomicAdd(dst, (double)s1);
  atomicAdd(dst + C, (double)s2);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace b200
