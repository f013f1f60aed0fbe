// Implicit-GEMM convolution on Hopper tensor cores (sm_90a wgmma): fprop, dgrad, wgrad.
//
//   fprop : y[m, k]   = sum_{tap, c} x_im2col[m, tap, c] * w[k, tap, c]        (A K-major, B K-major)
//   dgrad : dx[m, c]  = sum_{tap, k} dy_im2col[m, tap, k] * wt[c, tap, k]       (same kernel, tap table)
//   wgrad : dw[k, tap, c] += sum_{pix} dy[pix, k] * x_im2col[pix, tap, c]       (A MN-major, B MN-major)
//
// Operand tiles are staged by TMA (im2col mode for the activation side, tiled mode for weights / dy)
// into 32/64/128B-swizzled shared memory and consumed by wgmma.mma_async with fp32 accumulators in registers.
// Warp roles: warps 0..7 = two consumer warpgroups, warp 8 (of the third warpgroup) = TMA producer.  The implicit-GEMM
// kernel runs the consumers ping-pong: each owns whole 128-row tiles, alternating with the other, so one warpgroup's
// epilogue runs while the other's MMAs keep the tensor cores busy.  The weight-gradient kernel splits each tile's
// output channels between them.
//
// Replaces cuDNN's convolution behind nn.Conv2d in the reference (models/resnet.py:75-78,126-132,
// 226-227) and its autograd backward (trainer.py:162).
#include "common.cuh"
#include "host.h"
#include <stdlib.h>
#include <utility>

namespace b200 {

constexpr int kMaxStages = 8;
constexpr int kMaxTaps = 32;
constexpr int kConsumers = 256;
constexpr int kProducerWarp = 8;

struct TapEntry {
  uint16_t off_w, off_h;  // im2col filter offsets (added to the base pixel)
  uint16_t b_tap;         // which tap slice of the weight operand
  uint16_t pad_;
};

struct IgemmParams {
  int M_total;           // rows of the implicit GEMM = Nimg * I * J
  int I, J;              // base-pixel grid per image
  int trav;              // traversal stride of base pixels in the source tensor
  int lower_w, lower_h;  // source coordinate of base pixel (0,0)
  int N_total;           // GEMM N (channels produced)
  int block_n, n_tiles, m_tiles;
  int ck, c_chunks;      // channels per k-block, number of k-blocks per tap
  int ntaps;
  int num_stages;
  uint32_t a_bytes, b_bytes, tx_bytes;
  // output mapping: row m=(n,i,j) -> out pixel (n, i*os+oh0, j*os+ow0) of an [Nimg,OH,OW,ldo] tensor
  int OH, OW, os, oh0, ow0;
  int ldo;
  int act, out_fp32;
  int tma_store;         // 1: dense bf16 output staged in smem and written by TMA (tmC), residual via tmR
  int plain_a;           // 1: A is a dense [M_total, SC] matrix (1x1, stride 1, no padding): tiled TMA
  int b_stationary;      // 1: every (tap, k-block) weight slice stays in shared memory (small 1x1 layers): only A streams
  int own_ntile;         // 1 (with b_stationary): the CTA owns n-tile blockIdx.x % n_tiles -- its weight slices are loaded
                         // once -- and walks the m-tiles blockIdx.x / n_tiles, + gridDim.x / n_tiles, ... (the grid is a
                         // multiple of n_tiles).  Cuts the L2->SM re-streaming of the weights from once per tile to once
                         // per CTA for layers whose per-n-tile weights fit in shared memory beside the ring
  int window;            // > 0: block-diagonal convolution -- output channels [window*b, window*b + window) read source
                         // channels [window*b, window*b + window) only; the weight operand is [N_total][taps][window]
  uint32_t epi_bytes;    // one warpgroup's output staging tile
  int epi_bufs;          // staging tiles per warpgroup (1 or 2), used alternately: with 2, a tile's epilogue does not
                         // wait for the TMA store of the warpgroup's previous tile to leave shared memory
  double* stats;         // fused BN statistics accumulators [kReplicas][2][N_total] (BN workspace) or nullptr
  void* out;
  const void* res;
  const float* bias;
  TapEntry taps[kMaxTaps];
};

// Columns n, n+1 (n even) of one output row through the generic output mapping; off = element offset of the row.
__device__ __forceinline__ void store_pair(const IgemmParams& p, float v0, float v1, long long off, int n) {
  if (n >= p.N_total) return;
  const bool two = n + 1 < p.N_total;
  const bool vec = two && (p.ldo & 1) == 0;
  if (p.bias != nullptr) {
    v0 += __ldg(p.bias + n);
    if (two) v1 += __ldg(p.bias + n + 1);
  }
  if (p.res != nullptr) {
    const __nv_bfloat16* r = reinterpret_cast<const __nv_bfloat16*>(p.res) + off + n;
    if (vec) {
      const float2 t = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(r));
      v0 += t.x;
      v1 += t.y;
    } else {
      v0 += __bfloat162float(r[0]);
      if (two) v1 += __bfloat162float(r[1]);
    }
  }
  v0 = apply_act(v0, p.act);
  v1 = apply_act(v1, p.act);
  if (p.out_fp32) {
    float* o = reinterpret_cast<float*>(p.out) + off + n;
    if (vec) {
      *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
    } else {
      o[0] = v0;
      if (two) o[1] = v1;
    }
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + off + n;
    if (vec) {
      *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(v0, v1);
    } else {
      o[0] = __float2bfloat16(v0);
      if (two) o[1] = __float2bfloat16(v1);
    }
  }
}

// store_pair for every column pair of one output row of a fragment (accumulators a[j + 2h], a[j + 2h + 1] at column
// 2j), bf16, no bias or activation, all columns inside N_total and ldo even; off = element offset of the row's first
// column pair.  The same arithmetic as store_pair, without its run-time branches.
template <int BN, bool RES>
__device__ __forceinline__ void store_row_bf16(const IgemmParams& p, const float (&a)[BN / 2], int h, long long off) {
#pragma unroll
  for (int j = 0; j < BN / 2; j += 4) {
    float v0 = a[j + 2 * h], v1 = a[j + 2 * h + 1];
    if (RES) {
      const float2 t = unpack_bf16x2(*(reinterpret_cast<const uint32_t*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + off + 2 * j)));
      v0 += t.x;
      v1 += t.y;
    }
    *reinterpret_cast<uint32_t*>(reinterpret_cast<__nv_bfloat16*>(p.out) + off + 2 * j) = pack_bf16x2(v0, v1);
  }
}

// The MMAs of one operand stage for a warpgroup's 128-row tile: per 16-deep k-step, two m64 wgmmas (rows 0-63 and
// 64-127) that share the B descriptor.  KS is the stage's k-steps (ck / 16); scale0 == 0 starts the accumulators.
template <int KS, int SZ>
__device__ __forceinline__ void igemm_stage_mma(float (&acc)[2][SZ], uint64_t da, uint64_t db, uint32_t a_half,
                                                uint32_t scale0) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KS; ++k) {
    wgmma_bf16<0, 0>(acc[0], da + 2 * k, db + 2 * k, k != 0 ? 1u : scale0);
    wgmma_bf16<0, 0>(acc[1], da + a_half + 2 * k, db + 2 * k, k != 0 ? 1u : scale0);
  }
  wgmma_commit();
}

// Writes a warpgroup's 128 x BN accumulator tile, + bias, + residual (fetched into the same staging tile beforehand),
// activation, rounded to bf16, into the 128B-swizzled staging tile epi_w (64-column boxes of [128 rows][128 B]).
// FIXED = 1: no bias, no activation and the residual given by RES at compile time -- the epilogues of training (the
// statistics-fusing forward pass, the data gradient with or without residual) -- so that the unrolled loop has no
// branch.  With a run-time switch per value the scheduler could not overlap one value's residual load, adds, pack and
// store with the next value's, and staging a 128-column tile took several times as long as its MMAs.  FIXED = 0 reads
// the bias, residual and activation at run time.
template <int BN, int FIXED, bool RES>
__device__ __forceinline__ void stage_tile(uint8_t* epi_w, const float (&acc)[2][BN / 2], const IgemmParams& p,
                                           int nbase, int r_lo, int c_lo) {
  const bool res = FIXED ? RES : p.res != nullptr;
  const int act = FIXED ? B200_ACT_NONE : p.act;
#pragma unroll
  for (int j = 0; j < BN / 2; j += 4) {
    const int c = 2 * j + c_lo;
    float bias0 = 0.f, bias1 = 0.f;   // added even without a bias: x + 0 turns -0 into +0
    if (!FIXED && p.bias != nullptr) { bias0 = __ldg(p.bias + nbase + c); bias1 = __ldg(p.bias + nbase + c + 1); }
#pragma unroll
    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = mh * 64 + r_lo + 8 * h;
        uint32_t* dst = reinterpret_cast<uint32_t*>(epi_w + staged_offset(row, c, kTileM * 128));
        float v0 = acc[mh][j + 2 * h] + bias0, v1 = acc[mh][j + 2 * h + 1] + bias1;
        if (res) {
          const float2 t = unpack_bf16x2(*dst);
          v0 += t.x;
          v1 += t.y;
        }
        *dst = pack_bf16x2(apply_act(v0, act), apply_act(v1, act));
      }
  }
}

// BN = block_n, the tile width: it sizes the accumulators exactly and fixes the wgmma shape at compile time.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                  const __grid_constant__ IgemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ __align__(8) uint64_t turn_bar[2], res_bar[2], bstat_bar;   // [warpgroup]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  const uint32_t stage_bytes = p.b_stationary ? p.a_bytes : p.a_bytes + p.b_bytes;
  uint8_t* sBstat = smem + p.num_stages * stage_bytes;   // stationary weight slices [tap * c_chunks + k-block]
  uint8_t* epi = sBstat + (p.b_stationary ? static_cast<uint32_t>(p.ntaps * p.c_chunks) * p.b_bytes : 0u);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);   // released by the four warps of the warpgroup that consumed it
    }
    mbar_init(&bstat_bar, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&res_bar[i], 1);
      mbar_init(&turn_bar[i], 4);
    }
    fence_mbar_init();
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if (p.tma_store) {
      prefetch_tmap(&tmC);
      if (p.res != nullptr) prefetch_tmap(&tmR);
    }
  }
  __syncthreads();

  const int k_iters = p.ntaps * p.c_chunks;
  // tile walk: round-robin over all (m, n) tiles, or -- owned n-tile -- over the m-tiles of one n-tile
  const int walk_first = p.own_ntile ? static_cast<int>(blockIdx.x) / p.n_tiles : static_cast<int>(blockIdx.x);
  const int walk_step = p.own_ntile ? static_cast<int>(gridDim.x) / p.n_tiles : static_cast<int>(gridDim.x);
  const int walk_end = p.own_ntile ? p.m_tiles : p.m_tiles * p.n_tiles;
  const int own_n = static_cast<int>(blockIdx.x) % p.n_tiles;

  if (warp >= kProducerWarp) {
    producer_setmaxnreg();
    if (warp == kProducerWarp && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int IJ = p.I * p.J;
      if (p.b_stationary && walk_first < walk_end) {   // the same slices serve every tile of the CTA
        mbar_arrive_expect_tx(&bstat_bar, static_cast<uint32_t>(k_iters) * (p.tx_bytes - p.a_bytes));
        for (int t = 0; t < p.ntaps; ++t)
          for (int cc = 0; cc < p.c_chunks; ++cc)
            tma_load_3d(&tmB, &bstat_bar, sBstat + (t * p.c_chunks + cc) * p.b_bytes, cc * p.ck, p.taps[t].b_tap,
                        p.own_ntile ? own_n * BN : 0);
      }
      // the ring is filled in tile order; the consumer warpgroups take the CTA's tiles alternately
      for (int tile = walk_first; tile < walk_end; tile += walk_step) {
        const int m_tile = p.own_ntile ? tile : tile / p.n_tiles;
        const int n_tile = p.own_ntile ? own_n : tile - m_tile * p.n_tiles;
        const int m0 = m_tile * kTileM;
        const int img = m0 / IJ;
        const int rem = m0 - img * IJ;
        const int bi = rem / p.J;
        const int bj = rem - bi * p.J;
        const int base_w = bj * p.trav + p.lower_w;
        const int base_h = bi * p.trav + p.lower_h;
        const int a_c0 = p.window ? (n_tile * BN / p.window) * p.window : 0;
        for (int t = 0; t < p.ntaps; ++t) {
          const TapEntry te = p.taps[t];
          for (int cc = 0; cc < p.c_chunks; ++cc) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            uint8_t* sa = smem + stage * stage_bytes;
            uint8_t* sb = sa + p.a_bytes;
            mbar_arrive_expect_tx(&full_bar[stage], p.b_stationary ? p.a_bytes : p.tx_bytes);
            const int a_c = a_c0 + cc * p.ck;
            if (p.plain_a)  // 1x1 / stride 1: the A operand is a dense [M, C] matrix -> tiled TMA (faster than im2col)
              tma_load_2d(&tmA, &full_bar[stage], sa, a_c, m0);
            else
              tma_load_im2col_4d(&tmA, &full_bar[stage], sa, a_c, base_w, base_h, img, te.off_w, te.off_h);
            if (!p.b_stationary) tma_load_3d(&tmB, &full_bar[stage], sb, cc * p.ck, te.b_tap, n_tile * BN);
            if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
    return;
  }
  consumer_setmaxnreg();

  // ---- consumers, ping-pong: warpgroup wg computes the CTA's tiles local = wg, wg + 2, wg + 4, ... (128 rows x BN
  // columns each).  It issues a tile's MMAs only after the other warpgroup has issued those of the tile before
  // (turn_bar), so while one warpgroup runs its epilogue the other's MMAs run, and the two never compete for the tensor
  // cores with the same tile phase.  Each warpgroup has its own staging tile, residual fetch and statistics.
  const int wg = warp >> 2;
  const int wt = threadIdx.x & 127;                  // thread index inside the warpgroup
  const int r_lo = (warp & 3) * 16 + (lane >> 2);    // this thread's fragment rows of each 64-row half: r_lo, r_lo + 8
  const int c_lo = 2 * (lane & 3);
  const bool leader = wt == 0;
  const uint32_t row_bytes = p.ck * 2;
  const uint64_t proto = make_smem_desc(0, 16, 8 * row_bytes, layout_type_for_row_bytes(row_bytes));
  const uint32_t a_half = (64u * row_bytes) >> 4;   // descriptor offset of rows 64-127 of the A tile
  const int ksteps = p.ck / 16;
  const uint32_t bstat_addr = smem_u32(sBstat);
  constexpr int nbox = BN / 64;
  // fused-statistics bookkeeping (BN = 64 or 128): this thread owns column st_col, rows [st_row0, st_row0 + st_rows)
  // of each tile
  const int st_col = wt % BN;
  constexpr int st_rows = BN;
  const int st_row0 = (wt / BN) * st_rows;
  int st_ntile = -1;
  float st_s1 = 0.f, st_s2 = 0.f;
  const int IJ = p.I * p.J;
  if (p.b_stationary && walk_first < walk_end) mbar_wait(&bstat_bar, 0);

  float acc[2][BN / 2];
  int local = 0;
  for (int tile = walk_first; tile < walk_end; tile += walk_step, ++local) {
    if ((local & 1) != wg) continue;
    const int m_tile = p.own_ntile ? tile : tile / p.n_tiles;
    const int n_tile = p.own_ntile ? own_n : tile - m_tile * p.n_tiles;
    const int nbase = n_tile * BN;
    const int mine = local >> 1;   // this warpgroup's tile count so far
    // this tile's staging buffer: 64-column boxes of [128 rows][128 B]
    uint8_t* epi_w = epi + (wg * p.epi_bufs + (p.epi_bufs == 2 ? (mine & 1) : 0)) * p.epi_bytes;
    if (p.tma_store) {
      // The staging tile is reused: the store of the warpgroup's tile that last used it must have read it (with two
      // buffers, the store of the tile just before may still be reading the other one) and its threads must be done
      // with their statistics reads.  Then the residual tile is fetched into it, landing while the MMAs run.
      if (leader && mine > 0) {
        if (p.epi_bufs == 2) bulk_wait_group_read1();
        else bulk_wait_group_read0();
      }
      named_bar_sync(1 + wg, 128);
      if (leader && p.res != nullptr) {
        fence_proxy_async();
        mbar_arrive_expect_tx(&res_bar[wg], static_cast<uint32_t>(nbox) * kTileM * 128u);
        for (int b = 0; b < nbox; ++b)
          tma_load_2d(&tmR, &res_bar[wg], epi_w + b * (kTileM * 128), nbase + b * 64, m_tile * kTileM);
      }
    }

    // ring position of this tile's first k-block: the producer filled k_iters stages for each earlier tile of the CTA
    const int pos = local * k_iters;
    int stage = pos % p.num_stages;
    uint32_t phase = static_cast<uint32_t>(pos / p.num_stages) & 1u;
    if (local > 0) mbar_wait(&turn_bar[wg], static_cast<uint32_t>((local - 1) >> 1) & 1u);
    wgmma_fence_acc(acc[0]);
    wgmma_fence_acc(acc[1]);
    int prev = 0;
    for (int it = 0; it < k_iters; ++it) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem + stage * stage_bytes);
      const uint64_t da = proto + (a_addr >> 4);
      const uint64_t db = proto + ((p.b_stationary ? bstat_addr + it * p.b_bytes : a_addr + p.a_bytes) >> 4);
      const uint32_t scale0 = it != 0 ? 1u : 0u;
      if (ksteps == 4) igemm_stage_mma<4>(acc, da, db, a_half, scale0);
      else if (ksteps == 2) igemm_stage_mma<2>(acc, da, db, a_half, scale0);
      else igemm_stage_mma<1>(acc, da, db, a_half, scale0);
      wgmma_wait<1>();                                    // the previous iteration's MMAs are done with their stage
      if (it > 0) release_stage(&empty_bar[prev], lane);
      prev = stage;
      if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&turn_bar[wg ^ 1]);      // all MMAs of this tile are issued: the other warpgroup's turn
    wgmma_wait<0>();
    wgmma_fence_acc(acc[0]);
    wgmma_fence_acc(acc[1]);
    release_stage(&empty_bar[prev], lane);

    if (p.tma_store) {
      if constexpr (BN % 64 == 0) {
        // Dense bf16 output: stage the tile in 128B-swizzled shared memory and write it with TMA (coalesced, clipped at
        // the M tail); the residual was fetched into the same buffer.
        if (p.res != nullptr) mbar_wait(&res_bar[wg], static_cast<uint32_t>(mine & 1));
        if (p.bias != nullptr || p.act != B200_ACT_NONE) stage_tile<BN, 0, false>(epi_w, acc, p, nbase, r_lo, c_lo);
        else if (p.res != nullptr) stage_tile<BN, 1, true>(epi_w, acc, p, nbase, r_lo, c_lo);
        else stage_tile<BN, 1, false>(epi_w, acc, p, nbase, r_lo, c_lo);
        fence_proxy_async();                             // generic-proxy smem writes -> visible to TMA
        named_bar_sync(1 + wg, 128);
        if (leader) {
          for (int b = 0; b < nbox; ++b)
            tma_store_2d(&tmC, epi_w + b * (kTileM * 128), nbase + b * 64, m_tile * kTileM);
          bulk_commit_group();
        }
        if constexpr (BN == 64 || BN == 128) {
          if (p.stats != nullptr) {
            // Fused BN statistics: per-channel sum / sum of squares of the bf16-rounded outputs of this tile, read
            // back from the staged tile (rows beyond M_total are exact zeros).  Accumulated in registers across the
            // warpgroup's tiles while it stays on the same channel block, then one fp64 atomic each.
            if (st_ntile != n_tile) {
              if (st_ntile >= 0) {
                flush_bn_stats(p.stats, p.N_total, st_ntile * BN, st_col, st_s1, st_s2);
                st_s1 = 0.f; st_s2 = 0.f;
              }
              st_ntile = n_tile;
            }
            float s1 = 0.f, s2 = 0.f;
#pragma unroll 8
            for (int r = st_row0; r < st_row0 + st_rows; ++r) {
              const float vv = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(epi_w + staged_offset(r, st_col, kTileM * 128)));
              s1 += vv;
              s2 = fmaf(vv, vv, s2);
            }
            st_s1 += s1;
            st_s2 += s2;
          }
        }
      }
      continue;
    }
    // bf16 output, no bias or activation, no column tail (the strided data gradients): stored without a branch per value
    const bool plain = !p.out_fp32 && p.bias == nullptr && p.act == B200_ACT_NONE && (p.ldo & 1) == 0 &&
                       nbase + BN <= p.N_total;
#pragma unroll
    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m_tile * kTileM + mh * 64 + r_lo + 8 * h;
        if (m >= p.M_total) continue;
        const int img = m / IJ;
        const int rem = m - img * IJ;
        const int bi = rem / p.J;
        const int bj = rem - bi * p.J;
        const long long off = ((static_cast<long long>(img) * p.OH + (bi * p.os + p.oh0)) * p.OW + (bj * p.os + p.ow0)) *
                              static_cast<long long>(p.ldo);
        if (plain && p.res != nullptr) store_row_bf16<BN, true>(p, acc[mh], h, off + nbase + c_lo);
        else if (plain) store_row_bf16<BN, false>(p, acc[mh], h, off + nbase + c_lo);
        else {
#pragma unroll
          for (int j = 0; j < BN / 2; j += 4) store_pair(p, acc[mh][j + 2 * h], acc[mh][j + 2 * h + 1], off, nbase + 2 * j + c_lo);
        }
      }
  }
  if constexpr (BN == 64 || BN == 128)
    if (p.stats != nullptr && st_ntile >= 0) flush_bn_stats(p.stats, p.N_total, st_ntile * BN, st_col, st_s1, st_s2);
  if (p.tma_store && leader) bulk_wait_group0();  // smem must outlive the last TMA store
}

// ------------------------------------------------------------------------------------------------
// wgrad: dw[k, tap, c] += sum_pix dy[pix, k] * x[pix @ tap, c]
// A = dy tile, MN-major (rows of smem = pixels, 128/64/32B of k-channels); B = im2col(x) tile, MN-major.
// A CTA owns 128 output channels (one k-tile) x boxes_per_cta channel boxes of x (at most 256 accumulator columns).
constexpr int kBk = 64;   // pixels per wgrad stage: four 16-deep k-steps
struct WgradParams {
  int M_total;          // fwd output pixels N*P*Q
  int P, Q;
  int trav;             // conv stride
  int lower_w, lower_h; // -pad
  int K_out, C, taps_total;
  int ckA, ckB;         // channels per smem box on the dy side / x side
  int bk;               // pixels per stage
  int c_chunks;         // ceil(C / ckB)
  int total_boxes;      // taps * c_chunks
  int boxes_per_cta;    // boxes_per_cta * ckB <= 256 accumulator columns, <= 8
  int k_tiles, col_groups, splits;
  int blocks_per_split, total_blocks;  // in units of bk pixels
  int num_stages;
  uint32_t boxA_bytes, boxB_bytes, stage_bytes;
  float* dw;
  int plain_x;           // 1: x is a dense [M_total, C] matrix (1x1 stride 1): tiled TMA instead of im2col
  float* partial;        // split-K partial tiles [tile][split][128][pitch] (nullptr: splits == 1, add into dw)
  int pitch;             // boxes_per_cta * ckB
  int window;            // 0 dense; 128: k-tile t pairs with source channels [128t, 128t+128) only
  int S_filter;          // filter width: tap t = (r, s) = (t / S, t % S) gives the im2col offsets {s, r}
};

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// NC = boxes_per_cta * ckB, the accumulator width: the last column group may hold fewer boxes (ncols < NC); its
// missing columns are computed from whatever the stage holds and never stored.  The grid is one wave (splits fill the
// SMs), so those CTAs take no longer than the full-width ones beside them.
template <int NC>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                  const __grid_constant__ WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumers / 32);
    }
    fence_mbar_init();
    prefetch_tmap(&tmDy);
    prefetch_tmap(&tmX);
  }
  __syncthreads();

  // work decomposition
  const int tiles = p.k_tiles * p.col_groups;
  const int split = blockIdx.x / tiles;
  const int tile = blockIdx.x - split * tiles;
  const int k_tile = tile % p.k_tiles;
  const int cgroup = tile / p.k_tiles;
  const int k0 = k_tile * kTileM;
  const int box0 = cgroup * p.boxes_per_cta;
  const int nboxes = min(p.boxes_per_cta, p.total_boxes - box0);
  const int blk_begin = split * p.blocks_per_split;
  const int blk_end = min(p.total_blocks, blk_begin + p.blocks_per_split);
  const int nblk = blk_end - blk_begin;
  const uint32_t a_tile = (kTileM / p.ckA) * p.boxA_bytes;   // one k-tile of dy: 128 channels x bk pixels
  if (nblk <= 0) return;

  if (warp >= kProducerWarp) {
    producer_setmaxnreg();
    if (warp == kProducerWarp && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int PQ = p.P * p.Q;
      // everything that does not depend on the pixel block is computed once: the producer thread's issue rate bounds
      // the HBM-bound layers (one TMA request per 8 KB box)
      const int nA = min(kTileM / p.ckA, (p.K_out - k0 + p.ckA - 1) / p.ckA);   // dy boxes present (K_out tail)
      int box_c[8];
      uint16_t box_w[8], box_h[8];
      for (int x = 0; x < 8; ++x) {
        const int id = box0 + min(x, nboxes - 1);
        const int t = id / p.c_chunks;
        const int th = t / p.S_filter;
        box_c[x] = (id - t * p.c_chunks) * p.ckB + (p.window ? k0 : 0);
        box_w[x] = static_cast<uint16_t>(t - th * p.S_filter);
        box_h[x] = static_cast<uint16_t>(th);
      }
      const uint32_t tx = nA * p.boxA_bytes + nboxes * p.boxB_bytes;
      for (int b = blk_begin; b < blk_end; ++b) {
        const int pix0 = b * p.bk;
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        uint8_t* sa = smem + stage * p.stage_bytes;
        uint8_t* sb = sa + a_tile;
        mbar_arrive_expect_tx(&full_bar[stage], tx);
        for (int a = 0; a < nA; ++a)
          tma_load_2d(&tmDy, &full_bar[stage], sa + a * p.boxA_bytes, k0 + a * p.ckA, pix0);
        if (p.plain_x) {
#pragma unroll
          for (int x = 0; x < 8; ++x)
            if (x < nboxes) tma_load_2d(&tmX, &full_bar[stage], sb + x * p.boxB_bytes, box_c[x], pix0);
        } else {
          const int img = pix0 / PQ;
          const int rem = pix0 - img * PQ;
          const int pi = rem / p.Q;
          const int pj = rem - pi * p.Q;
          const int base_w = pj * p.trav + p.lower_w;
          const int base_h = pi * p.trav + p.lower_h;
#pragma unroll
          for (int x = 0; x < 8; ++x)
            if (x < nboxes)
              tma_load_im2col_4d(&tmX, &full_bar[stage], sb + x * p.boxB_bytes, box_c[x], base_w, base_h, img, box_w[x],
                                 box_h[x]);
        }
        if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  consumer_setmaxnreg();

  // ---- consumers: warpgroup wg computes output channels [k0 + 64 wg, k0 + 64 wg + 64) x all boxes of the CTA
  const int wg = warp >> 2;
  const bool wg_on = k0 + wg * 64 < p.K_out;
  const int ncols = nboxes * p.ckB;
  // A rows 64 wg.. start at dy box 64 wg / ckA; MN-major: LBO = box stride along M/N, SBO = 8 pixel rows
  const uint64_t protoA = make_smem_desc(0, p.boxA_bytes, 8 * p.ckA * 2, layout_type_for_row_bytes(p.ckA * 2));
  const uint64_t protoB = make_smem_desc(0, p.boxB_bytes, 8 * p.ckB * 2, layout_type_for_row_bytes(p.ckB * 2));
  const uint32_t a_wg = (wg * (64 / p.ckA) * p.boxA_bytes) >> 4;
  const uint32_t kincA = (16u * p.ckA * 2) >> 4, kincB = (16u * p.ckB * 2) >> 4;  // 16 pixel rows per K step
  float acc[NC / 2];
  wgmma_fence_acc(acc);
  int stage = 0, prev = 0;
  uint32_t phase = 0;
  for (int b = 0; b < nblk; ++b) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t a_addr = smem_u32(smem + stage * p.stage_bytes);
    if (wg_on) {
      const uint64_t da = protoA + (a_addr >> 4) + a_wg, db = protoB + ((a_addr + a_tile) >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBk / 16; ++k)
        wgmma_bf16<1, 1>(acc, da + k * kincA, db + k * kincB, (b | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
    }
    if (b > 0) release_stage(&empty_bar[prev], lane);
    prev = stage;
    if (++stage == p.num_stages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  wgmma_fence_acc(acc);
  release_stage(&empty_bar[prev], lane);
  if (!wg_on) return;

  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows r_lo, r_lo + 8 (output channels)
  const int c_lo = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = k0 + r_lo + 8 * h;
    if (k >= p.K_out) continue;
    if (p.partial != nullptr) {
      // split-K: plain stores of this CTA's fp32 tile; launch_wgrad_reduce sums the splits into dw
      float* dst = p.partial + ((static_cast<long long>(tile) * p.splits + split) * kTileM + (r_lo + 8 * h)) * p.pitch;
#pragma unroll
      for (int j = 0; j < NC / 2; j += 4)
        if (2 * j < ncols)
          *reinterpret_cast<float2*>(dst + 2 * j + c_lo) = make_float2(acc[j + 2 * h], acc[j + 2 * h + 1]);
    } else {
#pragma unroll
      for (int j = 0; j < NC / 2; j += 4) {
        const int col = 2 * j + c_lo;
        if (col < ncols) {
          const int x = col / p.ckB;
          const int id = box0 + x;
          const int tap = id / p.c_chunks;
          const int c = (id - tap * p.c_chunks) * p.ckB + (col - x * p.ckB);
          if (c < p.C) red_add_v2(p.dw + (static_cast<long long>(k) * p.taps_total + tap) * p.C + c, acc[j + 2 * h],
                                  acc[j + 2 * h + 1]);
        }
      }
    }
  }
}

// dw[k][tap][c] += sum over splits of the partial tiles of both weight-gradient kernels (fixed order => deterministic;
// layout in host.h, launch_wgrad_reduce).  A block owns 32 consecutive float4 outputs; its nw warps each sum every
// nw-th split (coalesced 512 B reads) and combine through shared memory -- with one thread per output the loop over up
// to 148 splits was a serial chain of L2 round trips.
__global__ void __launch_bounds__(256) conv_wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw,
                                                                int K_out, int taps, int C, int ck, int tap_stride,
                                                                int cc_stride, int bpc, int k_tiles, int splits,
                                                                int pitch) {
  __shared__ float4 red[8][32];
  const int c4n = C >> 2;
  const long long total = static_cast<long long>(K_out) * taps * c4n;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (long long base = static_cast<long long>(blockIdx.x) * 32; base < total; base += static_cast<long long>(gridDim.x) * 32) {
    const long long idx = base + lane;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int c = 0, tap = 0, k = 0;
    if (idx < total) {
      c = static_cast<int>(idx % c4n) * 4;
      tap = static_cast<int>((idx / c4n) % taps);
      k = static_cast<int>(idx / (static_cast<long long>(c4n) * taps));
      const int k_tile = k / kTileM, row = k - k_tile * kTileM;
      const int cc = c / ck;
      const int id = tap * tap_stride + cc * cc_stride;
      const int cgroup = id / bpc, x = id - cgroup * bpc;
      const int unit = cgroup * k_tiles + k_tile;
      const float* src = partial + ((static_cast<long long>(unit) * splits) * kTileM + row) * pitch + x * ck + (c - cc * ck);
      for (int s2 = w; s2 < splits; s2 += nw) {
        const float4 v = __ldcg(reinterpret_cast<const float4*>(src + static_cast<long long>(s2) * kTileM * pitch));
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    red[w][lane] = acc;
    __syncthreads();
    if (w == 0 && idx < total) {
      for (int j = 1; j < nw; ++j) {
        const float4 v = red[j][lane];
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      float4* o = reinterpret_cast<float4*>(dw + (static_cast<long long>(k) * taps + tap) * C + c);
      float4 cur = *o;
      cur.x += acc.x; cur.y += acc.y; cur.z += acc.z; cur.w += acc.w;
      *o = cur;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// host side
static int pick_ck(int channels) { return channels <= 16 ? 16 : (channels <= 32 ? 32 : 64); }

static int encode_im2col(CUtensorMap* tm, const void* base, int Nimg, int H, int W, int C, int ck, int pixels,
                         int lower_w, int lower_h, int upper_w, int upper_h, int trav, long long pix_stride = 0,
                         long long row_stride = 0, long long img_stride = 0) {
  EncodeIm2colFn fn = encode_im2col_fn();
  B200_REQUIRE(fn != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeIm2col entry point unavailable");
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)Nimg};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  if (pix_stride > 0) {  // explicit (possibly overlapping) layout, in elements
    strides[0] = (cuuint64_t)pix_stride * 2;
    strides[1] = (cuuint64_t)row_stride * 2;
    strides[2] = (cuuint64_t)img_stride * 2;
  }
  int lower[2] = {lower_w, lower_h};
  int upper[2] = {upper_w, upper_h};
  cuuint32_t estr[4] = {1, (cuuint32_t)trav, (cuuint32_t)trav, 1};
  B200_REQUIRE(lower_w >= -128 && lower_w <= 127 && lower_h >= -128 && lower_h <= 127 && upper_w >= -128 &&
                   upper_w <= 127 && upper_h >= -128 && upper_h <= 127,
               B200_ERR_UNSUPPORTED, "im2col corner offsets out of the TMA range");
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, lower, upper,
                  (cuuint32_t)ck, (cuuint32_t)pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_for_row_bytes(ck * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, B200_ERR_CUDA,
               "cuTensorMapEncodeIm2col failed (%d) N=%d H=%d W=%d C=%d ck=%d pix=%d lower=(%d,%d) upper=(%d,%d) trav=%d",
               (int)r, Nimg, H, W, C, ck, pixels, lower_w, lower_h, upper_w, upper_h, trav);
  // Driver quirk for small tensors (as worked around by CUTLASS' im2col descriptor builder):
  // for tensors below 128 KiB, bit 21 of the second descriptor word must be cleared on drivers <= 13.1.
  int drv = 0;
  cudaDriverGetVersion(&drv);
  if (drv <= 13010 && (size_t)Nimg * H * W * C * 2 < 131072) {
    reinterpret_cast<uint64_t*>(tm)[1] &= ~(1ull << 21);
  }
  return B200_OK;
}

static const int kSmemBudget = 200 * 1024;
static const int kSmemBudgetMax = 224 * 1024;   // + 1 KB alignment slack + static barriers < the 227 KB per-CTA limit

int launch_wgrad_reduce(const float* partial, float* dw, int K_out, int taps, int C, int ck, int tap_stride,
                        int cc_stride, int bpc, int k_tiles, int splits, int pitch, cudaStream_t stream) {
  const long long total = static_cast<long long>(K_out) * taps * (C / 4);
  long long blocks = (total + 31) / 32;
  if (blocks > 16LL * sm_count()) blocks = 16LL * sm_count();
  int warps = 8;
  while (warps > 1 && warps > splits) warps >>= 1;   // no idle warps when there are only a few splits
  b200::launch(conv_wgrad_reduce_kernel, static_cast<int>(blocks), 32 * warps, 0, stream, partial, dw, K_out, taps, C, ck,
               tap_stride, cc_stride, bpc, k_tiles, splits, pitch);
  B200_CHECK_LAUNCH("conv_wgrad_reduce_kernel");
  return B200_OK;
}

// One implicit-GEMM launch.  src: [Nimg, SH, SW, SC] bf16 (im2col source); wmat: [Nout][wtaps][SC] bf16.
struct IgemmLaunch {
  const void* src; int Nimg, SH, SW, SC;
  long long s_pix, s_row, s_img;   // optional explicit source strides (elements), 0 = dense
  const void* wmat; int Nout, wtaps;
  int I, J, trav, lower_w, lower_h;
  int ntaps; TapEntry taps[kMaxTaps];
  void* out; int OH, OW, os, oh0, ow0, ldo;
  const void* res; const float* bias; int act, out_fp32;
  double* stats;
  int window;
};

// The instantiations of a kernel templated on its tile width (16 * (I + 1) for I in Is), indexed by width.
template <int... Is>
static auto igemm_kernel_for(int block_n, std::integer_sequence<int, Is...>) {
  static constexpr decltype(&conv_igemm_kernel<16>) table[] = {&conv_igemm_kernel<16 * (Is + 1)>...};
  return table[block_n / 16 - 1];
}
// The weight-gradient widths b200_conv_wgrad reaches: boxes_per_cta * ckB with ckB in {16, 32, 64} and
// boxes_per_cta <= min(8, 256 / ckB), i.e. 16..128 in steps of 16 and 160, 192, 224, 256.
static auto wgrad_kernel_for(int ncols) {
  static constexpr decltype(&conv_wgrad_kernel<16>) table[] = {
      &conv_wgrad_kernel<16>,  &conv_wgrad_kernel<32>,  &conv_wgrad_kernel<48>,  &conv_wgrad_kernel<64>,
      &conv_wgrad_kernel<80>,  &conv_wgrad_kernel<96>,  &conv_wgrad_kernel<112>, &conv_wgrad_kernel<128>,
      nullptr,                 &conv_wgrad_kernel<160>, nullptr,                 &conv_wgrad_kernel<192>,
      nullptr,                 &conv_wgrad_kernel<224>, nullptr,                 &conv_wgrad_kernel<256>};
  return table[ncols / 16 - 1];
}

static int launch_igemm(const IgemmLaunch& L, cudaStream_t stream) {
  B200_REQUIRE(L.SC % 8 == 0, B200_ERR_UNSUPPORTED, "igemm: source channels (%d) must be a multiple of 8", L.SC);
  B200_REQUIRE(L.ntaps >= 1 && L.ntaps <= kMaxTaps, B200_ERR_UNSUPPORTED, "igemm: %d taps unsupported", L.ntaps);
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.M_total = L.Nimg * L.I * L.J;
  B200_REQUIRE(p.M_total > 0, B200_ERR_INVALID, "igemm: empty problem");
  p.I = L.I; p.J = L.J; p.trav = L.trav; p.lower_w = L.lower_w; p.lower_h = L.lower_h;
  p.N_total = L.Nout;
  // n-tiles of at most 128 columns (a warpgroup's 128 x block_n tile is block_n accumulator registers per thread):
  // 128 or 64 wide when that divides Nout, which keeps the TMA-store epilogue and computes no padding columns;
  // otherwise the fewest equal tiles, rounded up to 16 columns
  p.block_n = L.Nout % 128 == 0 ? 128 : (L.Nout % 64 == 0 ? 64 : 0);
  if (p.block_n == 0) {
    const int nt = (L.Nout + 127) / 128;
    p.block_n = (((L.Nout + nt - 1) / nt) + 15) / 16 * 16;
  }
  p.n_tiles = (L.Nout + p.block_n - 1) / p.block_n;
  p.m_tiles = (p.M_total + kTileM - 1) / kTileM;
  p.ck = pick_ck(L.SC);
  p.c_chunks = (L.SC + p.ck - 1) / p.ck;
  p.window = L.window;
  if (L.window) {   // block-diagonal: one 64-wide n-tile per window, the K loop covers the window's channels only
    B200_REQUIRE(L.window == 64 && L.SC == L.Nout && L.Nout % 64 == 0, B200_ERR_UNSUPPORTED,
                 "igemm: window %d needs window 64, C == K (C=%d K=%d), K %% 64 == 0", L.window, L.SC, L.Nout);
    p.block_n = 64;
    p.n_tiles = L.Nout / 64;
    p.ck = 64;
    p.c_chunks = 1;
  }
  p.ntaps = L.ntaps;
  p.a_bytes = kTileM * p.ck * 2;
  p.b_bytes = p.block_n * p.ck * 2;
  p.tx_bytes = p.a_bytes + p.b_bytes;
  // keep every stage 1024B aligned (128B-swizzle atoms are 1024B)
  uint32_t stage = p.a_bytes + p.b_bytes;
  if (stage % 1024) { p.b_bytes += 1024 - stage % 1024; stage = p.a_bytes + p.b_bytes; }
  // dense bf16 outputs with 64-channel granularity go out through shared memory + TMA store
  p.tma_store = (L.os == 1 && !L.out_fp32 && (p.block_n % 64) == 0 && (L.Nout % p.block_n) == 0 && L.ldo == L.Nout &&
                 L.OH == L.I && L.OW == L.J && L.oh0 == 0 && L.ow0 == 0) ? 1 : 0;
  const int epi_bytes = p.tma_store ? kTileM * p.block_n * 2 : 0;   // per staging tile
  // A tile that stores at least as many bytes as it loads (the expanding 1x1 layers and their data gradients with
  // C <= 128) is bound by its output stream.  With one staging tile per warpgroup, each epilogue first waits for the
  // warpgroup's previous TMA store to drain, so only about one store per warpgroup is in flight; two staging tiles let
  // the next epilogue start while that store is still leaving.
  const int k_iters = L.ntaps * p.c_chunks;
  p.epi_bufs = (p.tma_store && k_iters * (int)p.a_bytes <= epi_bytes) ? 2 : 1;
  int epi_total = 2 * p.epi_bufs * epi_bytes;
  // small 1x1 layers (all weight slices <= 64 KB): keep the weights resident, stream only the activations
  const int b_all = L.ntaps * p.c_chunks * (int)p.b_bytes;
  int bstat_bytes = 0;
  if (p.n_tiles == 1 && !L.window && (p.a_bytes % 1024) == 0 && (p.b_bytes % 1024) == 0 && b_all <= 64 * 1024) {
    p.b_stationary = 1;
    bstat_bytes = b_all;
    stage = p.a_bytes;
  }
  // several n-tiles whose weights fit one at a time: a CTA owns an n-tile.  Worth it when the weights dominate the
  // L2->SM traffic of the round-robin walk (bytes ~ A * n_tiles + W * m_tiles vs A * n_tiles + W_tile * CTAs) and
  // every CTA still gets a few m-tiles; needs >= 3 operand stages beside the resident weights and the staging tile.
  int grid_own = 0;
  if (!p.b_stationary && p.n_tiles > 1 && p.n_tiles <= 8 && !L.window &&
      (p.a_bytes % 1024) == 0 && (p.b_bytes % 1024) == 0 && (L.Nout % p.block_n) == 0) {
    const int ctas = sm_count() / p.n_tiles;
    const long long a_all = (long long)p.M_total * L.SC * 2 * L.ntaps;
    const long long w_all = (long long)b_all * p.n_tiles;
    const long long rr_bytes = a_all * p.n_tiles + w_all * p.m_tiles;
    const long long own_bytes = a_all * p.n_tiles + (long long)b_all * ctas * p.n_tiles;
    const int stages_left = (kSmemBudgetMax - epi_total - b_all) / (int)p.a_bytes;
    if (ctas >= 1 && p.m_tiles >= 4 * ctas && stages_left >= 3 && own_bytes * 4 <= rr_bytes * 3) {
      p.b_stationary = 1;
      p.own_ntile = 1;
      bstat_bytes = b_all;
      stage = p.a_bytes;
      grid_own = ctas * p.n_tiles;
    }
  }
  p.epi_bytes = (uint32_t)epi_bytes;
  p.num_stages = (kSmemBudgetMax - epi_total - bstat_bytes) / (int)stage;
  if (p.epi_bufs == 2 && p.num_stages < 2 * k_iters) {   // the ring must still hold two tiles' operands
    p.epi_bufs = 1;
    epi_total = 2 * epi_bytes;
    p.num_stages = (kSmemBudgetMax - epi_total - bstat_bytes) / (int)stage;
  }
  if (p.num_stages > kMaxStages) p.num_stages = kMaxStages;
  if (p.num_stages < 2) p.num_stages = 2;
  p.OH = L.OH; p.OW = L.OW; p.os = L.os; p.oh0 = L.oh0; p.ow0 = L.ow0; p.ldo = L.ldo;
  p.act = L.act; p.out_fp32 = L.out_fp32; p.out = L.out; p.res = L.res; p.bias = L.bias;
  p.stats = L.stats;
  if (L.stats != nullptr)
    B200_REQUIRE(p.tma_store && (128 % p.block_n) == 0 && L.res == nullptr && L.bias == nullptr && L.act == 0,
                 B200_ERR_UNSUPPORTED, "conv_fprop: fused BN statistics need a dense bf16 output with K %% 64 == 0 "
                 "(block_n=%d) and no bias/residual/activation", p.block_n);
  for (int t = 0; t < L.ntaps; ++t) p.taps[t] = L.taps[t];

  // bounding box of base pixels: [lower, lower + (I-1)*trav] in a source of extent SH x SW
  const int upper_w = L.lower_w + (L.J - 1) * L.trav + 1 - L.SW;
  const int upper_h = L.lower_h + (L.I - 1) * L.trav + 1 - L.SH;
  CUtensorMap tmA, tmB;
  int rc;
  p.plain_a = (L.ntaps == 1 && L.trav == 1 && L.lower_w == 0 && L.lower_h == 0 && L.taps[0].off_w == 0 &&
               L.taps[0].off_h == 0 && L.I == L.SH && L.J == L.SW && L.s_pix == 0) ? 1 : 0;
  if (p.plain_a)
    rc = encode_tiled(&tmA, L.src, 2, {L.SC, p.M_total}, {p.ck, kTileM}, "igemm A");
  else
    rc = encode_im2col(&tmA, L.src, L.Nimg, L.SH, L.SW, L.SC, p.ck, kTileM, L.lower_w, L.lower_h, upper_w, upper_h,
                       L.trav, L.s_pix, L.s_row, L.s_img);
  if (rc) return rc;
  rc = encode_tiled(&tmB, L.wmat, 3, {L.window ? L.window : L.SC, L.wtaps, L.Nout}, {p.ck, 1, p.block_n}, "igemm B");
  if (rc) return rc;

  CUtensorMap tmC, tmR;
  memset(&tmC, 0, sizeof(tmC));
  memset(&tmR, 0, sizeof(tmR));
  if (p.tma_store) {
    rc = encode_tiled(&tmC, L.out, 2, {L.ldo, p.M_total}, {64, kTileM}, "igemm output");
    if (rc) return rc;
    if (L.res != nullptr) {
      rc = encode_tiled(&tmR, L.res, 2, {L.ldo, p.M_total}, {64, kTileM}, "igemm residual");
      if (rc) return rc;
    }
  }
  const int smem_bytes = p.num_stages * (int)stage + bstat_bytes + epi_total + 1024;
  const auto kfn = igemm_kernel_for(p.block_n, std::make_integer_sequence<int, 8>{});
  rc = set_smem_attr((const void*)kfn, smem_bytes);
  if (rc) return rc;
  // With fewer tiles than SMs a CTA gets one tile and its second consumer warpgroup idles: the tiles are spread over
  // all SMs rather than paired up on half of them.
  const int total_tiles = p.m_tiles * p.n_tiles;
  const int grid = grid_own ? grid_own : (total_tiles < sm_count() ? total_tiles : sm_count());
  if (getenv("B200_IGEMM_DEBUG")) {
    // max_tiles: tiles of the busiest CTA (its warpgroups take them alternately, so >= 2 means warpgroup 1 computes)
    const int max_tiles = p.own_ntile ? (p.m_tiles + grid / p.n_tiles - 1) / (grid / p.n_tiles)
                                      : (total_tiles + grid - 1) / grid;
    fprintf(stderr, "[igemm] M=%d C=%d N=%d taps=%d os=%d block_n=%d n_tiles=%d m_tiles=%d ck=%d k_iters=%d stages=%d "
            "tma_store=%d plain_a=%d bstat=%d own=%d out_fp32=%d bias=%d res=%d act=%d stats=%d grid=%d max_tiles=%d "
            "smem=%d window=%d xs=%d epi_bufs=%d\n",
            p.M_total, L.SC, L.Nout, L.ntaps, L.os, p.block_n, p.n_tiles, p.m_tiles, p.ck, L.ntaps * p.c_chunks,
            p.num_stages, p.tma_store, p.plain_a, p.b_stationary, p.own_ntile, p.out_fp32, L.bias != nullptr,
            L.res != nullptr, p.act, L.stats != nullptr, grid, max_tiles, smem_bytes, L.window, (int)L.s_pix,
            p.epi_bufs);
  }
  b200::launch(kfn, grid, kThreads, smem_bytes, stream, tmA, tmB, tmC, tmR, p);
  B200_CHECK_LAUNCH("conv_igemm_kernel");
  return B200_OK;
}

static int check_desc(const b200_conv_desc* d) {
  B200_REQUIRE(d != nullptr, B200_ERR_INVALID, "conv: null descriptor");
  B200_REQUIRE(d->N > 0 && d->H > 0 && d->W > 0 && d->C > 0 && d->K > 0 && d->R > 0 && d->S > 0 && d->P > 0 &&
                   d->Q > 0 && d->stride >= 1 && d->stride <= 8,
               B200_ERR_INVALID, "conv: bad descriptor N=%d H=%d W=%d C=%d K=%d R=%d S=%d P=%d Q=%d stride=%d", d->N,
               d->H, d->W, d->C, d->K, d->R, d->S, d->P, d->Q, d->stride);
  B200_REQUIRE(d->R * d->S <= kMaxTaps, B200_ERR_UNSUPPORTED, "conv: %dx%d filter exceeds %d taps", d->R, d->S,
               kMaxTaps);
  B200_REQUIRE((d->x_pixel_stride == 0 && d->x_row_stride == 0 && d->x_image_stride == 0) ||
                   (d->x_pixel_stride > 0 && d->x_pixel_stride % 8 == 0 && d->x_row_stride % 8 == 0 &&
                    d->x_image_stride % 8 == 0 && d->x_row_stride > 0 && d->x_image_stride > 0),
               B200_ERR_INVALID, "conv: x strides must all be 0 (dense) or positive multiples of 8 elements");
  B200_REQUIRE(d->window == 0 || (d->window % 64 == 0 && d->C == d->K && d->C % d->window == 0 && d->x_pixel_stride == 0),
               B200_ERR_UNSUPPORTED, "conv: window %d needs C == K, C %% window == 0 (C=%d K=%d)", d->window, d->C, d->K);
  return B200_OK;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_conv_fprop(const b200_conv_desc* d, const void* x, const void* w, void* y,
                               const b200_epilogue* ep, b200_stream_t stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  B200_REQUIRE(x && w && y, B200_ERR_INVALID, "conv_fprop: null pointer");
  B200_REQUIRE(d->C % 8 == 0, B200_ERR_UNSUPPORTED, "conv_fprop: C=%d must be a multiple of 8 (pad the input)", d->C);
  B200_REQUIRE(d->window == 0 || d->window == 64, B200_ERR_UNSUPPORTED, "conv_fprop: window must be 0 or 64");
  if (d->stride == 1 && d->pad_h == d->pad_w && d->P == d->H + 2 * d->pad_h - d->R + 1 &&
      d->Q == d->W + 2 * d->pad_w - d->S + 1 && d->x_pixel_stride == 0 && (!ep || !ep->out_fp32) &&
      !(ep && ep->bias && ep->bn_stats_workspace) && (d->window == 0 || d->window == 64) &&
      halo_eligible(d->P, d->Q, d->C, d->K, d->R, d->S, d->pad_h)) {
    return launch_halo(x, w, y, ep ? ep->residual : nullptr, ep ? ep->bias : nullptr, d->N, d->P, d->Q, d->C, d->K,
                       d->R, d->S, d->pad_h, 0, ep ? ep->act : 0,
                       (ep && ep->bn_stats_workspace) ? reinterpret_cast<double*>(ep->bn_stats_workspace) : nullptr,
                       (cudaStream_t)stream, d->window);
  }
  IgemmLaunch L;
  memset(&L, 0, sizeof(L));
  L.src = x; L.Nimg = d->N; L.SH = d->H; L.SW = d->W; L.SC = d->C;
  L.s_pix = d->x_pixel_stride; L.s_row = d->x_row_stride; L.s_img = d->x_image_stride;
  L.wmat = w; L.Nout = d->K; L.wtaps = d->R * d->S;
  L.I = d->P; L.J = d->Q; L.trav = d->stride; L.lower_w = -d->pad_w; L.lower_h = -d->pad_h;
  L.ntaps = d->R * d->S;
  for (int r = 0; r < d->R; ++r)
    for (int s = 0; s < d->S; ++s) {
      TapEntry& t = L.taps[r * d->S + s];
      t.off_w = (uint16_t)s; t.off_h = (uint16_t)r; t.b_tap = (uint16_t)(r * d->S + s); t.pad_ = 0;
    }
  L.out = y; L.OH = d->P; L.OW = d->Q; L.os = 1; L.oh0 = 0; L.ow0 = 0; L.ldo = d->K;
  L.res = ep ? ep->residual : nullptr;
  L.bias = ep ? ep->bias : nullptr;
  L.act = ep ? ep->act : 0;
  L.out_fp32 = ep ? ep->out_fp32 : 0;
  L.stats = (ep && ep->bn_stats_workspace) ? reinterpret_cast<double*>(ep->bn_stats_workspace) : nullptr;
  L.window = d->window;
  return launch_igemm(L, (cudaStream_t)stream);
}

extern "C" int b200_conv_dgrad(const b200_conv_desc* d, const void* dy, const void* wt, void* dx,
                               const void* residual, b200_stream_t stream_) {
  int rc = check_desc(d);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  B200_REQUIRE(dy && wt && dx, B200_ERR_INVALID, "conv_dgrad: null pointer");
  B200_REQUIRE(d->K % 8 == 0, B200_ERR_UNSUPPORTED, "conv_dgrad: K=%d must be a multiple of 8", d->K);
  B200_REQUIRE(d->window == 0 || d->window == 64, B200_ERR_UNSUPPORTED, "conv_dgrad: window must be 0 or 64");
  const int st = d->stride;
  B200_REQUIRE(st == 1 || st == 2, B200_ERR_UNSUPPORTED, "conv_dgrad: stride %d unsupported", st);
  if (d->R == 3 && d->S == 3 && st == 1 && d->pad_h == 1 && d->pad_w == 1 && d->P == d->H && d->Q == d->W &&
      (d->window == 0 || d->window == 64) && halo_eligible(d->H, d->W, d->K, d->C, 3, 3, 1)) {
    return launch_halo(dy, wt, dx, residual, nullptr, d->N, d->H, d->W, d->K, d->C, 3, 3, 1, 1, 0, nullptr, stream,
                       d->window);
  }
  // dx[h,w] = sum_{r,s : (h+pad-r) % st == 0} dy[(h+pad-r)/st, (w+pad-s)/st] * w[r,s]
  // one launch per residue class (h % st, w % st); each class is a stride-1 correlation over dy.
  bool any_empty = false;
  for (int ph = 0; ph < st; ++ph)
    for (int pw = 0; pw < st; ++pw) {
      int nr = 0, ns = 0;
      for (int r = 0; r < d->R; ++r) if (((ph + d->pad_h - r) % st + st) % st == 0) ++nr;
      for (int s = 0; s < d->S; ++s) if (((pw + d->pad_w - s) % st + st) % st == 0) ++ns;
      if (nr * ns == 0 && (d->H - ph + st - 1) / st > 0 && (d->W - pw + st - 1) / st > 0) any_empty = true;
    }
  if (any_empty) {
    B200_REQUIRE(residual == nullptr, B200_ERR_UNSUPPORTED,
                 "conv_dgrad: residual add with an empty stride class is unsupported");
    cudaError_t e = cudaMemsetAsync(dx, 0, (size_t)d->N * d->H * d->W * d->C * 2, stream);
    B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "conv_dgrad: memset failed: %s", cudaGetErrorString(e));
    count_launch();
  }
  for (int ph = 0; ph < st; ++ph)
    for (int pw = 0; pw < st; ++pw) {
      const int I = (d->H - ph + st - 1) / st;
      const int J = (d->W - pw + st - 1) / st;
      if (I <= 0 || J <= 0) continue;
      IgemmLaunch L;
      memset(&L, 0, sizeof(L));
      int dh[kMaxTaps], dwv[kMaxTaps], rr[kMaxTaps], ss[kMaxTaps];
      int nr = 0, ns = 0;
      for (int r = 0; r < d->R; ++r) {
        const int v = ph + d->pad_h - r;
        if (((v % st) + st) % st == 0) { dh[nr] = (v - (((v % st) + st) % st)) / st; rr[nr] = r; ++nr; }
      }
      for (int s = 0; s < d->S; ++s) {
        const int v = pw + d->pad_w - s;
        if (((v % st) + st) % st == 0) { dwv[ns] = (v - (((v % st) + st) % st)) / st; ss[ns] = s; ++ns; }
      }
      if (nr * ns == 0) continue;
      int lo_h = dh[0], lo_w = dwv[0];
      for (int i = 1; i < nr; ++i) lo_h = dh[i] < lo_h ? dh[i] : lo_h;
      for (int i = 1; i < ns; ++i) lo_w = dwv[i] < lo_w ? dwv[i] : lo_w;
      L.ntaps = nr * ns;
      for (int a = 0; a < nr; ++a)
        for (int b = 0; b < ns; ++b) {
          TapEntry& t = L.taps[a * ns + b];
          t.off_h = (uint16_t)(dh[a] - lo_h);
          t.off_w = (uint16_t)(dwv[b] - lo_w);
          t.b_tap = (uint16_t)(rr[a] * d->S + ss[b]);
          t.pad_ = 0;
        }
      L.src = dy; L.Nimg = d->N; L.SH = d->P; L.SW = d->Q; L.SC = d->K;
      L.wmat = wt; L.Nout = d->C; L.wtaps = d->R * d->S;
      L.I = I; L.J = J; L.trav = 1; L.lower_w = lo_w; L.lower_h = lo_h;
      L.out = dx; L.OH = d->H; L.OW = d->W; L.os = st; L.oh0 = ph; L.ow0 = pw; L.ldo = d->C;
      L.res = residual; L.bias = nullptr; L.act = 0; L.out_fp32 = 0;
      L.window = d->window;
      rc = launch_igemm(L, stream);
      if (rc) return rc;
    }
  return B200_OK;
}

extern "C" size_t b200_conv_wgrad_workspace_bytes(void) {
  // splits * tiles <= SM count, each partial tile is 128 x 512 fp32
  return static_cast<size_t>(sm_count() + 8) * kTileM * 512 * sizeof(float);
}

extern "C" int b200_conv_wgrad(const b200_conv_desc* d, const void* x, const void* dy, float* dw, void* workspace,
                               size_t workspace_bytes, b200_stream_t stream_) {
  int rc = check_desc(d);
  if (rc) return rc;
  cudaStream_t stream = (cudaStream_t)stream_;
  B200_REQUIRE(x && dy && dw, B200_ERR_INVALID, "conv_wgrad: null pointer");
  B200_REQUIRE(d->C % 8 == 0 && d->K % 8 == 0, B200_ERR_UNSUPPORTED,
               "conv_wgrad: C=%d and K=%d must be multiples of 8", d->C, d->K);
  if (d->stride == 1 && d->pad_h == d->pad_w && d->P == d->H + 2 * d->pad_h - d->R + 1 &&
      d->Q == d->W + 2 * d->pad_w - d->S + 1 && d->x_pixel_stride == 0 &&
      (d->window == 0 || d->window == 128) &&
      halo_wgrad_eligible(d->P, d->Q, d->C, d->K, d->R, d->S, d->pad_h, d->window))
    return launch_halo_wgrad(x, dy, dw, workspace, workspace_bytes, d->N, d->P, d->Q, d->C, d->K, d->R, d->S, d->pad_h,
                             stream, d->window);
  B200_REQUIRE(d->window == 0 || d->window == 128, B200_ERR_UNSUPPORTED, "conv_wgrad: window must be 0 or 128");
  // window mode (block-diagonal): k-tile t pairs with input channels [128t, 128t+128) only; dw is [K][taps][128]
  const int Cw = d->window ? d->window : d->C;
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.M_total = d->N * d->P * d->Q;
  p.P = d->P; p.Q = d->Q; p.trav = d->stride; p.lower_w = -d->pad_w; p.lower_h = -d->pad_h;
  p.K_out = d->K; p.C = Cw; p.taps_total = d->R * d->S;
  p.window = d->window;
  p.ckA = pick_ck(d->K);
  p.ckB = pick_ck(Cw);
  p.bk = kBk;  // pixels per TMA box: fewer, larger TMA requests per byte (32-pixel boxes were request-rate bound)
  p.c_chunks = (Cw + p.ckB - 1) / p.ckB;
  p.total_boxes = p.taps_total * p.c_chunks;
  p.k_tiles = (d->K + kTileM - 1) / kTileM;
  p.boxA_bytes = p.bk * p.ckA * 2;
  p.boxB_bytes = p.bk * p.ckB * 2;
  // Tile shape: one k-tile (128 output channels, the two consumer warpgroups) x bpc channel boxes of x per CTA, with
  // bpc * ckB <= 256 accumulator columns (128 fp32 registers per consumer thread).  The x tile is fetched once for
  // all 128 output channels.
  p.boxes_per_cta = 256 / p.ckB;
  if (p.boxes_per_cta > 8) p.boxes_per_cta = 8;
  if (p.boxes_per_cta > p.total_boxes) p.boxes_per_cta = p.total_boxes;
  p.col_groups = (p.total_boxes + p.boxes_per_cta - 1) / p.boxes_per_cta;
  p.total_blocks = (p.M_total + p.bk - 1) / p.bk;
  const int tiles = p.k_tiles * p.col_groups;
  int splits = sm_count() / tiles;  // one wave: a CTA takes most of an SM's shared memory, two cannot share one
  if (splits > p.total_blocks) splits = p.total_blocks;
  if (splits < 1) splits = 1;
  p.blocks_per_split = (p.total_blocks + splits - 1) / splits;
  p.splits = (p.total_blocks + p.blocks_per_split - 1) / p.blocks_per_split;
  p.stage_bytes = (kTileM / p.ckA) * p.boxA_bytes + p.boxes_per_cta * p.boxB_bytes;
  p.stage_bytes = (p.stage_bytes + 1023u) & ~1023u;
  // 200 KB, not the full 224: the weight gradients run on the side stream BESIDE the main stream's BatchNorm kernels,
  // whose reduce blocks need ~10 KB of shared memory on the same SM
  p.num_stages = kSmemBudget / (int)p.stage_bytes;
  if (p.num_stages > kMaxStages) p.num_stages = kMaxStages;
  if (p.num_stages < 2) p.num_stages = 2;
  p.dw = dw;
  p.pitch = p.boxes_per_cta * p.ckB;
  p.partial = nullptr;
  if (p.splits > 1) {
    const size_t need = static_cast<size_t>(tiles) * p.splits * kTileM * p.pitch * sizeof(float);
    B200_REQUIRE(workspace != nullptr && workspace_bytes >= need, B200_ERR_INVALID,
                 "conv_wgrad: workspace too small (%zu < %zu); see b200_conv_wgrad_workspace_bytes()", workspace_bytes,
                 need);
    B200_REQUIRE((Cw & 3) == 0, B200_ERR_UNSUPPORTED, "conv_wgrad: C must be a multiple of 4");
    p.partial = static_cast<float*>(workspace);
  }
  p.S_filter = d->S;
  CUtensorMap tmDy, tmX;
  rc = encode_tiled(&tmDy, dy, 2, {d->K, p.M_total}, {p.ckA, p.bk}, "wgrad dy");
  if (rc) return rc;
  const int upper_w = p.lower_w + (d->Q - 1) * d->stride + 1 - d->W;
  const int upper_h = p.lower_h + (d->P - 1) * d->stride + 1 - d->H;
  p.plain_x = (d->R == 1 && d->S == 1 && d->stride == 1 && d->pad_h == 0 && d->pad_w == 0 && d->P == d->H &&
               d->Q == d->W && d->x_pixel_stride == 0) ? 1 : 0;
  if (getenv("B200_WGRAD_DEBUG"))   // keys kt (always 1) and k_groups (== k_tiles) stay for the parsers of this line
    fprintf(stderr, "[wgrad] K=%d C=%d taps=%d stride=%d ckA=%d ckB=%d kt=%d bpc=%d k_groups=%d col_groups=%d splits=%d "
            "bps=%d stages=%d stage=%u nc=%d nboxes_last=%d plain_x=%d partial=%d window=%d xs=%d\n", d->K, d->C,
            p.taps_total, d->stride, p.ckA, p.ckB, 1, p.boxes_per_cta, p.k_tiles, p.col_groups, p.splits,
            p.blocks_per_split, p.num_stages, p.stage_bytes, p.pitch, p.total_boxes - (p.col_groups - 1) * p.boxes_per_cta,
            p.plain_x, p.partial != nullptr, d->window, d->x_pixel_stride);
  if (p.plain_x)
    rc = encode_tiled(&tmX, x, 2, {d->C, p.M_total}, {p.ckB, p.bk}, "wgrad x");
  else
    rc = encode_im2col(&tmX, x, d->N, d->H, d->W, d->C, p.ckB, p.bk, p.lower_w, p.lower_h, upper_w, upper_h,
                       d->stride, d->x_pixel_stride, d->x_row_stride, d->x_image_stride);
  if (rc) return rc;
  const int smem_bytes = p.num_stages * (int)p.stage_bytes + 1024;
  const auto kfn = wgrad_kernel_for(p.pitch);
  rc = set_smem_attr((const void*)kfn, smem_bytes);
  if (rc) return rc;
  const int grid = tiles * p.splits;
  b200::launch(kfn, grid, kThreads, smem_bytes, stream, tmDy, tmX, p);
  B200_CHECK_LAUNCH("conv_wgrad_kernel");
  if (p.partial == nullptr) return B200_OK;
  // channel boxes are numbered tap-major, as in the kernel: id = tap * c_chunks + (c / ckB)
  return launch_wgrad_reduce(p.partial, dw, d->K, p.taps_total, Cw, p.ckB, p.c_chunks, 1, p.boxes_per_cta, p.k_tiles,
                             p.splits, p.pitch, stream);
}
