// Stride-1 RxS convolutions (3x3 pad 1 fprop/dgrad; the 4x4 pad 0 space-to-depth stem) as a "shift GEMM" on Hopper
// tensor cores (wgmma).
//
// The im2col kernel (conv.cu) re-fetches the activation tile once per filter tap: 9 TMA loads of the same
// pixels, shifted.  Here a tile is RT full image rows; its zero-padded halo box [(RT+2) x (W+2) pixels x 64 ch]
// is loaded ONCE per 64-channel block (tiled 4D TMA, out-of-bounds = padding), and the nine taps are nine views of
// that one shared-memory buffer: the wgmma descriptor start address is simply advanced by (r*(W+2)+s) pixel rows
// (row-shifted swizzled descriptors are valid because the swizzle is a function of the absolute smem address).
// The 128 accumulator rows are "virtual pixels" of the padded row pitch W+2; the two halo columns per row are
// computed and discarded (2/(W+2) of the MMA work).
// Activation traffic from L2 drops ~9x -> ~1.3x; weights stream through a separate ring.
//
// Pixel rows are 128 B (64-channel chunks, 128B swizzle) or, for the 16-channel stem, 32 B (32B swizzle, one K=16
// MMA per tap).  When all weight slices of a CTA fit in shared memory (64x64 3x3, the stem) they are loaded once
// ("stationary") instead of streaming through the ring with every tile.
#include "common.cuh"
#include "host.h"
#include <stdlib.h>

namespace b200 {

constexpr int kHMaxA = 6, kHMaxB = 8;
constexpr int kHMaxTaps = 16;

struct HaloParams {
  int N, H, W, C, Kout;    // H x W: OUTPUT map (the source is (H+R-1-2*pad) x (W+S-1-2*pad))
  int RT, Wp;              // output rows per tile, halo row pitch W+S-1
  int tiles_per_img, m_tiles, n_tiles, block_n, c_chunks;
  int sa, sb;              // ring depths (sb unused when the weights are stationary)
  uint32_t a_bytes, a_box_bytes, b_bytes;
  int act;
  int has_res;
  double* stats;
  const float* bias;       // [Kout] fp32 added before the residual / activation (BN folded for inference), or nullptr
  int ntaps, pad;
  int row_bytes;           // bytes of one source pixel chunk: 128 (64 channels) or 32 (16 channels)
  int b_stationary;        // 1: all c_chunks*ntaps weight slices of the n-tile stay in shared memory
  int diag;                // 1: block-diagonal ("window") convolution: n-tile b (64 outputs) reads input channels
                           //    [64b, 64b+64) only; a CTA keeps ONE n-tile (its 9 weight slices stay resident) and walks
                           //    the pixel tiles -- how grouped convolutions run (include/b200conv.h, desc.window)
  uint16_t a_off[kHMaxTaps];  // pixel-row offset of each tap's view inside the halo buffer
  uint16_t b_tap[kHMaxTaps];  // weight tap slice used with it
};

// Descriptors are built once per operand buffer and advanced by adding (byte offset >> 4) to the address field, with
// the tap / k-step loops fully unrolled.  BN = block_n (64, 128 or 256) sizes the accumulators exactly.
template <int NTAPS, int KSTEPS, int BN>
__global__ void __launch_bounds__(kThreads, 1)
conv_halo_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                 const __grid_constant__ HaloParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t a_full[kHMaxA], a_empty[kHMaxA], b_full[kHMaxB], b_empty[kHMaxB];
  __shared__ __align__(8) uint64_t res_bar, bstat_bar;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sA = smem;
  uint8_t* sB = sA + p.sa * p.a_bytes;
  const int b_slots = p.b_stationary ? p.c_chunks * p.ntaps : p.sb;
  uint8_t* epi = sB + b_slots * p.b_bytes;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.sa; ++i) { mbar_init(&a_full[i], 1); mbar_init(&a_empty[i], 8); }
    for (int i = 0; i < kHMaxB; ++i) { mbar_init(&b_full[i], 1); mbar_init(&b_empty[i], 8); }
    mbar_init(&bstat_bar, 1);
    mbar_init(&res_bar, 1);
    fence_mbar_init();
    prefetch_tmap(&tmX); prefetch_tmap(&tmB); prefetch_tmap(&tmC);
    if (p.has_res) prefetch_tmap(&tmR);
  }
  __syncthreads();
  // tile walk: dense -- tiles (m, n) round-robin over the CTAs; diagonal -- the CTA owns n-tile blockIdx.x % n_tiles and
  // walks the m-tiles with stride gridDim.x / n_tiles (the grid is a multiple of n_tiles)
  const int t_start = p.diag ? static_cast<int>(blockIdx.x) / p.n_tiles : static_cast<int>(blockIdx.x);
  const int t_step = p.diag ? static_cast<int>(gridDim.x) / p.n_tiles : static_cast<int>(gridDim.x);
  const int total_tiles = p.diag ? p.m_tiles : p.m_tiles * p.n_tiles;
  const int own_n = static_cast<int>(blockIdx.x) % p.n_tiles;

  if (warp >= 8) {
    producer_setmaxnreg();
    if (warp == 8 && lane == 0) {
      int ia = 0, ib = 0; uint32_t pa = 0, pb = 0;
      const int cw = p.row_bytes >> 1;   // channels per chunk
      if (p.b_stationary && t_start < total_tiles) {
        // stationary weights: every tile of this CTA uses the same slices (n_tiles == 1, or the CTA's own n-tile)
        mbar_arrive_expect_tx(&bstat_bar, static_cast<uint32_t>(p.c_chunks * NTAPS) * p.b_bytes);
        for (int cc = 0; cc < p.c_chunks; ++cc)
          for (int t = 0; t < NTAPS; ++t)
            tma_load_3d(&tmB, &bstat_bar, sB + (cc * NTAPS + t) * p.b_bytes, cc * cw, p.b_tap[t],
                        p.diag ? own_n * p.block_n : 0);
      }
      for (int tile = t_start; tile < total_tiles; tile += t_step) {
        const int m_tile = p.diag ? tile : tile / p.n_tiles, n_tile = p.diag ? own_n : tile - m_tile * p.n_tiles;
        const int img = m_tile / p.tiles_per_img;
        const int h0 = (m_tile - img * p.tiles_per_img) * p.RT;
        for (int cc = 0; cc < p.c_chunks; ++cc) {
          mbar_wait(&a_empty[ia], pa ^ 1u);
          mbar_arrive_expect_tx(&a_full[ia], p.a_box_bytes);
          tma_load_4d(&tmX, &a_full[ia], sA + ia * p.a_bytes, (p.diag ? n_tile : cc) * cw, -p.pad, h0 - p.pad, img);
          if (++ia == p.sa) { ia = 0; pa ^= 1u; }
          if (p.b_stationary) continue;
          for (int t = 0; t < NTAPS; ++t) {
            mbar_wait(&b_empty[ib], pb ^ 1u);
            mbar_arrive_expect_tx(&b_full[ib], p.b_bytes);
            tma_load_3d(&tmB, &b_full[ib], sB + ib * p.b_bytes, cc * cw, p.b_tap[t], n_tile * p.block_n);
            if (++ib == p.sb) { ib = 0; pb ^= 1u; }
          }
        }
      }
    }
    return;
  }
  consumer_setmaxnreg();

  // ---- consumers: warpgroup wg computes accumulator rows (virtual pixels) [64 wg, 64 wg + 64) of every tile
  const int wg = warp >> 2;
  const int r_lo = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows r_lo, r_lo + 8
  const int c_lo = 2 * (lane & 3);
  const bool leader = threadIdx.x == 0;
  const uint64_t proto = make_smem_desc(0, 16, 8u * p.row_bytes, layout_type_for_row_bytes(p.row_bytes));
  const uint32_t a_wg = (64u * wg * p.row_bytes) >> 4;
  const int nbox = BN >> 6;
  const uint32_t box_bytes = static_cast<uint32_t>(p.RT * p.W) * 128u;
  const uint32_t box_pitch = (box_bytes + 1023u) & ~1023u;
  int srow[2];
  bool in_tile[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int v = r_lo + 8 * h;
    const int ry = v / p.Wp, cx = v - ry * p.Wp;
    srow[h] = ry * p.W + cx;            // row of the staged output tile [RT][W][64]
    in_tile[h] = (ry < p.RT) && (cx < p.W);
  }
  // fused BN statistics: this thread owns one output column and a row range of every tile
  const int st_col = threadIdx.x % BN;
  const int st_rows = kTileM / (256 / BN);
  const int st_row0 = (threadIdx.x / BN) * st_rows;
  int st_ntile = -1;
  float st_s1 = 0.f, st_s2 = 0.f;
  if (p.b_stationary && t_start < total_tiles) mbar_wait(&bstat_bar, 0);

  float acc[BN / 2];
  int ia = 0, ib = 0; uint32_t pa = 0, pb = 0;
  int local = 0;
  for (int tile = t_start; tile < total_tiles; tile += t_step, ++local) {
    const int m_tile = p.diag ? tile : tile / p.n_tiles, n_tile = p.diag ? own_n : tile - m_tile * p.n_tiles;
    const int img = m_tile / p.tiles_per_img;
    const int h0 = (m_tile - img * p.tiles_per_img) * p.RT;
    const int nbase = n_tile * BN;
    // the staging tile is reused: the previous TMA store must have read it, every thread must be done with its
    // statistics reads; then the residual tile is fetched into it while the MMAs run
    if (leader && local > 0) bulk_wait_group_read0();
    named_bar_sync(1, 256);
    if (leader && p.has_res) {
      fence_proxy_async();
      mbar_arrive_expect_tx(&res_bar, static_cast<uint32_t>(nbox) * box_bytes);
      for (int b = 0; b < nbox; ++b) tma_load_4d(&tmR, &res_bar, epi + b * box_pitch, nbase + b * 64, 0, h0, img);
    }

    // one commit group per tap (streamed weights: each tap frees a weight slot) or per channel block (resident weights);
    // after wgmma_wait<1> all groups but the newest are complete, so the buffers whose last reader was the previous
    // group are released then
    wgmma_fence_acc(acc);
    int rel_a = -1, rel_b = -1;
    for (int cc = 0; cc < p.c_chunks; ++cc) {
      mbar_wait(&a_full[ia], pa);
      const uint64_t da0 = proto + (smem_u32(sA + ia * p.a_bytes) >> 4) + a_wg;
#pragma unroll
      for (int t = 0; t < NTAPS; ++t) {
        uint64_t db0;
        if (p.b_stationary) {
          db0 = proto + (smem_u32(sB + (cc * NTAPS + t) * p.b_bytes) >> 4);
        } else {
          mbar_wait(&b_full[ib], pb);
          db0 = proto + (smem_u32(sB + ib * p.b_bytes) >> 4);
        }
        const uint32_t tap_inc = (static_cast<uint32_t>(p.a_off[t]) * p.row_bytes) >> 4;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k)
          wgmma_bf16<0, 0>(acc, da0 + tap_inc + 2 * k, db0 + 2 * k, (cc | t | k) != 0 ? 1u : 0u);
        if (!p.b_stationary || t == NTAPS - 1) {
          wgmma_commit();
          wgmma_wait<1>();
          if (rel_b >= 0) release_stage(&b_empty[rel_b], lane);
          if (rel_a >= 0) release_stage(&a_empty[rel_a], lane);
          rel_a = (t == NTAPS - 1) ? ia : -1;
          rel_b = p.b_stationary ? -1 : ib;
        }
        if (!p.b_stationary && ++ib == p.sb) { ib = 0; pb ^= 1u; }
      }
      if (++ia == p.sa) { ia = 0; pa ^= 1u; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (rel_b >= 0) release_stage(&b_empty[rel_b], lane);
    if (rel_a >= 0) release_stage(&a_empty[rel_a], lane);

    if (p.has_res) mbar_wait(&res_bar, static_cast<uint32_t>(local & 1));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!in_tile[h] || h0 + (r_lo + 8 * h) / p.Wp >= p.H) continue;
      const int row = srow[h];
#pragma unroll
      for (int j = 0; j < BN / 2; j += 4) {
        const int c = 2 * j + c_lo;
        uint32_t* dst = reinterpret_cast<uint32_t*>(epi + staged_offset(row, c, box_pitch));
        float v0 = acc[j + 2 * h], v1 = acc[j + 2 * h + 1];
        if (p.bias != nullptr) { v0 += __ldg(p.bias + nbase + c); v1 += __ldg(p.bias + nbase + c + 1); }
        if (p.has_res) {
          const float2 t2 = unpack_bf16x2(*dst);
          v0 += t2.x;
          v1 += t2.y;
        }
        *dst = pack_bf16x2(apply_act(v0, p.act), apply_act(v1, p.act));
      }
    }
    fence_proxy_async();
    named_bar_sync(1, 256);
    if (leader) {
      for (int b = 0; b < nbox; ++b) tma_store_4d(&tmC, epi + b * box_pitch, nbase + b * 64, 0, h0, img);
      bulk_commit_group();
    }
    if (p.stats != nullptr) {
      if (st_ntile != n_tile) {
        if (st_ntile >= 0) flush_bn_stats(p.stats, p.Kout, st_ntile * BN, st_col, st_s1, st_s2);
        st_ntile = n_tile; st_s1 = 0.f; st_s2 = 0.f;
      }
      const int vrows = min(p.RT, p.H - h0) * p.W;   // staged rows that belong to the image
      const int r_end = min(st_row0 + st_rows, vrows);
      for (int r = st_row0; r < r_end; ++r) {
        const float x = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(epi + staged_offset(r, st_col, box_pitch)));
        st_s1 += x;
        st_s2 = fmaf(x, x, st_s2);
      }
    }
  }
  if (p.stats != nullptr && st_ntile >= 0) flush_bn_stats(p.stats, p.Kout, st_ntile * BN, st_col, st_s1, st_s2);
  if (leader) bulk_wait_group0();
}

typedef void (*HaloKernelFn)(const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap,
                             const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap,
                             const __grid_constant__ HaloParams);
// 3x3 (9 taps, four 16-deep k-steps per 64-channel chunk) or the 4x4 stem (16 taps, one k-step per 16-channel pixel)
static HaloKernelFn halo_kernel_for(int ntaps, int block_n) {
  if (ntaps == 9)
    return block_n == 64 ? conv_halo_kernel<9, 4, 64> : block_n == 128 ? conv_halo_kernel<9, 4, 128>
         : block_n == 256 ? conv_halo_kernel<9, 4, 256> : nullptr;
  if (ntaps == 16)
    return block_n == 64 ? conv_halo_kernel<16, 1, 64> : block_n == 128 ? conv_halo_kernel<16, 1, 128>
         : block_n == 256 ? conv_halo_kernel<16, 1, 256> : nullptr;
  return nullptr;
}

// Geometry shared by the fprop/dgrad and wgrad halo kernels: stride-1 RxS taps over an H x W OUTPUT map.
// Supported: 3x3 pad 1 with 64-channel source chunks, and the 4x4 pad 0 stem with a 16-channel source.
bool halo_geometry_ok(int H, int W, int Cs, int R, int S, int pad) {
  const bool k3 = (R == 3 && S == 3 && pad == 1 && Cs % 64 == 0);
  const bool k4 = (R == 4 && S == 4 && pad == 0 && Cs == 16);
  if (!k3 && !k4) return false;
  const int Wp = W + S - 1;
  if (Wp > 128 || W < 8) return false;
  int RT = 128 / Wp;
  if (RT > H) RT = H;
  const int tiles = (H + RT - 1) / RT;
  return (double)H * W / (128.0 * tiles) >= 0.6;   // fill of the 128 accumulator rows
}

bool halo_eligible(int H, int W, int Cs, int Nout, int R, int S, int pad) {
  if (!halo_geometry_ok(H, W, Cs, R, S, pad) || Nout % 64 != 0) return false;
  const int n_tiles = (Nout + 255) / 256;
  const int block_n = Nout / n_tiles;
  return Nout % n_tiles == 0 && block_n % 64 == 0 && 256 % block_n == 0;
}

// dir 0: fprop (tap (r,s) reads halo offset (r,s), weight slice r*S+s); dir 1: dgrad (offset (R-1-r, S-1-s))
int launch_halo(const void* src, const void* wmat, void* out, const void* res, const float* bias, int N, int H, int W,
                int Cs, int Nout, int R, int S, int pad, int dir, int act, double* stats, cudaStream_t stream, int window) {
  HaloParams p;
  memset(&p, 0, sizeof(p));
  p.diag = window > 0 ? 1 : 0;
  if (p.diag)
    B200_REQUIRE(window == 64 && Cs == Nout && Cs % 64 == 0 && R == 3 && S == 3, B200_ERR_UNSUPPORTED,
                 "conv halo: window mode needs window == 64, C == K, C %% 64 == 0 and a 3x3 filter (C=%d K=%d)", Cs, Nout);
  p.N = N; p.H = H; p.W = W; p.C = Cs; p.Kout = Nout;
  p.ntaps = R * S; p.pad = pad;
  p.row_bytes = (Cs == 16) ? 32 : 128;
  const int cw = p.row_bytes / 2;
  p.Wp = W + S - 1;
  p.RT = 128 / p.Wp;
  if (p.RT > H) p.RT = H;
  p.tiles_per_img = (H + p.RT - 1) / p.RT;
  p.m_tiles = N * p.tiles_per_img;
  p.n_tiles = p.diag ? Nout / 64 : (Nout + 255) / 256;
  p.block_n = Nout / p.n_tiles;
  p.c_chunks = p.diag ? 1 : Cs / cw;
  p.a_box_bytes = (uint32_t)(p.RT + R - 1) * p.Wp * p.row_bytes;
  uint32_t a_need = (uint32_t)(kTileM + (R - 1) * p.Wp + (S - 1)) * p.row_bytes;
  if (a_need < p.a_box_bytes) a_need = p.a_box_bytes;
  p.a_bytes = (a_need + 1023u) & ~1023u;
  p.b_bytes = (uint32_t)p.block_n * p.row_bytes;
  p.act = act;
  p.has_res = res != nullptr;
  p.stats = stats;
  p.bias = bias;
  for (int r = 0; r < R; ++r)
    for (int s = 0; s < S; ++s) {
      const int t = r * S + s;
      p.b_tap[t] = (uint16_t)t;
      p.a_off[t] = (uint16_t)(dir == 0 ? r * p.Wp + s : (R - 1 - r) * p.Wp + (S - 1 - s));
    }
  const uint32_t box_pitch = (((uint32_t)(p.RT * W) * 128u) + 1023u) & ~1023u;
  const uint32_t epi_bytes = (uint32_t)(p.block_n / 64) * box_pitch;
  int budget = 212 * 1024 - (int)epi_bytes;
  const int b_all = p.c_chunks * p.ntaps * (int)p.b_bytes;
  p.b_stationary = ((p.n_tiles == 1 || p.diag) && b_all <= 80 * 1024) ? 1 : 0;
  B200_REQUIRE(!p.diag || p.b_stationary, B200_ERR_UNSUPPORTED, "conv halo: window mode expects resident weights");
  int b_region;
  if (p.b_stationary) {
    b_region = b_all;
    p.sb = 0;
    p.sa = (budget - b_region) / (int)p.a_bytes;
    if (p.sa > kHMaxA) p.sa = kHMaxA;
  } else {
    p.sa = 2;
    p.sb = (budget - p.sa * (int)p.a_bytes) / (int)p.b_bytes;
    if (p.sb > kHMaxB) p.sb = kHMaxB;
    if (p.sb >= 6 && (int)(3 * p.a_bytes + 4 * p.b_bytes) <= budget) {
      p.sa = 3;
      p.sb = (budget - 3 * (int)p.a_bytes) / (int)p.b_bytes;
      if (p.sb > kHMaxB) p.sb = kHMaxB;
    }
    b_region = p.sb * (int)p.b_bytes;
  }
  B200_REQUIRE(p.sa >= 2 && (p.b_stationary || p.sb >= 2), B200_ERR_UNSUPPORTED,
               "conv halo: shared memory budget exceeded (W=%d, block_n=%d)", W, p.block_n);
  CUtensorMap tmX, tmB, tmC, tmR;
  memset(&tmR, 0, sizeof(tmR));
  int rc = encode_tiled(&tmX, src, 4, {Cs, W + S - 1 - 2 * pad, H + R - 1 - 2 * pad, N}, {cw, p.Wp, p.RT + R - 1, 1},
                        "conv halo source");
  if (rc) return rc;
  // the weight operand is [Nout][taps][window or Cs]
  rc = encode_tiled(&tmB, wmat, 3, {p.diag ? window : Cs, p.ntaps, Nout}, {cw, 1, p.block_n}, "conv halo weights");
  if (rc) return rc;
  rc = encode_tiled(&tmC, out, 4, {Nout, W, H, N}, {64, W, p.RT, 1}, "conv halo output");
  if (rc) return rc;
  if (res) {
    rc = encode_tiled(&tmR, res, 4, {Nout, W, H, N}, {64, W, p.RT, 1}, "conv halo residual");
    if (rc) return rc;
  }
  const int smem_bytes = p.sa * (int)p.a_bytes + b_region + (int)epi_bytes + 1024;
  HaloKernelFn kfn = halo_kernel_for(p.ntaps, p.block_n);
  B200_REQUIRE(kfn != nullptr, B200_ERR_UNSUPPORTED, "conv halo: %d taps with block_n %d unsupported", p.ntaps, p.block_n);
  rc = set_smem_attr((const void*)kfn, smem_bytes);
  if (rc) return rc;
  const int total = p.m_tiles * p.n_tiles;
  int grid = total < sm_count() ? total : sm_count();
  if (p.diag) {                       // a multiple of n_tiles: every CTA owns one n-tile
    int per_n = sm_count() / p.n_tiles;
    if (per_n > p.m_tiles) per_n = p.m_tiles;
    if (per_n < 1) per_n = 1;
    grid = per_n * p.n_tiles;
  }
  if (getenv("B200_HALO_DEBUG"))
    fprintf(stderr, "[halo] dir=%d N=%d H=%d W=%d C=%d K=%d taps=%d block_n=%d n_tiles=%d m_tiles=%d bstat=%d diag=%d "
            "sa=%d sb=%d bias=%d res=%d act=%d stats=%d grid=%d\n", dir, N, H, W, Cs, Nout, p.ntaps, p.block_n,
            p.n_tiles, p.m_tiles, p.b_stationary, p.diag, p.sa, p.sb, bias != nullptr, res != nullptr, act,
            stats != nullptr, grid);
  b200::launch(kfn, grid, kThreads, smem_bytes, stream, tmX, tmB, tmC, tmR, p);
  B200_CHECK_LAUNCH("conv_halo_kernel");
  return B200_OK;
}


// =================================================================================================
// Halo wgrad: dw[k, (r,s), c] += sum_pixels dy[pixel, k] * x[pixel + (r,s), c]   (stride 1)
//
// Both operands are MN-major (rows of shared memory = pixels = the GEMM K dimension).  A tile is RT output rows
// in the padded pitch Wp: dy is loaded as [RT x Wp] pixels (the S-1 extra columns are out of bounds -> TMA writes
// zeros), x as the [(RT+R-1) x Wp] halo, ONCE; the R*S taps are row-shifted views of that one x buffer, each
// accumulating into its own register block [128 k x cw c].  With cw = 16 the 9 taps of a 3x3 filter take 144
// accumulator columns (72 registers per consumer thread), the stem's 16 taps 256.  The im2col kernel re-fetched x
// once per tap.
// One CTA owns a (k-tile, channel-chunk) unit and a contiguous range of pixel tiles (split-K over pixels); partial
// fp32 tiles go to the workspace and launch_wgrad_reduce adds them into dw in a fixed order.
constexpr int kWMaxStages = 4;

struct HaloWgradParams {
  int N, H, W, K_out, C;
  int RT, Wp, tiles_per_img, m_tiles;
  int ntaps, pad, halo_rows;
  int x_row_bytes, cw, ncols;
  int c_chunks, k_tiles, units, splits, tiles_per_split;
  int stages;
  int window;              // 0 dense; 128: block-diagonal -- k-tile t only pairs with input channels [128t, 128t+128):
                           // units = 4 x k_tiles, dw is [K][taps][128]
  uint32_t a_box_bytes, a_bytes, x_box_bytes, x_bytes;
  float* partial;          // [unit][split][128][ncols]
  uint16_t x_off[kHMaxTaps];
};

// The S taps of one filter row are ONE MMA: their x views start one pixel row apart, so the descriptor's
// leading-dimension stride (distance between swizzle atoms along N) is set to one pixel row and N = S * cw.  The
// dy operand is then read from shared memory once per filter row instead of once per tap.
// Consumer warpgroup wg owns output channels [k0 + 64 wg, k0 + 64 wg + 64): R accumulator blocks of S * cw columns.
template <int R, int S>
__global__ void __launch_bounds__(kThreads, 1)
conv_halo_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX,
                       const __grid_constant__ HaloWgradParams p) {
  constexpr int kCols = S * 16;   // accumulator columns of one filter row (cw = 16 channels per x chunk)
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kWMaxStages], empty_bar[kWMaxStages];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  const uint32_t stage_bytes = p.a_bytes + p.x_bytes;

  // Rows that TMA never writes (dy rows >= RT*Wp, the second dy box when K_out = 64, x rows past the halo box) are
  // multiplied into the accumulators: they must be zero / finite, so the whole ring is cleared once.
  {
    uint4* z = reinterpret_cast<uint4*>(smem);
    const int n16 = static_cast<int>(p.stages * stage_bytes) >> 4;
    for (int i = threadIdx.x; i < n16; i += kThreads) z[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_mbar_init();
    prefetch_tmap(&tmDy);
    prefetch_tmap(&tmX);
  }
  fence_proxy_async();
  __syncthreads();

  const int split = blockIdx.x / p.units;
  const int unit = blockIdx.x - split * p.units;
  const int k_tile = unit % p.k_tiles;
  const int cc = unit / p.k_tiles;
  const int k0 = k_tile * kTileM;
  const int t_begin = split * p.tiles_per_split;
  const int t_end = min(p.m_tiles, t_begin + p.tiles_per_split);
  const int ntiles = t_end - t_begin;
  const int nA = min(2, (p.K_out - k0 + 63) / 64);
  if (ntiles <= 0) return;

  if (warp >= 8) {
    producer_setmaxnreg();
    if (warp == 8 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx = nA * p.a_box_bytes + p.x_box_bytes;
      for (int tile = t_begin; tile < t_end; ++tile) {
        const int img = tile / p.tiles_per_img;
        const int h0 = (tile - img * p.tiles_per_img) * p.RT;
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        uint8_t* sa = smem + stage * stage_bytes;
        mbar_arrive_expect_tx(&full_bar[stage], tx);
        for (int j = 0; j < nA; ++j) tma_load_4d(&tmDy, &full_bar[stage], sa + j * 16384, k0 + j * 64, 0, h0, img);
        tma_load_4d(&tmX, &full_bar[stage], sa + p.a_bytes, cc * p.cw + (p.window ? k0 : 0), -p.pad, h0 - p.pad, img);
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }
  consumer_setmaxnreg();

  const int wg = warp >> 2;
  const bool wg_on = wg < nA;
  // dy: one 64-channel box per warpgroup, MN-major, 128 B pixel rows; x: MN-major, LBO = one pixel row (the S taps)
  const uint64_t protoA = make_smem_desc(0, 16384, 1024, 1);
  const uint64_t protoX = make_smem_desc(0, p.x_row_bytes, 8u * p.x_row_bytes, layout_type_for_row_bytes(p.x_row_bytes));
  uint32_t row_inc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) row_inc[r] = (static_cast<uint32_t>(p.x_off[r * S]) * p.x_row_bytes) >> 4;
  const uint32_t kx_inc = (16u * p.x_row_bytes) >> 4;   // 16 pixel rows per K step
  float acc[R][kCols / 2];
#pragma unroll
  for (int r = 0; r < R; ++r) wgmma_fence_acc(acc[r]);
  int stage = 0, prev = 0; uint32_t phase = 0;
  for (int i = 0; i < ntiles; ++i) {
    mbar_wait(&full_bar[stage], phase);
    if (wg_on) {
      const uint32_t a_addr = smem_u32(smem + stage * stage_bytes);
      const uint64_t da0 = protoA + ((a_addr + wg * 16384) >> 4);
      const uint64_t dx0 = protoX + ((a_addr + p.a_bytes) >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const uint32_t scale = (k != 0 || i != 0) ? 1u : 0u;
#pragma unroll
        for (int r = 0; r < R; ++r)
          wgmma_bf16<1, 1>(acc[r], da0 + k * 128, dx0 + row_inc[r] + k * kx_inc, scale);
      }
      wgmma_commit();
      wgmma_wait<1>();
    }
    if (i > 0) release_stage(&empty_bar[prev], lane);
    prev = stage;
    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int r = 0; r < R; ++r) wgmma_fence_acc(acc[r]);
  release_stage(&empty_bar[prev], lane);
  if (!wg_on) return;

  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows row, row + 8 (output channels)
  const int c_lo = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* dst = p.partial + ((static_cast<long long>(unit) * p.splits + split) * kTileM + row + 8 * h) * p.ncols;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int j = 0; j < kCols / 2; j += 4)
        *reinterpret_cast<float2*>(dst + r * kCols + 2 * j + c_lo) = make_float2(acc[r][j + 2 * h], acc[r][j + 2 * h + 1]);
  }
}

// The partial tiles must also fit the split-K workspace (b200_conv_wgrad_workspace_bytes): units * splits <= SMs, or
// one split.
bool halo_wgrad_eligible(int H, int W, int C, int K_out, int R, int S, int pad, int window) {
  if (!halo_geometry_ok(H, W, C, R, S, pad) || K_out % 64 != 0) return false;
  const int units = ((window ? window : C) / 16) * ((K_out + kTileM - 1) / kTileM);   // as in launch_halo_wgrad
  return units <= sm_count() + 8;
}

int launch_halo_wgrad(const void* x, const void* dy, float* dw, void* workspace, size_t workspace_bytes, int N, int H,
                      int W, int C, int K_out, int R, int S, int pad, cudaStream_t stream, int window) {
  HaloWgradParams p;
  memset(&p, 0, sizeof(p));
  p.window = window;
  if (window)
    B200_REQUIRE(window == 128 && C == K_out && C % 128 == 0, B200_ERR_UNSUPPORTED,
                 "conv halo wgrad: window mode needs window == 128 and C == K, C %% 128 == 0 (C=%d K=%d)", C, K_out);
  p.N = N; p.H = H; p.W = W; p.K_out = K_out; p.C = C;
  p.ntaps = R * S; p.pad = pad;
  p.cw = 16;   // 16 channels per x chunk: R * S * 16 / 2 accumulator registers per consumer thread
  p.x_row_bytes = p.cw * 2;
  p.ncols = p.ntaps * p.cw;
  p.Wp = W + S - 1;
  p.RT = 128 / p.Wp;
  if (p.RT > H) p.RT = H;
  p.halo_rows = p.RT + R - 1;
  p.tiles_per_img = (H + p.RT - 1) / p.RT;
  p.m_tiles = N * p.tiles_per_img;
  p.c_chunks = (window ? window : C) / p.cw;       // channel chunks that pair with one k-tile
  p.k_tiles = (K_out + kTileM - 1) / kTileM;
  p.units = p.c_chunks * p.k_tiles;
  int splits = sm_count() / p.units;
  if (splits < 1) splits = 1;
  if (splits > p.m_tiles) splits = p.m_tiles;
  p.tiles_per_split = (p.m_tiles + splits - 1) / splits;
  p.splits = (p.m_tiles + p.tiles_per_split - 1) / p.tiles_per_split;   // every split owns at least one tile
  p.a_box_bytes = (uint32_t)(p.RT * p.Wp) * 128u;
  p.a_bytes = 2 * 16384;
  p.x_box_bytes = (uint32_t)(p.halo_rows * p.Wp) * p.x_row_bytes;
  int max_off = 0;
  for (int r = 0; r < R; ++r)
    for (int s = 0; s < S; ++s) {
      p.x_off[r * S + s] = (uint16_t)(r * p.Wp + s);
      if (r * p.Wp + s > max_off) max_off = r * p.Wp + s;
    }
  uint32_t x_need = (uint32_t)(kTileM + max_off) * p.x_row_bytes;
  if (x_need < p.x_box_bytes) x_need = p.x_box_bytes;
  p.x_bytes = (x_need + 1023u) & ~1023u;
  p.stages = (212 * 1024) / (int)(p.a_bytes + p.x_bytes);
  if (p.stages > kWMaxStages) p.stages = kWMaxStages;
  B200_REQUIRE(p.stages >= 2, B200_ERR_UNSUPPORTED, "conv halo wgrad: shared memory budget exceeded (W=%d)", W);
  const size_t need = (size_t)p.units * p.splits * kTileM * p.ncols * sizeof(float);
  B200_REQUIRE(workspace != nullptr && workspace_bytes >= need, B200_ERR_INVALID,
               "conv halo wgrad: workspace of %zu bytes needed (%zu given)", need, workspace_bytes);
  p.partial = reinterpret_cast<float*>(workspace);
  CUtensorMap tmDy, tmX;
  int rc = encode_tiled(&tmDy, dy, 4, {K_out, W, H, N}, {64, p.Wp, p.RT, 1}, "conv halo wgrad dy");
  if (rc) return rc;
  rc = encode_tiled(&tmX, x, 4, {C, W + S - 1 - 2 * pad, H + R - 1 - 2 * pad, N}, {p.cw, p.Wp, p.halo_rows, 1},
                    "conv halo wgrad x");
  if (rc) return rc;
  const int smem_bytes = p.stages * (int)(p.a_bytes + p.x_bytes) + 1024;
  const auto kfn = p.ntaps == 9 ? conv_halo_wgrad_kernel<3, 3> : conv_halo_wgrad_kernel<4, 4>;
  rc = set_smem_attr((const void*)kfn, smem_bytes);
  if (rc) return rc;
  if (getenv("B200_HALO_DEBUG"))
    fprintf(stderr, "[halo_wgrad] N=%d H=%d W=%d C=%d K=%d taps=%d k_tiles=%d c_chunks=%d m_tiles=%d units=%d "
            "splits=%d tiles_per_split=%d stages=%d grid=%d window=%d\n", N, H, W, C, K_out, p.ntaps, p.k_tiles,
            p.c_chunks, p.m_tiles, p.units, p.splits, p.tiles_per_split, p.stages, p.units * p.splits, window);
  b200::launch(kfn, p.units * p.splits, kThreads, smem_bytes, stream, tmDy, tmX, p);
  B200_CHECK_LAUNCH("conv_halo_wgrad_kernel");
  // dw is [K][taps][window or C]; channel boxes are numbered chunk-major, as the units: id = (c / cw) * taps + tap
  return launch_wgrad_reduce(p.partial, dw, K_out, p.ntaps, window ? window : C, p.cw, 1, p.ntaps, p.ntaps, p.k_tiles,
                             p.splits, p.ncols, stream);
}

}  // namespace b200
