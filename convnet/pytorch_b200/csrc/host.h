// Host-side plumbing shared by the C-ABI translation units: error text, launch counting,
// driver entry points for tensor-map encoding (resolved at run time: no libcuda link dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include "../../../include/b200conv.h"

namespace b200 {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);
int sm_count();

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeIm2colFn encode_im2col_fn();

// Tiled tensor map of a dense bf16 tensor of rank 2..4 (dims innermost first): box row bytes pick the swizzle, 128B L2
// promotion, out-of-bounds elements read as zero.  `what` names the map in the error text.
int encode_tiled(CUtensorMap* tm, const void* base, int rank, const long long (&dims)[4], const int (&box)[4],
                 const char* what);
// Raises a kernel's dynamic shared-memory limit to `bytes`.
int set_smem_attr(const void* fn, int bytes);

// conv.cu: dw[k][tap][c] += the sum over `splits` of the weight gradient's split-K partial tiles, in a fixed order.
// A partial element is partial[((unit * splits + s) * 128 + k % 128) * pitch + x * ck + c % ck], where channel box
// id = tap * tap_stride + (c / ck) * cc_stride gives unit = (id / bpc) * k_tiles + k / 128 and x = id % bpc.
int launch_wgrad_reduce(const float* partial, float* dw, int K_out, int taps, int C, int ck, int tap_stride,
                        int cc_stride, int bpc, int k_tiles, int splits, int pitch, cudaStream_t stream);

// conv3x3.cu: halo / shift-GEMM path for stride-1 convolutions (3x3 pad 1; the 4x4 pad 0 space-to-depth stem).
// H, W are the OUTPUT map dimensions.
bool halo_geometry_ok(int H, int W, int Cs, int R, int S, int pad);
bool halo_eligible(int H, int W, int Cs, int Nout, int R, int S, int pad);
int launch_halo(const void* src, const void* wmat, void* out, const void* res, const float* bias, int N, int H, int W,
                int Cs, int Nout, int R, int S, int pad, int dir, int act, double* stats, cudaStream_t stream,
                int window = 0);

bool halo_wgrad_eligible(int H, int W, int C, int K_out, int R, int S, int pad, int window);
int launch_halo_wgrad(const void* x, const void* dy, float* dw, void* workspace, size_t workspace_bytes, int N, int H,
                      int W, int C, int K_out, int R, int S, int pad, cudaStream_t stream, int window = 0);

// Kernel launch; each argument is converted to the kernel's parameter type.
template <typename... KArgs, typename... Args>
inline void launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  kernel<<<grid, block, smem, stream>>>(static_cast<KArgs>(args)...);   // errors surface in B200_CHECK_LAUNCH
}

inline CUtensorMapSwizzle swizzle_for_row_bytes(int row_bytes) {
  return row_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : (row_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

#define B200_CHECK_LAUNCH(name)                                                   \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      b200::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));    \
      return B200_ERR_CUDA;                                                       \
    }                                                                             \
    b200::count_launch();                                                         \
  } while (0)

#define B200_REQUIRE(cond, code, ...)   \
  do {                                  \
    if (!(cond)) {                      \
      b200::set_error(__VA_ARGS__);     \
      return code;                      \
    }                                   \
  } while (0)

}  // namespace b200
