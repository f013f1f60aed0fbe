// C-ABI plumbing: error text, launch counter, driver entry points.
#include "host.h"
#include <atomic>
#include <mutex>
#include <string.h>

namespace b200 {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (cached[dev] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cached[dev] = n > 0 ? n : 148;
  }
  return cached[dev];
}

static void* driver_entry(const char* name) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess) {
    return nullptr;
  }
  return fn;
}
EncodeIm2colFn encode_im2col_fn() {
  static EncodeIm2colFn fn = (EncodeIm2colFn)driver_entry("cuTensorMapEncodeIm2col");
  return fn;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tiled(CUtensorMap* tm, const void* base, int rank, const long long (&dims)[4], const int (&box)[4],
                 const char* what) {
  static EncodeTiledFn fn = (EncodeTiledFn)driver_entry("cuTensorMapEncodeTiled");
  B200_REQUIRE(fn != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t gdims[4], strides[3];
  cuuint32_t gbox[4], estr[4] = {1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) {
    gdims[i] = (cuuint64_t)dims[i];
    gbox[i] = (cuuint32_t)box[i];
    if (i + 1 < rank) strides[i] = (i == 0 ? 2 : strides[i - 1]) * gdims[i];
  }
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gdims, strides, gbox, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_for_row_bytes(box[0] * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char d[96] = "", b[64] = "";
    for (int i = 0, nd = 0, nb = 0; i < rank; ++i) {
      nd += snprintf(d + nd, sizeof(d) - nd, i ? ",%lld" : "%lld", dims[i]);
      nb += snprintf(b + nb, sizeof(b) - nb, i ? ",%d" : "%d", box[i]);
    }
    set_error("%s: cuTensorMapEncodeTiled(%dd) failed (%d) dims=(%s) box=(%s)", what, rank, (int)r, d, b);
    return B200_ERR_CUDA;
  }
  return B200_OK;
}

int set_smem_attr(const void* fn, int bytes) {
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  B200_REQUIRE(e == cudaSuccess, B200_ERR_CUDA, "cudaFuncSetAttribute(smem=%d): %s", bytes, cudaGetErrorString(e));
  return B200_OK;
}

}  // namespace b200

extern "C" {
const char* b200_last_error(void) { return b200::g_err; }
int b200_version(void) { return 100; }
long long b200_launch_count(void) { return b200::g_launches.load(); }
}
