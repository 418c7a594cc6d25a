// Host side of tma.cuh: the tensor-map encoder of the tf32 kernels and the watchdog flag of every mbarrier kernel.
#include "kernels.cuh"
#include "tma.cuh"

namespace srf {

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int encode_tensor_map_f32(CUtensorMap* tm, const float* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                          const cuuint32_t* box) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return -2;
  const cuuint32_t estr[3] = {1, 1, 1};
  return fn(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS ? 0 : -1;
}

// mapped pinned host memory: still readable after a device-side trap killed the context
static int* g_wd_host = nullptr;
static int* g_wd_dev = nullptr;

int* watchdog_device_flag() {
  if (!g_wd_host && cudaHostAlloc(reinterpret_cast<void**>(&g_wd_host), sizeof(int), cudaHostAllocMapped) == cudaSuccess) {
    *g_wd_host = 0;
    cudaHostGetDevicePointer(reinterpret_cast<void**>(&g_wd_dev), g_wd_host, 0);
  }
  return g_wd_dev;
}

int watchdog_flag() { return g_wd_host ? *reinterpret_cast<volatile int*>(g_wd_host) : 0; }

}  // namespace srf
