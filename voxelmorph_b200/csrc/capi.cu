// Error text, version string, launch counter and small device queries of the C ABI.
#include <stdarg.h>
#include <stdlib.h>

#include <atomic>

#include "tc_common.cuh"

namespace vxm {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(e));
    return VXM_ERR_CUDA;
  }
  count_launch(1);
  return VXM_OK;
}

int sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;   // H100 SXM
  if (dev != cached_dev) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached = n;
    cached_dev = dev;
  }
  return cached;
}

// Persistent CTAs of a tensor-core convolution launch: one per SM, or at most n with VXM_B200_CONV_CTAS=n (n >= 1; read
// at every launch).  The depth-chunk cost model and the grid both take this count, so a capped launch runs the
// decomposition of a GPU with n SMs.
int conv_ctas() {
  const int n = sm_count();
  const char* e = getenv("VXM_B200_CONV_CTAS");
  const int cap = e ? atoi(e) : 0;
  return cap >= 1 && cap < n ? cap : n;
}

namespace tc {

// cuTensorMapEncodeTiled through the runtime's driver entry-point query: no link-time dependency on libcuda, so the
// library still builds (and loads, for the symbol checks) in a container without a driver.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
  static std::atomic<void*> cached{nullptr};
  void* p = cached.load(std::memory_order_acquire);
  if (!p) {
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) p = nullptr;
    cached.store(p, std::memory_order_release);
  }
  return reinterpret_cast<EncodeTiledFn>(p);
}

int make_act_tmap(CUtensorMap* out, const void* base, int B, int D, int H, int W, int C, int boxC, int boxW, int boxH) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return -1; }
  const cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)D, (cuuint64_t)B};
  const cuuint64_t strides[4] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2, (cuuint64_t)D * H * W * C * 2};
  const cuuint32_t box[5] = {(cuuint32_t)boxC, (cuuint32_t)boxW, (cuuint32_t)boxH, 1u, 1u};
  const cuuint32_t estr[5] = {1u, 1u, 1u, 1u, 1u};
  const int rowb = boxC * 2;
  const CUtensorMapSwizzle sw = rowb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (rowb == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  if (rowb != 32 && rowb != 64 && rowb != 128) { set_error("make_act_tmap: row width %d bytes is not a swizzle width", rowb); return -1; }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) for (B,D,H,W,C)=(%d,%d,%d,%d,%d) box (%d,%d,%d)", (int)r, B, D, H, W, C, boxC, boxW, boxH);
    return -1;
  }
  return 0;
}

}  // namespace tc
}  // namespace vxm

extern "C" const char* vxm_last_error(void) { return vxm::g_err; }
extern "C" const char* vxm_version(void) { return "vxm_b200 0.1 sm_90a"; }
extern "C" uint64_t vxm_launch_count(void) { return vxm::g_launches.load(std::memory_order_relaxed); }
