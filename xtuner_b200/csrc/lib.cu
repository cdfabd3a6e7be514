// Library-level entry points of include/xtuner_b200.h: version, error string, init, launch counter.
#include <cuda.h>

#include <cstring>
#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"

namespace xtb {

std::atomic<int64_t> g_launch_count{0};

char* error_buffer() {
  static thread_local char buf[512] = {0};
  return buf;
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(error_buffer(), 512, fmt, ap);
  va_end(ap);
  return code;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

int smem_opt_in(const void* kernel, size_t bytes) {
  int dev = 0;
  XTB_CUDA(cudaGetDevice(&dev));
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> limits;  // (kernel, device) -> its dynamic shared-memory limit
  std::lock_guard<std::mutex> lock(mu);
  auto it = limits.find({kernel, dev});
  if (it == limits.end()) {
    cudaFuncAttributes fa;
    XTB_CUDA(cudaFuncGetAttributes(&fa, kernel));
    it = limits.emplace(std::make_pair(kernel, dev), (size_t)fa.maxDynamicSharedSizeBytes).first;
  }
  if (bytes <= it->second) return XTB_OK;
  XTB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  it->second = bytes;
  return XTB_OK;
}

typedef CUresult (*PFN_ctxGetCurrent)(CUcontext*);
typedef CUresult (*PFN_ctxSetCurrent)(CUcontext);
typedef CUresult (*PFN_ptrGetAttr)(void*, CUpointer_attribute, CUdeviceptr);
static PFN_ctxGetCurrent g_ctx_get = nullptr;
static PFN_ctxSetCurrent g_ctx_set = nullptr;
static PFN_ptrGetAttr g_ptr_attr = nullptr;

static int resolve_driver_fns() {
  if (g_ctx_get && g_ctx_set && g_ptr_attr) return XTB_OK;
  cudaDriverEntryPointQueryResult q;
  void* f = nullptr;
  XTB_CUDA(cudaGetDriverEntryPoint("cuCtxGetCurrent", &f, cudaEnableDefault, &q));
  if (q != cudaDriverEntryPointSuccess || !f) return fail(XTB_ERR_CUDA, "cuCtxGetCurrent unavailable");
  g_ctx_get = reinterpret_cast<PFN_ctxGetCurrent>(f);
  XTB_CUDA(cudaGetDriverEntryPoint("cuCtxSetCurrent", &f, cudaEnableDefault, &q));
  if (q != cudaDriverEntryPointSuccess || !f) return fail(XTB_ERR_CUDA, "cuCtxSetCurrent unavailable");
  g_ctx_set = reinterpret_cast<PFN_ctxSetCurrent>(f);
  XTB_CUDA(cudaGetDriverEntryPoint("cuPointerGetAttribute", &f, cudaEnableDefault, &q));
  if (q != cudaDriverEntryPointSuccess || !f) return fail(XTB_ERR_CUDA, "cuPointerGetAttribute unavailable");
  g_ptr_attr = reinterpret_cast<PFN_ptrGetAttr>(f);
  return XTB_OK;
}

int ensure_context(const void* device_ptr) {
  static thread_local bool bound = false;
  if (bound) return XTB_OK;
  int rc = resolve_driver_fns();
  if (rc != XTB_OK) return rc;
  CUcontext cur = nullptr;
  if (g_ctx_get(&cur) == CUDA_SUCCESS && cur != nullptr) {
    bound = true;
    return XTB_OK;
  }
  CUcontext owner = nullptr;
  const CUresult r = g_ptr_attr(&owner, CU_POINTER_ATTRIBUTE_CONTEXT, reinterpret_cast<CUdeviceptr>(device_ptr));
  if (r != CUDA_SUCCESS || owner == nullptr)
    return fail(XTB_ERR_CUDA, "no CUDA context is current and pointer %p is not a device pointer (CUresult %d)",
                device_ptr, (int)r);
  if (g_ctx_set(owner) != CUDA_SUCCESS) return fail(XTB_ERR_CUDA, "cuCtxSetCurrent failed");
  bound = true;
  return XTB_OK;
}

}  // namespace xtb

extern "C" {

int xtb_version(void) { return XTB_VERSION; }

const char* xtb_last_error(void) { return xtb::error_buffer(); }

int64_t xtb_launch_count(void) { return xtb::g_launch_count.load(); }

void xtb_reset_launch_count(void) { xtb::g_launch_count.store(0); }

int xtb_tma_init_();  // group_gemm.cu

int xtb_init(void) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return xtb::fail(XTB_ERR_CUDA, "no CUDA device: %s (this library has no CPU fallback)",
                     e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  int dev = 0, major = 0, minor = 0;
  XTB_CUDA(cudaGetDevice(&dev));
  XTB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  XTB_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9)
    return xtb::fail(XTB_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", dev,
                     major, minor);
  return xtb_tma_init_();
}

}  // extern "C"
