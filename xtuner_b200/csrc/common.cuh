// Shared host/device helpers for the sm_90a kernels behind include/xtuner_b200.h.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/xtuner_b200.h"

namespace xtb {

// ---- error reporting (thread-local message, returned through xtb_last_error) --------------------
char* error_buffer();  // 512-byte thread-local buffer
int fail(int code, const char* fmt, ...);
extern std::atomic<int64_t> g_launch_count;

#define XTB_CHECK_ARG(cond, ...)                                  \
  do {                                                            \
    if (!(cond)) return ::xtb::fail(XTB_ERR_INVALID, __VA_ARGS__); \
  } while (0)

#define XTB_CUDA(expr)                                                                               \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess)                                                                           \
      return ::xtb::fail(XTB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                         __LINE__);                                                                  \
  } while (0)

inline cudaStream_t as_stream(xtb_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// Raises `kernel`'s dynamic shared-memory limit on the current device to at least `bytes`.  The default limit is 48 KB
// less the kernel's static shared memory, so a kernel with static shared memory can need this below 48 KB of dynamic
// memory.  CUDA keeps the limit per device: the limit is recorded per (kernel, device), read from the kernel on the
// first call and raised only when a launch needs more; after the first call for a pair only a lookup remains.
// Thread-safe (autograd runs the backward on its own thread).  Returns XTB_OK or an error status.
int smem_opt_in(const void* kernel, size_t bytes);

int sm_count();  // cached multiProcessorCount of the current device

// Binds a CUDA context to the calling thread if none is current (fresh autograd / worker threads have
// none until their first runtime call), using the context that owns `device_ptr`.  Driver-API entry
// points such as cuTensorMapEncodeTiled need one.  Returns XTB_OK or an error status.
int ensure_context(const void* device_ptr);

// lm_head logits GEMM with the cross-entropy epilogue (group_gemm.cu), driven by xtb_lm_head_ce (lm_head_ce.cu)
int lm_head_ce_vocab_tiles(int V);
int lm_head_logits_ce(const void* h, const void* w, const int64_t* tokens_per_expert, int64_t T, int H, int V, void* z,
                      float2* ce_part, cudaStream_t st);

#define XTB_ENSURE_CTX(ptr)                                   \
  do {                                                        \
    const int _rc = ::xtb::ensure_context(ptr);               \
    if (_rc != XTB_OK) return _rc;                            \
  } while (0)

// ---- device helpers ------------------------------------------------------------------------------
#ifdef __CUDACC__

// Programmatic dependent launch.  A kernel launched with XTB_LAUNCH(..., pdl = true, ...) may become resident while
// its predecessor in the stream is still draining (its CTAs take over SMs as the predecessor's CTAs retire, hiding launch
// latency and set-up); it must not touch global memory before pdl_sync().  Launched without the attribute, both
// instructions are no-ops.
__device__ __forceinline__ void pdl_trigger() {  // the kernel after this one may start launching too
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() {  // predecessor grids complete, their writes visible
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void pdl_sync() {
  pdl_trigger();
  pdl_wait();
}

// Every kernel of the library is launched here: raises the kernel's dynamic shared-memory limit when `smem` is above
// it (smem_opt_in), launches it (programmatic dependent launch exactly when `pdl` is set: only kernels that wait with
// pdl_sync() / pdl_wait() may take it), counts the launch and checks for a launch error.  Use XTB_LAUNCH, which
// supplies the call site and returns from the caller on error.
template <typename... P, typename... A>
inline int launch(const char* file, int line, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem,
                  cudaStream_t st, bool pdl, A&&... args) {
  if (smem > 0) {
    const int rc = smem_opt_in(reinterpret_cast<const void*>(kernel), smem);
    if (rc != XTB_OK) return rc;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, P(args)...);
  if (e != cudaSuccess) {
    cudaGetLastError();  // the refusal is not sticky: clear it, or the next launch's check would report it again
    return fail(XTB_ERR_CUDA, "kernel launch refused: %s (%s:%d)", cudaGetErrorString(e), file, line);
  }
  g_launch_count.fetch_add(1);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail(XTB_ERR_CUDA, "kernel launch: %s (%s:%d)", cudaGetErrorString(e), file, line);
  return XTB_OK;
}

#define XTB_LAUNCH(...)                                                  \
  do {                                                                   \
    const int _rc = ::xtb::launch(__FILE__, __LINE__, __VA_ARGS__);      \
    if (_rc != XTB_OK) return _rc;                                       \
  } while (0)

constexpr int kWarp = 32;

__device__ __forceinline__ float bf16_bits_to_float(uint32_t lo16) { return __uint_as_float(lo16 << 16); }

// round-to-nearest-even float -> bf16 bits (same as __float2bfloat16_rn)
__device__ __forceinline__ uint32_t float_to_bf16_bits(float f) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(f));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  return float_to_bf16_bits(lo) | (float_to_bf16_bits(hi) << 16);
}

__device__ __forceinline__ void unpack_bf16x2(uint32_t v, float& lo, float& hi) {
  lo = __uint_as_float(v << 16);
  hi = __uint_as_float(v & 0xffff0000u);
}

// one 16-byte vector of 8 bf16 <-> 8 floats, element j in f[j].  The vector is taken by reference, which leaves the
// callers' generated code as it is with four unpack_bf16x2 calls.
__device__ __forceinline__ void unpack_bf16x8(const uint4& v, float (&f)[8]) {
  unpack_bf16x2(v.x, f[0], f[1]);
  unpack_bf16x2(v.y, f[2], f[3]);
  unpack_bf16x2(v.z, f[4], f[5]);
  unpack_bf16x2(v.w, f[6], f[7]);
}
__device__ __forceinline__ uint4 pack_bf16x8(const float (&f)[8]) {
  uint4 v;
  v.x = pack_bf16x2(f[0], f[1]);
  v.y = pack_bf16x2(f[2], f[3]);
  v.z = pack_bf16x2(f[4], f[5]);
  v.w = pack_bf16x2(f[6], f[7]);
  return v;
}

// 16-byte streaming global accesses (read-once / write-once data: bypass L1 allocation)
__device__ __forceinline__ uint4 ld_stream_16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_16(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

__device__ __forceinline__ uint2 ld_stream_8(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream_8(void* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}

// SiLU pieces shared by the SwiGLU kernels and the GEMM epilogue (so forward and recomputed-in-backward
// values agree bit for bit).  sigmoid via ex2.approx + rcp: ~2 ulp in fp32, invisible after the bf16 rounding
// the reference applies to silu's output (ops/act_fn.py:9) except for rare 1-ulp bf16 flips.
__device__ __forceinline__ float sigmoid_fast(float x) { return __frcp_rn(1.f + __expf(-x)); }
__device__ __forceinline__ float silu_fast(float x) { return x * sigmoid_fast(x); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// out[i] = sum_p partial[p][i] (p < n_part, i < n), deterministic: a block owns 32 consecutive outputs, warp w adds the rows
// p = w, w + W, ... in that order with up to 8 loads in flight (a row segment is one coalesced 128-byte line), then the W
// warp sums are added in warp order.  The previous 8-lanes-per-output version chained n_part / 8 dependent 4-byte loads per
// lane from half-used sectors: 8-9 us for 2.4 MB at C2, twice per layer.
template <int W>
__global__ void __launch_bounds__(32 * W) reduce_partial_rows_kernel(const float* __restrict__ partial,
                                                                     float* __restrict__ out, int n_part, int64_t n) {
  pdl_sync();
  __shared__ float s_part[W][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t i = (int64_t)blockIdx.x * 32 + lane;
  float s = 0.f;
  if (i < n) {
    constexpr int U = 8;
    for (int p0 = w; p0 < n_part; p0 += W * U) {
      float v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int p = p0 + u * W;
        v[u] = (p < n_part) ? __ldcs(partial + (size_t)p * n + i) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) s += v[u];
    }
  }
  s_part[w][lane] = s;
  __syncthreads();
  if (w == 0 && i < n) {
    float t = s_part[0][lane];
#pragma unroll
    for (int k = 1; k < W; ++k) t += s_part[k][lane];
    out[i] = t;
  }
}

#endif  // __CUDACC__
}  // namespace xtb
