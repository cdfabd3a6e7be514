// (The file keeps the name it had when the project targeted sm_100a.)
// Thin inline-PTX wrappers for the sm_90a features the grouped GEMM uses: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait), setmaxnreg and the wgmma
// shared-memory matrix descriptor.  Bit layouts follow the PTX ISA "warpgroup-level matrix
// shared memory layout / matrix descriptor" tables.
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace xtb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Blocking wait with a watchdog: a protocol bug traps (-> CUDA error on the host) instead of hanging
// the GPU until an external timeout kills the process.  No printf here: a function call between two wgmma
// groups makes ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();  // ~2 s at 2 GHz
  }
}

// ---- proxies / fences ---------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 2-D tiled load: coordinates are (c0 = innermost/contiguous element index, c1 = row index)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// 2-D tiled store shared -> global (bulk async-group completion).  The source tile must have been written with the
// generic proxy, fenced with fence.proxy.async.shared::cta by every writer, and the writers synchronised with the issuer.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all of this thread's bulk groups have finished READING their shared-memory source (it may be overwritten)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... have completed entirely (global writes performed)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- wgmma ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle.
//   bits [0,14)  start address >> 4        bits [16,30) leading-dim byte offset >> 4
//   bits [32,46) stride-dim byte offset >> 4     bits [62,64) layout (1 = 128-byte swizzle)
// K-major: 8-row groups `sbo` bytes apart (lbo unused).  MN-major: 64-element MN atoms `lbo`, 8-k groups `sbo` apart.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// at most N of this warpgroup's committed wgmma groups are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// pins the accumulator registers around an asynchronous wgmma
template <int N>
__device__ __forceinline__ void fence_accumulator(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int REGS>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS));
}
template <int REGS>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS));
}
// named barrier over `threads` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_barrier_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// D[64 x N, registers of one warpgroup] (+)= A[smem, 64 x 16] * B[smem, 16 x N].  TNSP = 1: MN-major operand.  Thread t
// holds, per 8-column chunk j, d[4j + {0,1}] = row 16 (t / 32) + (t % 32) / 4, columns 8j + 2 (t % 4) + {0,1}; d[4j + {2,3}]: row + 8.
#define XTB_D8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define XTB_D64(i) XTB_D8(i), XTB_D8(i + 8), XTB_D8(i + 16), XTB_D8(i + 24), XTB_D8(i + 32), XTB_D8(i + 40), XTB_D8(i + 48), XTB_D8(i + 56)
#define XTB_R16(a, b, c, d, e, f, g, h, i, j, k, l, m, n, o, p) \
  "%" #a ",%" #b ",%" #c ",%" #d ",%" #e ",%" #f ",%" #g ",%" #h ",%" #i ",%" #j ",%" #k ",%" #l ",%" #m ",%" #n ",%" #o ",%" #p
#define XTB_R64_0 XTB_R16(0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15) "," XTB_R16(16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31) "," \
  XTB_R16(32, 33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47) "," XTB_R16(48, 49, 50, 51, 52, 53, 54, 55, 56, 57, 58, 59, 60, 61, 62, 63)
#define XTB_R64_1 XTB_R16(64, 65, 66, 67, 68, 69, 70, 71, 72, 73, 74, 75, 76, 77, 78, 79) "," XTB_R16(80, 81, 82, 83, 84, 85, 86, 87, 88, 89, 90, 91, 92, 93, 94, 95) "," \
  XTB_R16(96, 97, 98, 99, 100, 101, 102, 103, 104, 105, 106, 107, 108, 109, 110, 111) "," XTB_R16(112, 113, 114, 115, 116, 117, 118, 119, 120, 121, 122, 123, 124, 125, 126, 127)
template <int TNSP_A, int TNSP_B>
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {" XTB_R64_0 "}, %64, %65, p, 1, 1, %67, %68;\n}\n"
      : XTB_D64(0)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TNSP_A), "n"(TNSP_B));
}
template <int TNSP_A, int TNSP_B>
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {" XTB_R64_0 "," XTB_R64_1 "}, %128, %129, p, 1, 1, %131, %132;\n}\n"
      : XTB_D64(0), XTB_D64(64)
      : "l"(desc_a), "l"(desc_b), "r"(accumulate), "n"(TNSP_A), "n"(TNSP_B));
}
#undef XTB_D8
#undef XTB_D64
#undef XTB_R16
#undef XTB_R64_0
#undef XTB_R64_1

}  // namespace ptx
}  // namespace xtb
