// Peer-memory (NVLink / NVSwitch) kernels for the two exchange steps of the path (SURVEY.md §8a rows a12, a14):
//   * Ulysses head<->sequence all-to-all  (xtuner/v1/ops/comm/all_to_all.py:6-51)
//   * FSDP all-gather of expert params fused with the fp32->bf16 cast, and reduce-scatter of their grads with
//     fp32 accumulation (xtuner/v1/model/base.py:650-721, model/moe/moe.py:1197-1217)
//
// All buffers that peers touch are "symmetric": every rank allocates the same size and all ranks' virtual
// addresses are visible to every rank (mapped by the host with torch.distributed._symmetric_memory or CUDA
// IPC); the kernels receive a DEVICE array of the world's base pointers.  One-hop algorithms (NVSwitch gives
// every pair full bandwidth): each rank PULLS what it needs straight into the final layout (all-to-all,
// reduce-scatter) or PUSHES its cast shard to every peer (all-gather).  No ring; the only extra copy is the host
// wrapper's copy-in of a non-symmetric tensor into its symmetric staging buffer (xtuner_b200/comm.py).
//
// Ordering between ranks is provided by xtb_peer_barrier (signal pads in symmetric memory, system-scope
// release/acquire), enqueued by the host wrapper on the same stream before (data ready) the transfer; double
// buffering on the host side makes a second barrier unnecessary.
#include <cstdlib>

#include "common.cuh"

namespace xtb {

// ---- system-scope signalling -----------------------------------------------------------------------------
__device__ __forceinline__ void put_signal_sys(uint32_t* addr) {
  uint32_t old;
  do {
    asm volatile("atom.global.release.sys.cas.b32 %0, [%1], 0, 1;" : "=r"(old) : "l"(addr) : "memory");
  } while (old != 0u);
}
__device__ __forceinline__ void wait_signal_sys(uint32_t* addr) {
  uint32_t old;
  long long t0 = clock64();
  do {
    asm volatile("atom.global.acquire.sys.cas.b32 %0, [%1], 1, 0;" : "=r"(old) : "l"(addr) : "memory");
    if (old != 1u && clock64() - t0 > 20000000000ll) {  // ~10 s: a peer died; trap instead of hanging forever
      printf("xtuner_b200: peer barrier timed out\n");
      __trap();
    }
  } while (old != 1u);
}

// One block; thread r < world: tell rank r "I arrived" and wait for rank r's arrival.  pad[channel*world + src].
__global__ void peer_barrier_kernel(uint32_t* const* __restrict__ pads, int me, int world, int channel) {
  const int r = threadIdx.x;
  if (r < world && r != me) {
    put_signal_sys(pads[r] + (size_t)channel * world + me);
    wait_signal_sys(pads[me] + (size_t)channel * world + r);
  }
}

__device__ __forceinline__ uint4 ld_peer_16(const void* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}

// ---- a12: all-to-all pull with layout transform -------------------------------------------------------------
// rows are indexed (o, x, m); row length L bytes (multiple of 16); blockIdx.y = source rank.
struct A2AArgs {
  long long n_o, n_x, n_m;
  long long row_vec;                 // L / 16
  long long s_o, s_x, s_m, s_base;   // source offsets in 16-byte units (s_base already includes `me`)
  long long d_o, d_x, d_m, d_peer;   // destination offsets in 16-byte units; base = src * d_peer
};

__global__ void __launch_bounds__(256) a2a_pull_kernel(const uint4* const* __restrict__ peer_in,
                                                       uint4* __restrict__ out, A2AArgs a) {
  const int src = blockIdx.y;
  const uint4* in = peer_in[src];
  const long long total = a.n_o * a.n_x * a.n_m * a.row_vec;
  const long long stride = (long long)gridDim.x * blockDim.x;
  constexpr int U = 8;
  for (long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i0 < total; i0 += stride * U) {
    uint4 buf[U];
    long long doff[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + (long long)u * stride;
      if (i < total) {
        const long long v = i % a.row_vec;
        long long row = i / a.row_vec;
        const long long m = row % a.n_m;
        row /= a.n_m;
        const long long x = row % a.n_x;
        const long long o = row / a.n_x;
        buf[u] = ld_peer_16(in + a.s_base + o * a.s_o + x * a.s_x + m * a.s_m + v);
        doff[u] = (long long)src * a.d_peer + o * a.d_o + x * a.d_x + m * a.d_m + v;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + (long long)u * stride;
      if (i < total) st_stream_16(out + doff[u], buf[u]);
    }
  }
}

// ---- a14: all-gather push (optionally casting fp32 -> bf16 on the way) ---------------------------------------
// every rank writes its shard (n_vec 16-byte bf16 vectors) at offset me*n_vec of EVERY rank's output buffer
template <bool FROM_F32>
__global__ void __launch_bounds__(256) allgather_push_kernel(const void* __restrict__ local_in,
                                                             uint4* const* __restrict__ peer_out, int me, int world,
                                                             long long n_vec) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    uint4 v;
    if constexpr (FROM_F32) {
      const float4* src = reinterpret_cast<const float4*>(local_in) + 2 * i;
      const float4 a = __ldcs(src), b = __ldcs(src + 1);
      v.x = pack_bf16x2(a.x, a.y);
      v.y = pack_bf16x2(a.z, a.w);
      v.z = pack_bf16x2(b.x, b.y);
      v.w = pack_bf16x2(b.z, b.w);
    } else {
      v = ld_stream_16(reinterpret_cast<const uint4*>(local_in) + i);
    }
    for (int r = 0; r < world; ++r) {
      const int dst = (me + r) % world;  // stagger destinations so ranks do not all hit the same peer at once
      st_stream_16(peer_out[dst] + (long long)me * n_vec + i, v);
    }
  }
}

// ---- a14: reduce-scatter pull: out[i] = scale * sum_r float(in_r[me*n + i]), fixed rank order (deterministic) ---
template <bool OUT_F32>
__global__ void __launch_bounds__(256) reduce_scatter_pull_kernel(const uint4* const* __restrict__ peer_in,
                                                                  void* __restrict__ out, int me, int world,
                                                                  long long n_vec, float scale) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int r0 = 0; r0 < world; r0 += 4) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (r0 + j < world) v[j] = ld_peer_16(peer_in[r0 + j] + (long long)me * n_vec + i);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (r0 + j < world) {
          float f[8];
          unpack_bf16x2(v[j].x, f[0], f[1]);
          unpack_bf16x2(v[j].y, f[2], f[3]);
          unpack_bf16x2(v[j].z, f[4], f[5]);
          unpack_bf16x2(v[j].w, f[6], f[7]);
#pragma unroll
          for (int q = 0; q < 8; ++q) acc[q] += f[q];
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[q] *= scale;
    if constexpr (OUT_F32) {
      float4* dst = reinterpret_cast<float4*>(out) + 2 * i;
      dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
      dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    } else {
      uint4 o;
      o.x = pack_bf16x2(acc[0], acc[1]);
      o.y = pack_bf16x2(acc[2], acc[3]);
      o.z = pack_bf16x2(acc[4], acc[5]);
      o.w = pack_bf16x2(acc[6], acc[7]);
      st_stream_16(reinterpret_cast<uint4*>(out) + i, o);
    }
  }
}

// ---- a16: one-shot all-reduce of the (small) replicated gradients: out[i] = scale * sum_r in_r[i] in fp32, fixed rank
// order on every rank => bit-identical results everywhere (model/moe/moe.py:1381-1390 averages them with NCCL) -----------
__global__ void __launch_bounds__(256) allreduce_pull_f32_kernel(const float4* const* __restrict__ peer_in,
                                                                 float4* __restrict__ out, int world, long long n_vec,
                                                                 float scale) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r0 = 0; r0 < world; r0 += 4) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (r0 + j < world) v[j] = ld_peer_16(peer_in[r0 + j] + i);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (r0 + j < world) {
          acc.x += __uint_as_float(v[j].x);
          acc.y += __uint_as_float(v[j].y);
          acc.z += __uint_as_float(v[j].z);
          acc.w += __uint_as_float(v[j].w);
        }
      }
    }
    out[i] = make_float4(acc.x * scale, acc.y * scale, acc.z * scale, acc.w * scale);
  }
}

// CTAs of an exchange kernel: 2 per SM.  The kernels run under the grouped GEMMs of the neighbouring layer; capping the
// grid lower makes the exchange outlast the compute it hides under.  The grid size has not been measured on H100.
static int comm_blocks(long long n_vec) {
  const long long want = (n_vec + 256 * 8 - 1) / (256 * 8);
  return (int)max(1ll, min(want, (long long)sm_count() * 2));
}

}  // namespace xtb

using namespace xtb;

extern "C" int xtb_peer_barrier(void* const* signal_pad_ptrs_dev, int rank, int world, int channel,
                                xtb_stream_t stream) {
  XTB_CHECK_ARG(signal_pad_ptrs_dev, "xtb_peer_barrier: null pointer");
  XTB_CHECK_ARG(world >= 1 && world <= 64 && rank >= 0 && rank < world && channel >= 0, "xtb_peer_barrier: bad rank/world");
  XTB_ENSURE_CTX(signal_pad_ptrs_dev);
  if (world == 1) return XTB_OK;
  XTB_LAUNCH(peer_barrier_kernel, dim3(1), dim3(64), 0, as_stream(stream), false,
             reinterpret_cast<uint32_t* const*>(signal_pad_ptrs_dev), rank, world, channel);
  return XTB_OK;
}

extern "C" int xtb_a2a_pull(void* const* peer_in_ptrs_dev, void* out, int rank, int world, int64_t n_o, int64_t n_x,
                            int64_t n_m, int64_t row_bytes, int64_t src_stride_o, int64_t src_stride_x,
                            int64_t src_stride_m, int64_t src_base, int64_t dst_stride_o, int64_t dst_stride_x,
                            int64_t dst_stride_m, int64_t dst_peer_stride, xtb_stream_t stream) {
  XTB_CHECK_ARG(peer_in_ptrs_dev && out, "xtb_a2a_pull: null pointer");
  XTB_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "xtb_a2a_pull: bad rank/world");
  XTB_CHECK_ARG(n_o >= 0 && n_x >= 0 && n_m >= 0 && row_bytes > 0 && row_bytes % 16 == 0,
                "xtb_a2a_pull: row_bytes=%lld must be a positive multiple of 16", (long long)row_bytes);
  XTB_CHECK_ARG((src_stride_o | src_stride_x | src_stride_m | src_base | dst_stride_o | dst_stride_x | dst_stride_m |
                 dst_peer_stride) % 16 == 0,
                "xtb_a2a_pull: strides must be multiples of 16 bytes");
  XTB_ENSURE_CTX(out);
  if (n_o * n_x * n_m == 0) return XTB_OK;
  A2AArgs a;
  a.n_o = n_o; a.n_x = n_x; a.n_m = n_m; a.row_vec = row_bytes / 16;
  a.s_o = src_stride_o / 16; a.s_x = src_stride_x / 16; a.s_m = src_stride_m / 16; a.s_base = src_base / 16;
  a.d_o = dst_stride_o / 16; a.d_x = dst_stride_x / 16; a.d_m = dst_stride_m / 16; a.d_peer = dst_peer_stride / 16;
  const long long total = n_o * n_x * n_m * a.row_vec;
  const int per_src = max(1, min((int)((total + 256 * 8 - 1) / (256 * 8)), max(1, sm_count() * 2 / world)));
  dim3 grid(per_src, world);
  XTB_LAUNCH(a2a_pull_kernel, grid, dim3(256), 0, as_stream(stream), false,
             reinterpret_cast<const uint4* const*>(peer_in_ptrs_dev), static_cast<uint4*>(out), a);
  return XTB_OK;
}

extern "C" int xtb_allgather_push(const void* local_in, void* const* peer_out_ptrs_dev, int rank, int world,
                                  int64_t n_local_elems, int in_is_f32, xtb_stream_t stream) {
  XTB_CHECK_ARG(local_in && peer_out_ptrs_dev, "xtb_allgather_push: null pointer");
  XTB_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "xtb_allgather_push: bad rank/world");
  XTB_CHECK_ARG(n_local_elems >= 0 && n_local_elems % 8 == 0, "xtb_allgather_push: n_local_elems must be a multiple of 8");
  XTB_ENSURE_CTX(local_in);
  if (n_local_elems == 0) return XTB_OK;
  const long long n_vec = n_local_elems / 8;
  const int blocks = comm_blocks(n_vec);
  XTB_LAUNCH(in_is_f32 ? allgather_push_kernel<true> : allgather_push_kernel<false>, dim3(blocks), dim3(256), 0,
             as_stream(stream), false, local_in, reinterpret_cast<uint4* const*>(peer_out_ptrs_dev), rank, world, n_vec);
  return XTB_OK;
}

extern "C" int xtb_reduce_scatter_pull(void* const* peer_in_ptrs_dev, void* out, int rank, int world,
                                       int64_t n_local_elems, float scale, int out_is_f32, xtb_stream_t stream) {
  XTB_CHECK_ARG(peer_in_ptrs_dev && out, "xtb_reduce_scatter_pull: null pointer");
  XTB_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "xtb_reduce_scatter_pull: bad rank/world");
  XTB_CHECK_ARG(n_local_elems >= 0 && n_local_elems % 8 == 0, "xtb_reduce_scatter_pull: n_local_elems must be a multiple of 8");
  XTB_ENSURE_CTX(out);
  if (n_local_elems == 0) return XTB_OK;
  const long long n_vec = n_local_elems / 8;
  const int blocks = comm_blocks(n_vec);
  XTB_LAUNCH(out_is_f32 ? reduce_scatter_pull_kernel<true> : reduce_scatter_pull_kernel<false>, dim3(blocks), dim3(256),
             0, as_stream(stream), false, reinterpret_cast<const uint4* const*>(peer_in_ptrs_dev), out, rank, world, n_vec,
             scale);
  return XTB_OK;
}

extern "C" int xtb_allreduce_pull_f32(void* const* peer_in_ptrs_dev, void* out, int rank, int world, int64_t n_elems,
                                      float scale, xtb_stream_t stream) {
  XTB_CHECK_ARG(peer_in_ptrs_dev && out, "xtb_allreduce_pull_f32: null pointer");
  XTB_CHECK_ARG(world >= 1 && rank >= 0 && rank < world, "xtb_allreduce_pull_f32: bad rank/world");
  XTB_CHECK_ARG(n_elems >= 0 && n_elems % 4 == 0, "xtb_allreduce_pull_f32: n_elems must be a multiple of 4");
  XTB_ENSURE_CTX(out);
  if (n_elems == 0) return XTB_OK;
  const long long n_vec = n_elems / 4;
  XTB_LAUNCH(allreduce_pull_f32_kernel, dim3(comm_blocks(n_vec)), dim3(256), 0, as_stream(stream), false,
             reinterpret_cast<const float4* const*>(peer_in_ptrs_dev), static_cast<float4*>(out), world, n_vec, scale);
  return XTB_OK;
}

// ---- exchange on the copy engines: a batch of device-to-device copies between (peer-mapped) addresses.  Used by the
// FSDP engine's XTB_FSDP_DMA mode: no SM is taken from the GEMMs the exchange runs under; ordering between ranks stays
// with xtb_peer_barrier.  Host arrays.
extern "C" int xtb_peer_memcpy_batch(void* const* dst_ptrs_host, const void* const* src_ptrs_host,
                                     const int64_t* nbytes_host, int n, xtb_stream_t stream) {
  XTB_CHECK_ARG(dst_ptrs_host && src_ptrs_host && nbytes_host, "xtb_peer_memcpy_batch: null pointer");
  XTB_CHECK_ARG(n >= 0 && n <= 4096, "xtb_peer_memcpy_batch: bad n=%d", n);
  // every entry is checked before the first copy is enqueued: a refused batch copies nothing
  for (int i = 0; i < n; ++i)
    XTB_CHECK_ARG(dst_ptrs_host[i] && src_ptrs_host[i] && nbytes_host[i] >= 0, "xtb_peer_memcpy_batch: bad entry %d", i);
  cudaStream_t st = as_stream(stream);
  for (int i = 0; i < n; ++i) {
    if (nbytes_host[i] == 0 || dst_ptrs_host[i] == src_ptrs_host[i]) continue;
    XTB_ENSURE_CTX(src_ptrs_host[i]);
    XTB_CUDA(cudaMemcpyAsync(dst_ptrs_host[i], src_ptrs_host[i], (size_t)nbytes_host[i], cudaMemcpyDeviceToDevice, st));
  }
  return XTB_OK;
}
