// Dropless token dispatch / combine (SURVEY.md §8a rows a4, a5): stable bucketing of the flat
// [T*K] expert ids, row gather into expert-sorted order, and the probability-weighted combine with its
// backward.  HBM-bound byte movers: 16-byte vectorised, L1-bypassing accesses; index work is a
// two-level counting sort (per-chunk histograms -> scan -> per-chunk stable ranks with no sort pass).
//
// Index scheme
//   chunk c        = CT = 32 consecutive tokens (CT*K consecutive flat indices); the scatter kernel works on
//                    sub-chunks of 8 tokens and ranks against the preceding entries of its chunk
//   counts[c][e]   = number of entries of expert e in chunk c; after the scan: exclusive prefix over c
//   expert_start[e]= exclusive prefix of tokens_per_expert
//   dest(f)        = expert_start[e] + counts[c][e] + |{ f' in chunk c, f' < f, id[f'] == e }|
// which is exactly the position a stable sort by expert id assigns (reference: argsort(stable=True),
// ops/moe/cuda/permute_unpermute.py:215).
#include "common.cuh"
#include "dispatch_scan.cuh"

namespace xtb {

// ---- kernel A: per-chunk histograms; the last block to finish turns them into exclusive prefixes -----
__global__ void __launch_bounds__(256) permute_count_scan_kernel(const int32_t* __restrict__ ids, int T, int K,
                                                                 int E, int n_chunks, int* __restrict__ counts,
                                                                 int* __restrict__ expert_start,
                                                                 unsigned long long* __restrict__ tokens_per_expert,
                                                                 unsigned* __restrict__ ticket) {
  extern __shared__ int s_mem[];  // [warps_per_block][E] histograms; reused by the scan
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int warps_per_block = blockDim.x >> 5;
  int* hist = s_mem + warp * E;
  const int64_t total = (int64_t)T * K;

  for (int c = blockIdx.x * warps_per_block + warp; c < n_chunks; c += gridDim.x * warps_per_block) {
    for (int e = lane; e < E; e += 32) hist[e] = 0;
    __syncwarp();
    const int64_t f0 = (int64_t)c * kChunkTokens * K;
    const int64_t f1 = min(total, f0 + (int64_t)kChunkTokens * K);
    for (int64_t f = f0 + lane; f < f1; f += 32) {
      const int e = ids[f];
      if (e >= 0 && e < E) atomicAdd(&hist[e], 1);
    }
    __syncwarp();
    for (int e = lane; e < E; e += 32) counts[(size_t)c * E + e] = hist[e];
    __syncwarp();
  }

  scan_counts_last_block(counts, expert_start, tokens_per_expert, ticket, n_chunks, E, s_mem);
}

// ---- kernel B: per-chunk stable ranks -> maps, then the row gather/scatter ---------------------------
// The index work of one block (sub-chunk `sub` of chunk `c`), shared by both scatter kernels: the chunk's ids up to the
// end of the sub-chunk into s_ids, then each entry's stable rank among the preceding entries of its chunk gives its
// destination row, written to s_dest (for the row movement), row_id_map and sorted_indices.  Ends on a barrier.
__device__ __forceinline__ void scatter_index(const int32_t* __restrict__ ids, int T, int K, int E, int c, int sub,
                                              const int* __restrict__ counts, const int* __restrict__ expert_start,
                                              int* s_ids, int* s_dest, int32_t* __restrict__ row_id_map,
                                              int64_t* __restrict__ sorted_indices) {
  const int64_t fc = (int64_t)c * kChunkTokens * K;  // first flat index of the chunk
  const int base = sub * kSubTokens * K;             // entries of the chunk that precede this block
  const int n_mine = (int)min((int64_t)kSubTokens * K, (int64_t)T * K - (fc + base));
  const int n_load = base + n_mine;
  for (int j = threadIdx.x; j < n_load; j += blockDim.x) s_ids[j] = ids[fc + j];
  __syncthreads();
  for (int j = threadIdx.x; j < n_mine; j += blockDim.x) {
    const int e = s_ids[base + j];
    int rank = 0;
    for (int i = 0; i < base + j; ++i) rank += (s_ids[i] == e);
    const int dest = (e >= 0 && e < E) ? expert_start[e] + counts[(size_t)c * E + e] + rank : -1;
    s_dest[j] = dest;
    row_id_map[fc + base + j] = dest;
    if (sorted_indices && dest >= 0) sorted_indices[dest] = fc + base + j;
  }
  __syncthreads();
}

// One block per sub-chunk.  The rows pass through registers: the path for rows too long to stage kSubTokens of in shared
// memory (kernel B' below).
__global__ void __launch_bounds__(128) permute_scatter_kernel(const uint4* __restrict__ x,
                                                              const int32_t* __restrict__ ids, int T, int K, int E,
                                                              int row_vec /* 16-byte vectors per row */,
                                                              const int* __restrict__ counts,
                                                              const int* __restrict__ expert_start,
                                                              uint4* __restrict__ permuted,
                                                              int32_t* __restrict__ row_id_map,
                                                              int64_t* __restrict__ sorted_indices) {
  pdl_sync();
  extern __shared__ int s_buf[];  // ids of the chunk up to the end of this sub-chunk [<= CT*K] | dest [SUB*K]
  constexpr int kSubPerChunk = kChunkTokens / kSubTokens;
  const int c = blockIdx.x / kSubPerChunk;           // histogram chunk
  const int sub = blockIdx.x % kSubPerChunk;         // sub-chunk inside it
  const int t0 = c * kChunkTokens + sub * kSubTokens;  // first token of this block
  if (t0 >= T) return;
  int* s_dest = s_buf + kChunkTokens * K;
  scatter_index(ids, T, K, E, c, sub, counts, expert_start, s_buf, s_dest, row_id_map, sorted_indices);

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  const int t_in_block = min(kSubTokens, T - t0);
  for (int tt = warp; tt < t_in_block; tt += n_warps) {
    const uint4* src = x + (size_t)(t0 + tt) * row_vec;
    for (int v0 = 0; v0 < row_vec; v0 += 32 * 8) {
      uint4 buf[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int v = v0 + u * 32 + lane;
        if (v < row_vec) buf[u] = ld_stream_16(src + v);
      }
      for (int k = 0; k < K; ++k) {
        const int dest = s_dest[tt * K + k];
        if (dest < 0) continue;
        uint4* dst = permuted + (size_t)dest * row_vec;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int v = v0 + u * 32 + lane;
          if (v < row_vec) st_stream_16(dst + v, buf[u]);
        }
      }
    }
  }
}

// ---- kernel B', rows moved by the bulk-copy engine (TMA, cp.async.bulk: SASS UBLKCP) ---------------------------------
// Same index work as permute_scatter_kernel (scatter_index); the token rows never pass through registers: thread 0 stages the block's
// kSubTokens rows in shared memory with one bulk load each (issued BEFORE the index work, which they overlap) and, as
// each row lands (mbarrier complete_tx), one lane fans it out to its K destinations with bulk stores.
__device__ __forceinline__ uint32_t pm_smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__global__ void __launch_bounds__(128) permute_scatter_bulk_kernel(const uint8_t* __restrict__ x,
                                                                   const int32_t* __restrict__ ids, int T, int K, int E,
                                                                   uint32_t row_bytes, const int* __restrict__ counts,
                                                                   const int* __restrict__ expert_start,
                                                                   uint8_t* __restrict__ permuted,
                                                                   int32_t* __restrict__ row_id_map,
                                                                   int64_t* __restrict__ sorted_indices) {
  pdl_sync();
  extern __shared__ __align__(128) uint8_t s_raw[];
  constexpr int kSubPerChunk = kChunkTokens / kSubTokens;
  const int c = blockIdx.x / kSubPerChunk;
  const int sub = blockIdx.x % kSubPerChunk;
  const int t0 = c * kChunkTokens + sub * kSubTokens;
  if (t0 >= T) return;
  uint8_t* s_rows = s_raw;                                                   // [kSubTokens][row_bytes]
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_rows + (size_t)kSubTokens * row_bytes);  // [kSubTokens]
  int* s_ids = reinterpret_cast<int*>(s_bar + kSubTokens);
  int* s_dest = s_ids + kChunkTokens * K;
  const int t_in_block = min(kSubTokens, T - t0);
  if (threadIdx.x == 0) {
    for (int tt = 0; tt < t_in_block; ++tt)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(pm_smem_u32(&s_bar[tt])) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    for (int tt = 0; tt < t_in_block; ++tt) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(pm_smem_u32(&s_bar[tt])), "r"(row_bytes) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                       pm_smem_u32(s_rows + (size_t)tt * row_bytes)),
                   "l"(x + (size_t)(t0 + tt) * row_bytes), "r"(row_bytes), "r"(pm_smem_u32(&s_bar[tt]))
                   : "memory");
    }
  }
  scatter_index(ids, T, K, E, c, sub, counts, expert_start, s_ids, s_dest, row_id_map, sorted_indices);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  if (lane == 0) {
    for (int tt = warp; tt < t_in_block; tt += n_warps) {
      uint32_t ok = 0;
      while (!ok)  // the row has landed (phase 0 of its barrier)
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(pm_smem_u32(&s_bar[tt])) : "memory");
      for (int k = 0; k < K; ++k) {
        const int dest = s_dest[tt * K + k];
        if (dest < 0) continue;
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(permuted + (size_t)dest * row_bytes),
                     "r"(pm_smem_u32(s_rows + (size_t)tt * row_bytes)), "r"(row_bytes)
                     : "memory");
      }
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory stays valid until the stores have read it
  }
}

// combined = bf16(acc); optionally  bf16(combined * hidden_factor)  then  bf16(. + residual)  — the two eager
// ops of MoEDecoderLayer._post_moe_forward (moe_decoder_layer.py:696-705) with their bf16 roundings.
__device__ __forceinline__ float rbf(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ uint4 combine_epilogue(const float (&acc)[8], const uint4* __restrict__ residual,
                                                  float hidden_factor, size_t vec_index) {
  float c[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) c[j] = acc[j];
  if (residual != nullptr) {
    float r[8];
    unpack_bf16x8(ld_stream_16(residual + vec_index), r);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = rbf(c[j]);
      if (hidden_factor != 1.0f) v = rbf(v * hidden_factor);
      c[j] = v + r[j];
    }
  } else if (hidden_factor != 1.0f) {
#pragma unroll
    for (int j = 0; j < 8; ++j) c[j] = rbf(c[j]) * hidden_factor;
  }
  return pack_bf16x8(c);
}

// ---- a5 unpermute (combine): one warp per token -----------------------------------------------------
template <int KT>  // KT > 0: compile-time K; KT == 0: runtime K
__global__ void __launch_bounds__(256) unpermute_kernel(const uint4* __restrict__ y,
                                                        const int32_t* __restrict__ row_id_map,
                                                        const float* __restrict__ probs, int T, int K_rt,
                                                        int row_vec, uint4* __restrict__ out,
                                                        const uint4* __restrict__ residual, float hidden_factor) {
  pdl_sync();
  const int K = KT > 0 ? KT : K_rt;
  const int lane = threadIdx.x & 31;
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= T) return;
  constexpr int KMAX = KT > 0 ? KT : 1;
  if constexpr (KT > 0) {
    int rows[KMAX];
    float p[KMAX];
#pragma unroll
    for (int k = 0; k < KT; ++k) {
      rows[k] = row_id_map[(size_t)t * KT + k];
      p[k] = probs ? probs[(size_t)t * KT + k] : 1.f;
    }
    constexpr int U = (KT <= 2) ? 4 : (KT <= 4 ? 2 : 1);
    for (int v0 = lane; v0 < row_vec; v0 += 32 * U) {
      uint4 in[U][KMAX];
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int k = 0; k < KT; ++k) {
          const int v = v0 + u * 32;
          if (v < row_vec && rows[k] >= 0) in[u][k] = ld_stream_16(y + (size_t)rows[k] * row_vec + v);
          else in[u][k] = make_uint4(0, 0, 0, 0);
        }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int v = v0 + u * 32;
        if (v >= row_vec) continue;
        float acc[8];
#pragma unroll
        for (int k = 0; k < KT; ++k) {
          float f[8];
          unpack_bf16x8(in[u][k], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            // products are rounded before the add, as in `(tokens * probs).sum(dim=1)` of the reference
            const float prod = probs ? __fmul_rn(f[j], p[k]) : f[j];
            acc[j] = (k == 0) ? prod : __fadd_rn(acc[j], prod);
          }
        }
        st_stream_16(out + (size_t)t * row_vec + v, combine_epilogue(acc, residual, hidden_factor, (size_t)t * row_vec + v));
      }
    }
  } else {
    for (int v = lane; v < row_vec; v += 32) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      for (int k = 0; k < K; ++k) {
        const int r = row_id_map[(size_t)t * K + k];
        if (r < 0) continue;
        const float pk = probs ? probs[(size_t)t * K + k] : 1.f;
        const uint4 in = ld_stream_16(y + (size_t)r * row_vec + v);
        float f[8];
        unpack_bf16x8(in, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float prod = probs ? __fmul_rn(f[j], pk) : f[j];
          acc[j] = (k == 0) ? prod : __fadd_rn(acc[j], prod);
        }
      }
      st_stream_16(out + (size_t)t * row_vec + v, combine_epilogue(acc, residual, hidden_factor, (size_t)t * row_vec + v));
    }
  }
}

// ---- a5 backward: act_grad rows + prob_grad, one warp per token ---------------------------------------
__global__ void __launch_bounds__(256) unpermute_bwd_kernel(const uint4* __restrict__ grad_out,
                                                            const uint4* __restrict__ y_fwd,
                                                            const int32_t* __restrict__ row_id_map,
                                                            const float* __restrict__ probs, int T, int K,
                                                            int row_vec, uint4* __restrict__ act_grad,
                                                            float* __restrict__ prob_grad) {
  pdl_sync();
  const int lane = threadIdx.x & 31;
  const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (t >= T) return;
  for (int k = 0; k < K; ++k) {
    const int r = row_id_map[(size_t)t * K + k];
    const float pk = probs ? probs[(size_t)t * K + k] : 1.f;
    float dot = 0.f;
    if (r >= 0) {
      for (int v0 = lane; v0 < row_vec; v0 += 32 * 4) {
        uint4 g[4], yv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int v = v0 + u * 32;
          if (v < row_vec) {
            g[u] = __ldg(grad_out + (size_t)t * row_vec + v);  // re-read K times: keep in L1
            if (prob_grad) yv[u] = ld_stream_16(y_fwd + (size_t)r * row_vec + v);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int v = v0 + u * 32;
          if (v >= row_vec) continue;
          float gf[8];
          unpack_bf16x8(g[u], gf);
          uint4 o;
          o.x = pack_bf16x2(gf[0] * pk, gf[1] * pk);
          o.y = pack_bf16x2(gf[2] * pk, gf[3] * pk);
          o.z = pack_bf16x2(gf[4] * pk, gf[5] * pk);
          o.w = pack_bf16x2(gf[6] * pk, gf[7] * pk);
          st_stream_16(act_grad + (size_t)r * row_vec + v, o);
          if (prob_grad) {
            float yf[8];
            unpack_bf16x8(yv[u], yf);
#pragma unroll
            for (int j = 0; j < 8; ++j) dot = fmaf(gf[j], yf[j], dot);
          }
        }
      }
    }
    if (prob_grad) {
      dot = warp_sum(dot);
      if (lane == 0) prob_grad[(size_t)t * K + k] = dot;
    }
  }
}

// ---- a8 swiglu fwd / bwd: 8 elements per thread --------------------------------------------------------
__device__ __forceinline__ float silu_f(float x) { return silu_fast(x); }
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__global__ void __launch_bounds__(256) swiglu_kernel(const uint4* __restrict__ h, uint4* __restrict__ out,
                                                     int64_t M, int I8 /* I/8 */) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * I8) return;
  const int64_t m = idx / I8;
  const int j = (int)(idx % I8);
  const uint4 g = ld_stream_16(h + m * (2 * I8) + j);
  const uint4 u = ld_stream_16(h + m * (2 * I8) + I8 + j);
  const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, uw[4] = {u.x, u.y, u.z, u.w};
  uint32_t ow[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float g0, g1, u0, u1;
    unpack_bf16x2(gw[q], g0, g1);
    unpack_bf16x2(uw[q], u0, u1);
    const float s0 = round_bf16(silu_f(g0)), s1 = round_bf16(silu_f(g1));
    ow[q] = pack_bf16x2(s0 * u0, s1 * u1);
  }
  st_stream_16(out + idx, make_uint4(ow[0], ow[1], ow[2], ow[3]));
}

// One element pair of the SwiGLU backward with the reference's rounding points (ops/act_fn.py:7-9 under autograd).
__device__ __forceinline__ void swiglu_bwd_vec(const uint4& g, const uint4& u, const uint4& go, uint4& o_g, uint4& o_u) {
  const uint32_t gw[4] = {g.x, g.y, g.z, g.w}, uw[4] = {u.x, u.y, u.z, u.w}, dw[4] = {go.x, go.y, go.z, go.w};
  uint32_t o1[4], o2[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float x1[2], x2[2], d[2], r1[2], r2[2];
    unpack_bf16x2(gw[q], x1[0], x1[1]);
    unpack_bf16x2(uw[q], x2[0], x2[1]);
    unpack_bf16x2(dw[q], d[0], d[1]);
#pragma unroll
    for (int z = 0; z < 2; ++z) {
      const float sig = sigmoid_fast(x1[z]);
      const float s = round_bf16(x1[z] * sig);    // forward's silu output (a bf16 tensor), recomputed identically
      r2[z] = d[z] * s;                           // grad wrt x2  (rounded at pack)
      const float ds = round_bf16(d[z] * x2[z]);  // grad wrt silu output, a bf16 tensor in the reference
      r1[z] = ds * sig * (1.f + x1[z] * (1.f - sig));
    }
    o1[q] = pack_bf16x2(r1[0], r1[1]);
    o2[q] = pack_bf16x2(r2[0], r2[1]);
  }
  o_g = make_uint4(o1[0], o1[1], o1[2], o1[3]);
  o_u = make_uint4(o2[0], o2[1], o2[2], o2[3]);
}

// A 64-bit divide per thread to find its row, with one 16-byte vector per thread, is instruction-bound.  A block owns
// kSwRows consecutive rows, the row of a vector comes from a
// 32-bit multiply-high with a host-made reciprocal, and every thread keeps two vectors' loads in flight.
constexpr int kSwRows = 8;
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const uint4* __restrict__ grad_out,
                                                         const uint4* __restrict__ h, uint4* __restrict__ grad_h,
                                                         int64_t M, int I8, uint32_t inv_I8 /* ceil(2^32 / I8) */) {
  pdl_sync();
  const int64_t m0 = (int64_t)blockIdx.x * kSwRows;
  const int rows = (int)min((int64_t)kSwRows, M - m0);
  const uint32_t n = (uint32_t)rows * (uint32_t)I8;  // vectors of this block (small: the reciprocal trick is exact)
  const uint4* hb = h + m0 * (2 * I8);
  const uint4* gb = grad_out + m0 * I8;
  uint4* ob = grad_h + m0 * (2 * I8);
  for (uint32_t i0 = threadIdx.x; i0 < n; i0 += 2 * blockDim.x) {
    uint32_t i[2], r[2], j[2];
    uint4 g[2], u[2], go[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      i[k] = i0 + k * blockDim.x;
      r[k] = (I8 == 1) ? i[k] : __umulhi(i[k], inv_I8);  // ceil(2^32 / 1) does not fit 32 bits
      j[k] = i[k] - r[k] * (uint32_t)I8;
      if (i[k] < n) {
        g[k] = ld_stream_16(hb + (size_t)r[k] * (2 * I8) + j[k]);
        u[k] = ld_stream_16(hb + (size_t)r[k] * (2 * I8) + I8 + j[k]);
        go[k] = ld_stream_16(gb + i[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (i[k] < n) {
        uint4 og, ou;
        swiglu_bwd_vec(g[k], u[k], go[k], og, ou);
        st_stream_16(ob + (size_t)r[k] * (2 * I8) + j[k], og);
        st_stream_16(ob + (size_t)r[k] * (2 * I8) + I8 + j[k], ou);
      }
    }
  }
}

}  // namespace xtb

using namespace xtb;

extern "C" size_t xtb_moe_permute_workspace_bytes(int T, int K, int E) {
  (void)K;
  if (T < 0 || E <= 0) return 0;
  return 256 + align_up((size_t)E * sizeof(int), 256) + align_up((size_t)n_chunks_of(T) * E * sizeof(int), 256);
}

static int permute_impl(const void* x, const int32_t* ids, int T, int K, int E, int64_t row_bytes, void* permuted,
                        int32_t* row_id_map, int64_t* sorted_indices, int64_t* tokens_per_expert, void* workspace,
                        xtb_stream_t stream, bool prepared) {
  XTB_CHECK_ARG(ids && row_id_map && workspace, "xtb_moe_permute: null pointer");
  XTB_CHECK_ARG(T >= 0 && K > 0 && K <= 64 && E > 0 && E <= 1024, "xtb_moe_permute: bad T=%d K=%d E=%d", T, K, E);
  XTB_CHECK_ARG((int64_t)T * K < (1ll << 31), "xtb_moe_permute: T*K overflows int32");
  XTB_ENSURE_CTX(ids);
  XTB_CHECK_ARG(x && permuted, "xtb_moe_permute: null activation pointer");
  XTB_CHECK_ARG(row_bytes > 0 && row_bytes % 16 == 0, "xtb_moe_permute: row_bytes=%lld must be a multiple of 16",
                (long long)row_bytes);
  XTB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(permuted)) % 16 == 0,
                "xtb_moe_permute: pointers must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  if (T == 0) {
    if (tokens_per_expert) XTB_CUDA(cudaMemsetAsync(tokens_per_expert, 0, sizeof(int64_t) * E, st));
    return XTB_OK;
  }
  PermuteWorkspace w = carve_permute_workspace(workspace, E);
  const int n_chunks = n_chunks_of(T);
  if (!prepared) {
    const int wpb = 8;
    const int blocks = max(1, min((n_chunks + wpb - 1) / wpb, sm_count() * 4));
    const size_t smem = (size_t)wpb * E * sizeof(int);
    permute_count_scan_kernel<<<blocks, wpb * 32, smem, st>>>(
        ids, T, K, E, n_chunks, w.counts, w.expert_start,
        reinterpret_cast<unsigned long long*>(tokens_per_expert), w.ticket);
    XTB_LAUNCH_OK();
  }
  {
    const size_t smem = (size_t)(kChunkTokens + kSubTokens) * K * sizeof(int);
    const int n_sub = (T + kSubTokens - 1) / kSubTokens;
    const int row_vec = (int)(row_bytes / 16);
    // rows through shared memory with the bulk-copy engine; rows too long for kSubTokens staged rows (bf16 at K = 2:
    // H >= 12784) through registers
    const size_t smem_bulk = (size_t)kSubTokens * row_bytes + kSubTokens * sizeof(uint64_t) + smem;
    if (smem_bulk <= 200 * 1024) {
      static bool attr = false;
      if (!attr) {
        XTB_CUDA(cudaFuncSetAttribute(permute_scatter_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr = true;
      }
      XTB_CUDA(launch_pdl(permute_scatter_bulk_kernel, dim3(n_sub), dim3(128), smem_bulk, st, static_cast<const uint8_t*>(x), ids, T, K, E, (uint32_t)row_bytes,
                                                                  w.counts, w.expert_start, static_cast<uint8_t*>(permuted),
                                                                  row_id_map, sorted_indices));
    } else {
      XTB_CUDA(launch_pdl(permute_scatter_kernel, dim3(n_sub), dim3(128), smem, st, static_cast<const uint4*>(x), ids, T, K, E, row_vec,
                                                                w.counts, w.expert_start,
                                                                static_cast<uint4*>(permuted), row_id_map,
                                                                sorted_indices));
    }
    XTB_LAUNCH_OK();
  }
  return XTB_OK;
}

extern "C" int xtb_moe_permute(const void* x, const int32_t* ids, int T, int K, int E, int64_t row_bytes,
                               void* permuted, int32_t* row_id_map, int64_t* sorted_indices,
                               int64_t* tokens_per_expert, void* workspace, xtb_stream_t stream) {
  return permute_impl(x, ids, T, K, E, row_bytes, permuted, row_id_map, sorted_indices, tokens_per_expert,
                      workspace, stream, false);
}

extern "C" int xtb_moe_permute_prepared(const void* x, const int32_t* ids, int T, int K, int E, int64_t row_bytes,
                                        void* permuted, int32_t* row_id_map, int64_t* sorted_indices,
                                        const void* prepared_workspace, xtb_stream_t stream) {
  return permute_impl(x, ids, T, K, E, row_bytes, permuted, row_id_map, sorted_indices, nullptr,
                      const_cast<void*>(prepared_workspace), stream, true);
}

// xtb_moe_combine and xtb_moe_unpermute; `entry` names the one that was called in the refusal messages
static int combine_impl(const char* entry, const void* y_bf16, const int32_t* row_id_map, const float* probs,
                        const void* residual_bf16, float hidden_factor, int T, int K, int H, void* out_bf16,
                        xtb_stream_t stream) {
  XTB_CHECK_ARG(y_bf16 && row_id_map && out_bf16, "%s: null pointer", entry);
  XTB_CHECK_ARG(T >= 0 && K > 0 && H > 0 && H % 8 == 0, "%s: bad T=%d K=%d H=%d (H%%8==0)", entry, T, K, H);
  XTB_ENSURE_CTX(y_bf16);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  const int row_vec = H / 8;
  const int blocks = (T + 7) / 8;
  const auto* y = static_cast<const uint4*>(y_bf16);
  const auto* res = static_cast<const uint4*>(residual_bf16);
  auto* out = static_cast<uint4*>(out_bf16);
#define XTB_UNPERMUTE(KT) XTB_CUDA(launch_pdl(unpermute_kernel<KT>, dim3(blocks), dim3(256), 0, st, y, row_id_map, probs, T, K, row_vec, out, res, hidden_factor))
  switch (K) {
    case 1: XTB_UNPERMUTE(1); break;
    case 2: XTB_UNPERMUTE(2); break;
    case 4: XTB_UNPERMUTE(4); break;
    case 6: XTB_UNPERMUTE(6); break;
    case 8: XTB_UNPERMUTE(8); break;
    default: XTB_UNPERMUTE(0); break;
  }
#undef XTB_UNPERMUTE
  XTB_LAUNCH_OK();
  return XTB_OK;
}

extern "C" int xtb_moe_combine(const void* y_bf16, const int32_t* row_id_map, const float* probs,
                               const void* residual_bf16, float hidden_factor, int T, int K, int H, void* out_bf16,
                               xtb_stream_t stream) {
  return combine_impl("xtb_moe_combine", y_bf16, row_id_map, probs, residual_bf16, hidden_factor, T, K, H, out_bf16,
                      stream);
}

extern "C" int xtb_moe_unpermute(const void* y_bf16, const int32_t* row_id_map, const float* probs, int T, int K,
                                 int H, void* out_bf16, xtb_stream_t stream) {
  return combine_impl("xtb_moe_unpermute", y_bf16, row_id_map, probs, nullptr, 1.0f, T, K, H, out_bf16, stream);
}

extern "C" int xtb_moe_unpermute_bwd(const void* grad_out_bf16, const void* y_fwd_bf16, const int32_t* row_id_map,
                                     const float* probs, int T, int K, int H, void* act_grad_bf16,
                                     float* prob_grad, xtb_stream_t stream) {
  XTB_CHECK_ARG(grad_out_bf16 && row_id_map && act_grad_bf16, "xtb_moe_unpermute_bwd: null pointer");
  XTB_CHECK_ARG(!prob_grad || y_fwd_bf16, "xtb_moe_unpermute_bwd: prob_grad needs y_fwd");
  XTB_CHECK_ARG(T >= 0 && K > 0 && H > 0 && H % 8 == 0, "xtb_moe_unpermute_bwd: bad shape");
  XTB_ENSURE_CTX(grad_out_bf16);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  XTB_CUDA(launch_pdl(unpermute_bwd_kernel, dim3((T + 7) / 8), dim3(256), 0, st, static_cast<const uint4*>(grad_out_bf16),
                                                    static_cast<const uint4*>(y_fwd_bf16), row_id_map, probs, T, K,
                                                    H / 8, static_cast<uint4*>(act_grad_bf16), prob_grad));
  XTB_LAUNCH_OK();
  return XTB_OK;
}

extern "C" int xtb_swiglu(const void* h_bf16, void* out_bf16, int64_t M, int I, xtb_stream_t stream) {
  XTB_CHECK_ARG(h_bf16 && out_bf16, "xtb_swiglu: null pointer");
  XTB_CHECK_ARG(M >= 0 && I > 0 && I % 8 == 0, "xtb_swiglu: bad M=%lld I=%d (I%%8==0)", (long long)M, I);
  XTB_CHECK_ARG((reinterpret_cast<uintptr_t>(h_bf16) | reinterpret_cast<uintptr_t>(out_bf16)) % 16 == 0,
                "xtb_swiglu: pointers must be 16-byte aligned");
  XTB_ENSURE_CTX(h_bf16);
  if (M == 0) return XTB_OK;
  const int64_t n = M * (I / 8);
  swiglu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(static_cast<const uint4*>(h_bf16),
                                                                           static_cast<uint4*>(out_bf16), M, I / 8);
  XTB_LAUNCH_OK();
  return XTB_OK;
}

extern "C" int xtb_swiglu_bwd(const void* grad_out_bf16, const void* h_bf16, void* grad_h_bf16, int64_t M, int I,
                              xtb_stream_t stream) {
  XTB_CHECK_ARG(grad_out_bf16 && h_bf16 && grad_h_bf16, "xtb_swiglu_bwd: null pointer");
  XTB_CHECK_ARG(M >= 0 && I > 0 && I % 8 == 0, "xtb_swiglu_bwd: bad shape");
  XTB_CHECK_ARG((reinterpret_cast<uintptr_t>(grad_out_bf16) | reinterpret_cast<uintptr_t>(h_bf16) |
                 reinterpret_cast<uintptr_t>(grad_h_bf16)) % 16 == 0,
                "xtb_swiglu_bwd: pointers must be 16-byte aligned");
  const int64_t n = M * (I / 8);
  const int I8 = I / 8;
  // floor(i / I8) == umulhi(i, ceil(2^32 / I8)) as long as i * I8 < 2^32; i < kSwRows * I8 inside a block
  XTB_CHECK_ARG((int64_t)kSwRows * I8 * I8 < (1ll << 32), "xtb_swiglu_bwd: I=%d too wide", I);
  XTB_ENSURE_CTX(h_bf16);
  if (M == 0) return XTB_OK;
  const uint32_t inv_I8 = (uint32_t)(((1ull << 32) + I8 - 1) / I8);
  (void)n;
  XTB_CUDA(launch_pdl(swiglu_bwd_kernel, dim3((unsigned)((M + kSwRows - 1) / kSwRows)), dim3(256), 0, as_stream(stream), 
      static_cast<const uint4*>(grad_out_bf16), static_cast<const uint4*>(h_bf16), static_cast<uint4*>(grad_h_bf16),
      M, I8, inv_I8));
  XTB_LAUNCH_OK();
  return XTB_OK;
}
