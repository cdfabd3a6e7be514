// Statistics behind the MoE auxiliary losses (AuxLossContext.accumulate, loss/aux_loss.py:84-151): the per-expert token
// counts (the torch.histc chain), the column sums of the router weights that every BalancingLossContext keeps
// (moe_loss.py:106-119), and the z-loss sum of squared row logsumexps (ZLossContext.accumulate, moe_loss.py:242-289).
// The reference runs these as a dozen eager kernels per layer over [N, E] fp32; here one kernel reads the weights, the
// logits and the ids once, and one elementwise kernel writes both input gradients.  Formulas and rounding points:
// include/xtuner_b200.h.
//
// Mapping (forward): a row of E values is held by L = min(32, pow2ceil(E)) lanes with J = ceil(E / L) columns each, so a
// warp covers 32 / L rows side by side.  A CTA owns a contiguous block of rows.  Each lane keeps the column sums of its J
// columns in registers; at the end the row groups of a warp are added by a fixed butterfly, the warps of the CTA in warp
// order, and the CTA writes one partial row [rw_sum (E) | z_sum (1)] plus one row of counts.  The last CTA to finish
// (ticket in the workspace, reset by that CTA) adds the partial rows in CTA order: no float atomics, identical bits run
// to run, and no memset between calls.
#include "common.cuh"

namespace xtb {

constexpr int kAuxThreads = 256;
constexpr int kAuxMaxE = 512;
constexpr int64_t kAuxElemsPerCta = 16384;  // [N, E] elements per CTA and operand (64 KB)

struct AuxWorkspace {
  unsigned* ticket;  // [1]        last-CTA-done counter, zero between calls
  float* part;       // [G][E + 1] per-CTA column sums of rw, then the CTA's sum of lse^2
  int* cnt;          // [G][E]     per-CTA expert counts
};

static size_t aux_align(size_t v) { return (v + 255) / 256 * 256; }

static int aux_max_blocks(int64_t N, int E) {
  const int64_t want = (N * E + kAuxElemsPerCta - 1) / kAuxElemsPerCta;
  return (int)max((int64_t)1, min((int64_t)sm_count() * 2, want));
}

static AuxWorkspace carve_aux_workspace(void* ws, int G, int E) {
  char* p = static_cast<char*>(ws);
  AuxWorkspace w;
  w.ticket = reinterpret_cast<unsigned*>(p);
  p += 256;
  w.part = reinterpret_cast<float*>(p);
  p += aux_align((size_t)G * (E + 1) * sizeof(float));
  w.cnt = reinterpret_cast<int*>(p);
  return w;
}

template <int L>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
template <int L>
__device__ __forceinline__ float group_max(float v) {
#pragma unroll
  for (int o = L / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// sum_b p[b * stride] for b < n, added in b order with 8 loads in flight
template <typename T, typename A>
__device__ __forceinline__ A ordered_sum(const T* p, int64_t stride, int n) {
  A s = 0;
  int b = 0;
  for (; b + 8 <= n; b += 8) {
    T v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = __ldcg(p + (int64_t)(b + u) * stride);
#pragma unroll
    for (int u = 0; u < 8; ++u) s += (A)v[u];
  }
  for (; b < n; ++b) s += (A)__ldcg(p + (int64_t)b * stride);
  return s;
}

template <int L, int J>
__global__ void __launch_bounds__(kAuxThreads) moe_aux_stats_kernel(const float* __restrict__ rw,
                                                                     const float* __restrict__ logits,
                                                                     const int64_t* __restrict__ ids, int64_t N, int E,
                                                                     int K, int64_t rows_per_cta, AuxWorkspace ws,
                                                                     int64_t* __restrict__ tokens_per_expert,
                                                                     float* __restrict__ rw_sum,
                                                                     float* __restrict__ z_sum, float* __restrict__ lse) {
  constexpr int RPW = 32 / L;                        // rows per warp and pass
  constexpr int RPP = RPW * (kAuxThreads / 32);      // rows per CTA and pass
  constexpr int U = J >= 4 ? 1 : 4 / J;              // passes in flight
  __shared__ float s_col[kAuxThreads / 32][L * J];
  __shared__ float s_z[kAuxThreads / 32];
  __shared__ int s_cnt[kAuxMaxE];
  __shared__ bool is_last;
  pdl_sync();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, c = lane % L;
  const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta, r1 = min(N, r0 + rows_per_cta);
  const bool do_rw = rw_sum != nullptr, do_z = z_sum != nullptr;
  for (int e = threadIdx.x; e < E; e += kAuxThreads) s_cnt[e] = 0;
  __syncthreads();

  // counts, with histc's edges: bin = id for 0 <= id < E, E - 1 for id == E, nothing otherwise
  {
    const int64_t i1 = r1 * K;
#pragma unroll 4
    for (int64_t i = r0 * K + threadIdx.x; i < i1; i += kAuxThreads) {
      const int64_t id = ids[i];
      if (id >= 0 && id <= E) atomicAdd(&s_cnt[id == E ? E - 1 : (int)id], 1);
    }
  }

  float acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = 0.f;
  float zacc = 0.f;
  // warp-uniform loop: every lane of a warp runs the same passes, dead rows are masked
  for (int64_t rb = r0 + warp * RPW; rb < r1; rb += (int64_t)U * RPP) {
    float v[U][J], x[U][J];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t r = rb + u * RPP + lane / L;
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const int col = c + j * L;
        const bool ok = r < r1 && col < E;
        v[u][j] = (do_rw && ok) ? __ldcs(rw + r * E + col) : 0.f;
        x[u][j] = (do_z && ok) ? __ldcs(logits + r * E + col) : -INFINITY;
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
#pragma unroll
      for (int j = 0; j < J; ++j) acc[j] += v[u][j];
      if (do_z) {
        float m = x[u][0];
#pragma unroll
        for (int j = 1; j < J; ++j) m = fmaxf(m, x[u][j]);
        m = group_max<L>(m);  // NaN is skipped here and reaches lse through the sum, as in torch.logsumexp
        if (fabsf(m) == INFINITY) m = 0.f;  // torch.logsumexp's masked_fill of an infinite max
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < J; ++j) s += expf(x[u][j] - m);
        const float l = logf(group_sum<L>(s)) + m;
        const int64_t r = rb + u * RPP + lane / L;
        if (c == 0 && r < r1) {
          lse[r] = l;
          zacc = fmaf(l, l, zacc);
        }
      }
    }
  }

  // CTA partials: the row groups of a warp by butterfly, then the warps in order
#pragma unroll
  for (int j = 0; j < J; ++j) {
#pragma unroll
    for (int o = L; o < 32; o <<= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    if (lane < L) s_col[warp][c + j * L] = acc[j];
  }
  zacc = warp_sum(zacc);
  if (lane == 0) s_z[warp] = zacc;
  __syncthreads();
  float* part = ws.part + (int64_t)blockIdx.x * (E + 1);
  for (int e = threadIdx.x; e <= E; e += kAuxThreads) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kAuxThreads / 32; ++w) s += e < E ? s_col[w][e] : s_z[w];
    part[e] = s;
  }
  int* cnt = ws.cnt + (int64_t)blockIdx.x * E;
  for (int e = threadIdx.x; e < E; e += kAuxThreads) cnt[e] = s_cnt[e];

  // the last CTA adds the partial rows in CTA order (fence + ticket as in dispatch_scan.cuh) and resets the ticket
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    is_last = atomicAdd(ws.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const int G = gridDim.x;
  for (int col = threadIdx.x; col < 2 * E + 1; col += kAuxThreads) {
    if (col < E) {
      if (do_rw) rw_sum[col] = ordered_sum<float, float>(ws.part + col, E + 1, G);
    } else if (col == E) {
      if (do_z) *z_sum = ordered_sum<float, float>(ws.part + E, E + 1, G);
    } else {
      const int e = col - E - 1;
      tokens_per_expert[e] = ordered_sum<int, int64_t>(ws.cnt + e, E, G);
    }
  }
  if (threadIdx.x == 0) *ws.ticket = 0u;
}

// g_rw[t, e] = g_rw_sum[e];  g_logits[t, e] = (g_z (2 lse_t)) exp(x_te - lse_t)
__global__ void __launch_bounds__(256) moe_aux_stats_bwd_kernel(const float* __restrict__ g_rw_sum,
                                                               const float* __restrict__ g_z,
                                                               const float* __restrict__ logits,
                                                               const float* __restrict__ lse, int64_t N, int E,
                                                               float* __restrict__ g_rw, float* __restrict__ g_logits) {
  pdl_sync();
  const float gz = g_logits ? *g_z : 0.f;
  const int64_t total = N * E, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t t = i / E;
    const int e = (int)(i - t * E);
    if (g_rw) __stcs(g_rw + i, __ldg(g_rw_sum + e));
    if (g_logits) {
      const float l = __ldg(lse + t);
      __stcs(g_logits + i, (gz * (2.f * l)) * expf(__ldcs(logits + i) - l));
    }
  }
}

}  // namespace xtb

using namespace xtb;

extern "C" size_t xtb_moe_aux_stats_workspace_bytes(int64_t N, int E) {
  if (N < 0 || E < 1) return 0;
  const int G = aux_max_blocks(N, E);
  return 256 + aux_align((size_t)G * (E + 1) * sizeof(float)) + (size_t)G * E * sizeof(int);
}

extern "C" int xtb_moe_aux_stats(const float* rw, const float* logits, const int64_t* ids, int64_t N, int E, int K,
                                 int64_t* tokens_per_expert, float* rw_sum, float* z_sum, float* lse, void* workspace,
                                 xtb_stream_t stream) {
  XTB_CHECK_ARG(tokens_per_expert && workspace, "xtb_moe_aux_stats: tokens_per_expert and workspace are required");
  XTB_CHECK_ARG(N >= 0 && E >= 1 && E <= kAuxMaxE && K >= 1, "xtb_moe_aux_stats: N=%lld E=%d K=%d (1 <= E <= %d, K >= 1)",
                (long long)N, E, K, kAuxMaxE);
  XTB_CHECK_ARG(N == 0 || ids, "xtb_moe_aux_stats: null ids");
  XTB_CHECK_ARG(N == 0 || !rw_sum || rw, "xtb_moe_aux_stats: rw_sum needs rw");
  XTB_CHECK_ARG(!z_sum || ((N == 0 || logits) && (N == 0 || lse)), "xtb_moe_aux_stats: z_sum needs logits and lse");
  XTB_ENSURE_CTX(tokens_per_expert);
  cudaStream_t st = as_stream(stream);
  const int G = aux_max_blocks(N, E);
  const int64_t rows = N ? (N + G - 1) / G : 1;
  const int grid = N ? (int)((N + rows - 1) / rows) : 1;
  const AuxWorkspace ws = carve_aux_workspace(workspace, G, E);
  auto* kernel = E <= 1     ? moe_aux_stats_kernel<1, 1>
                 : E <= 2   ? moe_aux_stats_kernel<2, 1>
                 : E <= 4   ? moe_aux_stats_kernel<4, 1>
                 : E <= 8   ? moe_aux_stats_kernel<8, 1>
                 : E <= 16  ? moe_aux_stats_kernel<16, 1>
                 : E <= 32  ? moe_aux_stats_kernel<32, 1>
                 : E <= 64  ? moe_aux_stats_kernel<32, 2>
                 : E <= 128 ? moe_aux_stats_kernel<32, 4>
                 : E <= 256 ? moe_aux_stats_kernel<32, 8>
                            : moe_aux_stats_kernel<32, 16>;
  XTB_LAUNCH(kernel, dim3(grid), dim3(kAuxThreads), 0, st, true, rw, logits, ids, N, E, K, rows, ws, tokens_per_expert,
             rw_sum, z_sum, lse);
  return XTB_OK;
}

extern "C" int xtb_moe_aux_stats_bwd(const float* g_rw_sum, const float* g_z, const float* logits, const float* lse,
                                     int64_t N, int E, float* g_rw, float* g_logits, xtb_stream_t stream) {
  XTB_CHECK_ARG(g_rw_sum || g_z, "xtb_moe_aux_stats_bwd: g_rw_sum or g_z is required");
  XTB_CHECK_ARG(N >= 0 && E >= 1 && E <= kAuxMaxE, "xtb_moe_aux_stats_bwd: N=%lld E=%d (1 <= E <= %d)", (long long)N, E,
                kAuxMaxE);
  XTB_CHECK_ARG(!g_rw || g_rw_sum, "xtb_moe_aux_stats_bwd: g_rw needs g_rw_sum");
  XTB_CHECK_ARG(!g_logits || (g_z && logits && lse), "xtb_moe_aux_stats_bwd: g_logits needs g_z, logits and lse");
  if (N == 0 || (!g_rw && !g_logits)) return XTB_OK;
  XTB_ENSURE_CTX(g_rw ? (const void*)g_rw : (const void*)g_logits);
  const int64_t total = N * E;
  const int blocks = (int)min((int64_t)sm_count() * 8, (total + 255) / 256);
  XTB_LAUNCH(moe_aux_stats_bwd_kernel, dim3(blocks), dim3(256), 0, as_stream(stream), true, g_rw_sum, g_z, logits,
             lse, N, E, g_rw, g_logits);
  return XTB_OK;
}
