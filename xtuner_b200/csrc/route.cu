// Router kernels (SURVEY.md §8a rows a1, a2, a2'): gate logits, greedy softmax/top-k router, no-aux
// (DeepSeek-V3 style) router, and their backward passes.  All fp32 CUDA-core math — these ops are
// HBM/latency bound ([T,E] tensors), not tensor-core work.
#include "common.cuh"
#include "dispatch_scan.cuh"
#include "greedy_router.cuh"

namespace xtb {

// =====================================================================================================
// a1  gate logits, small-E specialisation (E <= 16): one warp streams TW tokens at a time; lane owns an
// 8-wide slice of every 256-wide chunk of H.  x is read once (16 B per lane per token per chunk);
// the fp32 gate weight (E*H*4 bytes, e.g. 64 KiB) is re-read from L1/L2.
// =====================================================================================================
template <int E_MAX, int TW>
__global__ void __launch_bounds__(512, 1) gate_logits_small_kernel(const __nv_bfloat16* __restrict__ x,
                                                                   const float* __restrict__ w,
                                                                   const float* __restrict__ bias,
                                                                   float* __restrict__ logits, int T, int H, int E) {
  pdl_sync();
  // Persistent: one 16-warp CTA per SM; the fp32 gate weight [E,H] lives in shared memory for the CTA's
  // lifetime (short-scoreboard LDS instead of L1 round trips), x streams through registers with the next
  // chunk's loads in flight while the current one is multiplied.
  extern __shared__ float s_w[];  // [E][H]
  {
    const float4* src = reinterpret_cast<const float4*>(w);
    float4* dst = reinterpret_cast<float4*>(s_w);
    for (int i = threadIdx.x; i < E * H / 4; i += blockDim.x) dst[i] = __ldg(src + i);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int n_warps = (gridDim.x * blockDim.x) >> 5;
  for (int t0 = warp_global * TW; t0 < T; t0 += n_warps * TW) {
    float acc[TW][E_MAX];
#pragma unroll
    for (int i = 0; i < TW; ++i)
#pragma unroll
      for (int e = 0; e < E_MAX; ++e) acc[i][e] = 0.f;

    uint4 nxt[TW];
#pragma unroll
    for (int i = 0; i < TW; ++i) nxt[i] = ld_stream_16(x + (size_t)min(t0 + i, T - 1) * H + lane * 8);
    for (int h = lane * 8; h < H; h += 256) {
      uint4 cur[TW];
#pragma unroll
      for (int i = 0; i < TW; ++i) cur[i] = nxt[i];
      if (h + 256 < H) {
#pragma unroll
        for (int i = 0; i < TW; ++i) nxt[i] = ld_stream_16(x + (size_t)min(t0 + i, T - 1) * H + h + 256);
      }
      float xv[TW][8];
#pragma unroll
      for (int i = 0; i < TW; ++i) {
        unpack_bf16x2(cur[i].x, xv[i][0], xv[i][1]);
        unpack_bf16x2(cur[i].y, xv[i][2], xv[i][3]);
        unpack_bf16x2(cur[i].z, xv[i][4], xv[i][5]);
        unpack_bf16x2(cur[i].w, xv[i][6], xv[i][7]);
      }
#pragma unroll
      for (int e = 0; e < E_MAX; ++e) {
        if (e < E) {
          const float4 w0 = *reinterpret_cast<const float4*>(s_w + (size_t)e * H + h);
          const float4 w1 = *reinterpret_cast<const float4*>(s_w + (size_t)e * H + h + 4);
#pragma unroll
          for (int i = 0; i < TW; ++i) {
            float a = acc[i][e];
            a = fmaf(xv[i][0], w0.x, a);
            a = fmaf(xv[i][1], w0.y, a);
            a = fmaf(xv[i][2], w0.z, a);
            a = fmaf(xv[i][3], w0.w, a);
            a = fmaf(xv[i][4], w1.x, a);
            a = fmaf(xv[i][5], w1.y, a);
            a = fmaf(xv[i][6], w1.z, a);
            a = fmaf(xv[i][7], w1.w, a);
            acc[i][e] = a;
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < TW; ++i) {
#pragma unroll
      for (int e = 0; e < E_MAX; ++e) {
        const float s = warp_sum(acc[i][e]);
        if (lane == 0 && e < E && t0 + i < T) logits[(size_t)(t0 + i) * E + e] = s + (bias ? bias[e] : 0.f);
      }
    }
  }
}

// =====================================================================================================
// Generic strided fp32 GEMM on CUDA cores (64x64 tile, 4x4 micro-tile, K-chunk 16).  Used for the gate
// when E > 16 and for the gate backward in that regime.   C[m,n] = sum_k A(m,k) * B(k,n)
// A element type is bf16 or fp32, B is fp32; both addressed through (row, col) strides.
// =====================================================================================================
template <typename TA, typename TC>
__global__ void __launch_bounds__(256) sgemm_strided_kernel(const TA* __restrict__ A, int64_t sam, int64_t sak,
                                                            const float* __restrict__ B, int64_t sbk,
                                                            int64_t sbn, TC* __restrict__ C, int64_t scm,
                                                            int64_t scn, const float* __restrict__ bias_n, int M,
                                                            int N, int Kd) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < Kd; k0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      int kk, mm;
      if (sak == 1) { kk = i & 15; mm = i >> 4; } else { mm = i & 63; kk = i >> 6; }
      const int m = m0 + mm, k = k0 + kk;
      float v = 0.f;
      if (m < M && k < Kd) {
        if constexpr (sizeof(TA) == 2) v = __bfloat162float(A[m * sam + k * sak]);
        else v = (float)A[m * sam + k * sak];
      }
      As[kk][mm] = v;
    }
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      int kk, nn;
      if (sbk == 1) { kk = i & 15; nn = i >> 4; } else { nn = i & 63; kk = i >> 6; }
      const int n = n0 + nn, k = k0 + kk;
      Bs[kk][nn] = (n < N && k < Kd) ? B[k * sbk + n * sbn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      const float v = acc[i][j] + (bias_n ? bias_n[n] : 0.f);
      if constexpr (sizeof(TC) == 2) C[m * scm + n * scn] = __float2bfloat16_rn(v);
      else C[m * scm + n * scn] = v;
    }
  }
}

// =====================================================================================================
// a1 backward, small-E specialisation: block b owns a contiguous token range; thread j owns 8 columns
// of H per pass.  grad_x[t,h] = bf16(sum_e gl[t,e] * w[e,h]);  partial grad_w in registers, written to a
// [n_blocks, E, H] workspace and reduced (deterministically) by a second kernel.
// =====================================================================================================
// The next batch of U token rows is requested before the current one is consumed, so the block's loop is bound by
// max(load latency, FMA issue) instead of their sum.
// The streaming part is shared by the plain kernel (grad_logits read from global memory) and the variant that computes
// them in its prologue from the router's saved tensors (router_gate_bwd_kernel).
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

template <int E_MAX>
__device__ __forceinline__ void gate_bwd_main(const float* __restrict__ s_gl, const __nv_bfloat16* __restrict__ x,
                                              const float* __restrict__ w, float* __restrict__ partial_gw,
                                              __nv_bfloat16* __restrict__ gx, int H, int E, int t_begin, int t_end) {
  // 4 columns per thread (512 threads cover H = 2048): half the accumulators per thread of the 8-column version, so twice
  // the warps fit next to each other and hide the row loads.
  for (int h = threadIdx.x * 4; h < H; h += blockDim.x * 4) {
    float2 wr[E_MAX][2];
    float2 acc[E_MAX][2];
#pragma unroll
    for (int e = 0; e < E_MAX; ++e) {
      if (e < E) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(w + (size_t)e * H + h));
        wr[e][0] = make_float2(a.x, a.y);
        wr[e][1] = make_float2(a.z, a.w);
      } else {
        wr[e][0] = wr[e][1] = make_float2(0.f, 0.f);
      }
      acc[e][0] = acc[e][1] = make_float2(0.f, 0.f);
    }
    constexpr int U = 8;
    uint2 nxt[U];
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (t_begin + u < t_end) nxt[u] = ld_stream_8(x + (size_t)(t_begin + u) * H + h);
    for (int tb = t_begin; tb < t_end; tb += U) {
      uint2 raw[U];
#pragma unroll
      for (int u = 0; u < U; ++u) raw[u] = nxt[u];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (tb + U + u < t_end) nxt[u] = ld_stream_8(x + (size_t)(tb + U + u) * H + h);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = tb + u;
        if (t >= t_end) break;
        float2 xv0, xv1;
        unpack_bf16x2(raw[u].x, xv0.x, xv0.y);
        unpack_bf16x2(raw[u].y, xv1.x, xv1.y);
        float2 g0 = make_float2(0.f, 0.f), g1 = make_float2(0.f, 0.f);
        const float4* glt = reinterpret_cast<const float4*>(s_gl + (t - t_begin) * E_MAX);
#pragma unroll
        for (int e4 = 0; e4 < E_MAX / 4; ++e4) {
          const float4 q = glt[e4];
          const float ge[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int e = e4 * 4 + i;
            const float2 g2 = make_float2(ge[i], ge[i]);
            g0 = fma2(g2, wr[e][0], g0);
            g1 = fma2(g2, wr[e][1], g1);
            acc[e][0] = fma2(g2, xv0, acc[e][0]);
            acc[e][1] = fma2(g2, xv1, acc[e][1]);
          }
        }
        uint2 o;
        o.x = pack_bf16x2(g0.x, g0.y);
        o.y = pack_bf16x2(g1.x, g1.y);
        st_stream_8(gx + (size_t)t * H + h, o);
      }
    }
#pragma unroll
    for (int e = 0; e < E_MAX; ++e) {
      if (e < E) {
        float* dst = partial_gw + ((size_t)blockIdx.x * E + e) * H + h;
        *reinterpret_cast<float4*>(dst) = make_float4(acc[e][0].x, acc[e][0].y, acc[e][1].x, acc[e][1].y);
      }
    }
  }
}

template <int E_MAX>
__global__ void __launch_bounds__(E_MAX <= 8 ? 512 : 256) gate_bwd_small_kernel(const float* __restrict__ gl,
                                                             const __nv_bfloat16* __restrict__ x,
                                                             const float* __restrict__ w,
                                                             float* __restrict__ partial_gw,
                                                             __nv_bfloat16* __restrict__ gx, int T, int H, int E,
                                                             int tokens_per_block) {
  pdl_sync();
  const int t_begin = blockIdx.x * tokens_per_block;
  const int t_end = min(T, t_begin + tokens_per_block);
  extern __shared__ __align__(16) float s_gl[];  // [tokens_per_block][E_MAX]
  for (int i = threadIdx.x; i < tokens_per_block * E_MAX; i += blockDim.x) {
    const int tt = i / E_MAX, e = i % E_MAX;
    s_gl[i] = (t_begin + tt < t_end && e < E) ? gl[(size_t)(t_begin + tt) * E + e] : 0.f;
  }
  __syncthreads();
  gate_bwd_main<E_MAX>(s_gl, x, w, partial_gw, gx, H, E, t_begin, t_end);
}

// a2 backward + a1 backward in one launch (xtb_router_gate_bwd; E <= 8): the prologue computes this block's
// grad_logits rows from the router's saved outputs straight into the shared-memory tile the gate backward streams
// from, so the [T,E] grad_logits tensor and the 9.7 us router-backward launch disappear.
__global__ void __launch_bounds__(512) router_gate_bwd_kernel(
    const float* __restrict__ router_weights, const float* __restrict__ topk_weights,
    const int64_t* __restrict__ topk_ids, const float* __restrict__ g_tw, const float* __restrict__ g_rw,
    const float* __restrict__ g_direct, int K, int scoring, int norm_topk, float scaling,
    const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, float* __restrict__ partial_gw,
    __nv_bfloat16* __restrict__ gx, int T, int H, int E, int tokens_per_block) {
  pdl_sync();
  const int t_begin = blockIdx.x * tokens_per_block;
  const int t_end = min(T, t_begin + tokens_per_block);
  extern __shared__ __align__(16) float s_gl[];  // [tokens_per_block][8]
  for (int tt = threadIdx.x; tt < tokens_per_block; tt += blockDim.x) {
    const int tok = t_begin + tt;
    float gl[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (tok < t_end)
      greedy_route_token_bwd<1, 8>(router_weights, topk_weights, topk_ids, g_tw, g_rw, g_direct, tok, 0, E, K, scoring,
                                   norm_topk, scaling, gl);
#pragma unroll
    for (int j = 0; j < 8; ++j) s_gl[tt * 8 + j] = gl[j];
  }
  __syncthreads();
  gate_bwd_main<8>(s_gl, x, w, partial_gw, gx, H, E, t_begin, t_end);
}

// column sums of grad_logits -> grad_bias (tiny)
__global__ void colsum_kernel(const float* __restrict__ gl, float* __restrict__ out, int T, int E) {
  const int e = blockIdx.x;
  float s = 0.f;
  for (int t = threadIdx.x; t < T; t += blockDim.x) s += gl[(size_t)t * E + e];
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) out[e] = v;
  }
}

// =====================================================================================================
// a2  greedy router.  LPT lanes cooperate on one token; each lane holds VPL consecutive experts
// (e = sub*VPL + j); the per-token arithmetic is greedy_route_token (greedy_router.cuh).  Histogram:
// warp-aggregated shared-memory counters, one global atomic per (block, expert).  REPLAY: the experts are the
// rows of replay_ids (row stride replay_stride elements) instead of a top-k (greedy_replay_token).
// =====================================================================================================
// (REPLAY asks for one resident block per SM: left to itself, ptxas gives <32, 8, true> 32 registers and a spill)
template <int LPT, int VPL, bool REPLAY = false>
__global__ void __launch_bounds__((LPT * 32 > 256) ? LPT * 32 : 256, REPLAY ? 1 : 0)
router_greedy_kernel(const float* __restrict__ logits, int T, int E, int K, int scoring, int norm_topk, float scaling,
                     float* __restrict__ router_weights, float* __restrict__ topk_weights,
                     int64_t* __restrict__ topk_ids, int32_t* __restrict__ topk_ids_i32,
                     unsigned long long* __restrict__ tokens_per_expert,
                     // optional: prepare the dispatch workspace (per-chunk histograms + scan) in this launch
                     int* __restrict__ chunk_counts, int* __restrict__ expert_start, unsigned* __restrict__ ticket,
                     int n_chunks, const int64_t* __restrict__ replay_ids = nullptr, int64_t replay_stride = 0) {
  pdl_sync();
  // blockDim.x / LPT tokens per block, always a multiple of kChunkTokens (= 32)
  extern __shared__ int s_hist[];  // [E] block histogram | [chunks_per_block][E] per-chunk histograms
  const int chunks_per_block = (blockDim.x / LPT) / kChunkTokens;
  int* s_chunk = s_hist + E;
  for (int i = threadIdx.x; i < E * (1 + (chunk_counts ? chunks_per_block : 0)); i += blockDim.x) s_hist[i] = 0;
  __syncthreads();

  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int token = gtid / LPT;
  const int sub = threadIdx.x % LPT;
  const bool active = token < T;
  const int tok = active ? token : T - 1;  // keep all lanes in the shuffles
  const int e0 = sub * VPL;

  float p[VPL], sel_w[8];
  int sel_e[8];
  if constexpr (REPLAY)
    greedy_replay_token<LPT, VPL>(logits + (size_t)tok * E, replay_ids + tok * replay_stride, e0, E, K, scoring,
                                  norm_topk, scaling, p, sel_w, sel_e);
  else
    greedy_route_token<LPT, VPL>(logits + (size_t)tok * E, e0, E, K, scoring, norm_topk, scaling, p, sel_w, sel_e);
  if (active) {
#pragma unroll
    for (int j = 0; j < VPL; ++j)
      if (e0 + j < E) router_weights[(size_t)token * E + e0 + j] = p[j];
  }
  if (active && sub == 0) {
    for (int k = 0; k < K; ++k) {
      topk_weights[(size_t)token * K + k] = sel_w[k];
      topk_ids[(size_t)token * K + k] = (int64_t)sel_e[k];
      if (topk_ids_i32) topk_ids_i32[(size_t)token * K + k] = sel_e[k];
      if (chunk_counts) atomicAdd(&s_chunk[((threadIdx.x / LPT) / kChunkTokens) * E + sel_e[k]], 1);
      else atomicAdd(&s_hist[sel_e[k]], 1);
    }
  }
  __syncthreads();
  if (chunk_counts == nullptr) {
    for (int i = threadIdx.x; i < E; i += blockDim.x)
      if (s_hist[i]) atomicAdd(&tokens_per_expert[i], (unsigned long long)s_hist[i]);
    return;
  }
  const int chunk0 = blockIdx.x * chunks_per_block;
  for (int i = threadIdx.x; i < chunks_per_block * E; i += blockDim.x) {
    const int c = chunk0 + i / E;
    if (c < n_chunks) chunk_counts[(size_t)c * E + (i % E)] = s_chunk[i];
  }
  // the last block scans the histograms; tokens_per_expert falls out of the same scan (no atomics)
  scan_counts_last_block(chunk_counts, expert_start, tokens_per_expert, ticket, n_chunks, E, s_hist);
}

// backward of the greedy router (see header for the formula); same lane mapping as the forward.
template <int LPT, int VPL>
__global__ void __launch_bounds__(256) router_greedy_bwd_kernel(
    const float* __restrict__ router_weights, const float* __restrict__ topk_weights,
    const int64_t* __restrict__ topk_ids, const float* __restrict__ g_tw, const float* __restrict__ g_rw,
    const float* __restrict__ g_direct, int T, int E, int K, int scoring, int norm_topk, float scaling,
    float* __restrict__ grad_logits) {
  pdl_sync();
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int token = gtid / LPT;
  const int sub = threadIdx.x % LPT;
  const bool active = token < T;
  const int tok = active ? token : T - 1;
  const int e0 = sub * VPL;

  float gl[VPL];
  greedy_route_token_bwd<LPT, VPL>(router_weights, topk_weights, topk_ids, g_tw, g_rw, g_direct, tok, e0, E, K, scoring,
                                   norm_topk, scaling, gl);
  if (active) {
#pragma unroll
    for (int j = 0; j < VPL; ++j)
      if (e0 + j < E) grad_logits[(size_t)token * E + e0 + j] = gl[j];
  }
}

// =====================================================================================================
// a2' no-aux router: the forward is one warp per token, lane holds VPL = E/32 consecutive experts; the backward
// takes the XTB_ROUTER_DISPATCH lane mapping.
// =====================================================================================================
// Which of a token's experts the no-aux router's group mask keeps, computed from the choice scores ch = s + b; the
// forward and the backward both call it.  A group's score is its exact largest plus its exact second largest choice
// score, and topk_group rounds of (score desc, group index asc) over the groups not kept yet pick topk_group distinct
// groups; both are independent of how the experts are spread over lanes, so every lane mapping keeps the same groups.
// A group whose score is -inf (fewer than two of its scores above -inf) is still picked, lowest index first, once no
// group above -inf is left; only a NaN group score (+inf and -inf in one group: an infinite bias) is never picked.
// LPT lanes hold VPL consecutive experts each; groups of gs = E / n_group experts (a power of two) either lie whole
// inside one lane (gs <= VPL) or span gs / VPL neighbouring lanes.  The router weight of a kept expert may be exactly 0
// (s + b == 0), so router_weights cannot tell kept from masked experts.
template <int LPT, int VPL>
__device__ __forceinline__ void noaux_kept_experts(const float (&ch)[VPL], int e0, int E, int n_group, int topk_group,
                                                   bool (&keep)[VPL]) {
  const int gs = E / n_group;
  if constexpr (LPT == 32) {
    // One warp per token: VPL = E / 32 (the only 32-lane geometry the host accepts with a group mask) divides gs, so
    // the lane lies inside one group g, whose first lane holds its score: one candidate per lane, and the same rounds
    // as the slot loop below.
    float a = -INFINITY, b = -INFINITY;  // a >= b
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      const float v = ch[j];
      if (v > a) { b = a; a = v; } else if (v > b) { b = v; }
    }
    for (int o = 1; o < gs / VPL; o <<= 1) {
      const float oa = __shfl_xor_sync(0xffffffffu, a, o);
      const float ob = __shfl_xor_sync(0xffffffffu, b, o);
      const float na = fmaxf(a, oa);
      const float nb = fmaxf(fminf(a, oa), fmaxf(b, ob));
      a = na;
      b = nb;
    }
    const float gv = a + b;
    const int g = e0 / gs;
    const bool cand = (e0 % gs) == 0;
    unsigned kept = 0;
    for (int r = 0; r < topk_group; ++r) {
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      if (cand && !((kept >> g) & 1u) && gv >= bv) {  // not NaN: the slot loop's test against the initial (-inf, max)
        bv = gv;
        bi = g;
      }
      group_argmax<32>(bv, bi);
      if (bi < n_group) kept |= 1u << bi;
    }
#pragma unroll
    for (int j = 0; j < VPL; ++j) keep[j] = (kept >> g) & 1u;
    return;
  }
  // gv[j]: score of the group whose last local expert is j (candidate slots); others -inf and not candidates
  float gv[VPL];
  bool cand[VPL];
  float a = -INFINITY, b = -INFINITY;  // a >= b: top two of the current group
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const float v = ch[j];
    if (v > a) { b = a; a = v; } else if (v > b) { b = v; }
    const bool last = gs <= VPL && ((j + 1) % gs == 0);
    gv[j] = last ? a + b : -INFINITY;
    cand[j] = last;
    if (last) a = b = -INFINITY;
  }
  if (gs > VPL) {  // merge the top-2 pairs of the gs / VPL lanes of the group; its first lane holds the candidate
    for (int o = 1; o < gs / VPL; o <<= 1) {
        const float oa = __shfl_xor_sync(0xffffffffu, a, o);
        const float ob = __shfl_xor_sync(0xffffffffu, b, o);
        const float na = fmaxf(a, oa);
        const float nb = fmaxf(fminf(a, oa), fmaxf(b, ob));
        a = na;
        b = nb;
    }
    gv[VPL - 1] = a + b;
    cand[VPL - 1] = (e0 % gs) == 0;
  }
  unsigned kept = 0;  // bit g: group g kept (n_group <= 32); the same on every lane of the token
  for (int r = 0; r < topk_group; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      const int gi = (e0 + j) / gs;
      if (cand[j] && !((kept >> gi) & 1u) && (gv[j] > bv || (gv[j] == bv && gi < bi))) {
        bv = gv[j];
        bi = gi;
      }
    }
    group_argmax<LPT>(bv, bi);
    if (bi < n_group) kept |= 1u << bi;
  }
#pragma unroll
  for (int j = 0; j < VPL; ++j) keep[j] = (kept >> ((e0 + j) / gs)) & 1u;
}

// Forward.  The group mask is noaux_kept_experts<32, VPL>.  REPLAY (noaux_router.py:114-121): router_weights as
// routing — they do not depend on the ids — and the topk weights gathered from the unbiased scores at the rows of
// replay_ids (row stride replay_stride elements) in place of the top-k, which the reference computes and discards.  An
// id outside [0, E) becomes expert 0 and makes every topk weight of its token NaN.
template <int VPL, bool REPLAY = false>
__global__ void __launch_bounds__(256) router_noaux_kernel(const float* __restrict__ logits,
                                                           const float* __restrict__ bias, int T, int E, int K,
                                                           int n_group, int topk_group, int norm_topk,
                                                           float scaling, float* __restrict__ router_weights,
                                                           float* __restrict__ topk_weights,
                                                           int64_t* __restrict__ topk_ids,
                                                           int32_t* __restrict__ topk_ids_i32,
                                                           float* __restrict__ tokens_per_expert,
                                                           const int64_t* __restrict__ replay_ids,
                                                           int64_t replay_stride) {
  pdl_sync();
  extern __shared__ int s_hist[];
  for (int i = threadIdx.x; i < E; i += blockDim.x) s_hist[i] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int token = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const bool active = token < T;
  const int tok = active ? token : T - 1;
  const int e0 = lane * VPL;

  float sc[VPL], ch[VPL];
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const float x = logits[(size_t)tok * E + e0 + j];
    sc[j] = 1.f / (1.f + expf(-x));
    ch[j] = sc[j] + bias[e0 + j];
  }
  if (n_group != topk_group) {
    bool keep[VPL];
    noaux_kept_experts<32, VPL>(ch, e0, E, n_group, topk_group, keep);
#pragma unroll
    for (int j = 0; j < VPL; ++j)
      if (!keep[j]) ch[j] = 0.0f;  // masked_fill(~mask, 0.0)
  }
  // router_weights = choice / row-sum
  float rs = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j) rs += ch[j];
  rs = warp_sum(rs);
  if (active) {
#pragma unroll
    for (int j = 0; j < VPL; ++j) router_weights[(size_t)token * E + e0 + j] = ch[j] / rs;
  }
  // top-k over the (masked) choice scores, weights from the unbiased scores.  K <= 32: lane k keeps pick k.
  float my_w = 0.f;
  int my_e = 0;
  float sum = 0.f;
  bool bad = false;
  if constexpr (REPLAY) {
    const int64_t* ids = replay_ids + tok * replay_stride;
    for (int k = 0; k < K; ++k) {
      const int64_t raw = ids[k];
      const bool ok = raw >= 0 && raw < E;
      const int id = ok ? (int)raw : 0;
      float bw = 0.f;
#pragma unroll
      for (int j = 0; j < VPL; ++j)
        if (e0 + j == id) bw = sc[j];
      bw = warp_sum(bw);  // one lane holds expert id; the others add 0
      bad |= !ok;
      if (lane == k) { my_w = bw; my_e = id; }
      sum += bw;
    }
  } else {
    unsigned taken = 0;  // bit j set: expert e0 + j already selected
    unsigned used = 0;   // bit e set: expert e < 32 already selected (the same on every lane)
    for (int k = 0; k < K; ++k) {
      float bv = -INFINITY, bw = 0.f;
      int be = 0x7fffffff;
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        if (!((taken >> j) & 1u) && ch[j] > bv) { bv = ch[j]; be = e0 + j; bw = sc[j]; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oe = __shfl_xor_sync(0xffffffffu, be, o);
        const float ow = __shfl_xor_sync(0xffffffffu, bw, o);
        if (ov > bv || (ov == bv && oe < be)) { bv = ov; be = oe; bw = ow; }
      }
      if (be < 0 || be >= E) {  // no score left that compares (NaN or -inf): the lowest index not selected yet, with
                                // weight 0; that index is at most k < K <= 32, so `used` tracks it.
        be = __ffs(~used) - 1;
        bw = 0.f;
      }
      if (be >= e0 && be < e0 + VPL) taken |= 1u << (be - e0);
      if (be < 32) used |= 1u << be;
      if (lane == k) { my_w = bw; my_e = be; }
      sum += bw;
    }
  }
  if (active && lane < K) {
    const float denom = sum + 1e-20f;
    float wv = my_w;
    if (K > 1 && norm_topk) wv = wv / denom;
    wv = wv * scaling;
    if (REPLAY && bad) wv = __int_as_float(0x7fffffff);  // NaN
    topk_weights[(size_t)token * K + lane] = wv;
    topk_ids[(size_t)token * K + lane] = (int64_t)my_e;
    if (topk_ids_i32) topk_ids_i32[(size_t)token * K + lane] = my_e;
    atomicAdd(&s_hist[my_e], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < E; i += blockDim.x)
    if (s_hist[i]) atomicAdd(&tokens_per_expert[i], (float)s_hist[i]);  // exact: integer counts < 2^24
}

// backward of the no-aux router (closed form: oracle/moe_oracle.py noaux_router_bwd).  LPT lanes per token, each
// holding VPL consecutive experts.  The group mask is recomputed from logits and bias (noaux_kept_experts).
template <int LPT, int VPL>
__global__ void __launch_bounds__(256) router_noaux_bwd_kernel(
    const float* __restrict__ logits, const float* __restrict__ bias, const float* __restrict__ router_weights,
    const float* __restrict__ topk_weights, const int64_t* __restrict__ topk_ids, const float* __restrict__ g_tw,
    const float* __restrict__ g_rw, int T, int E, int K, int n_group, int topk_group, int norm_topk, float scaling,
    float* __restrict__ grad_logits) {
  pdl_sync();
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int token = gtid / LPT;
  const int sub = threadIdx.x % LPT;
  const bool active = token < T;
  const int tok = active ? token : T - 1;
  const int e0 = sub * VPL;

  float sg[VPL], ds[VPL];
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int e = e0 + j;
    const float x = (e < E) ? logits[(size_t)tok * E + e] : 0.f;
    sg[j] = 1.f / (1.f + expf(-x));
    ds[j] = 0.f;
  }
  if (g_rw) {
    // r = c / S with c = mask * (s + b):  dc_j = mask_j * (g_j - sum_i g_i r_i) / S
    float S = 0.f, dot = 0.f, g[VPL];
    bool keep[VPL];
    if (n_group != topk_group) {
      float ch[VPL];
#pragma unroll
      for (int j = 0; j < VPL; ++j) ch[j] = (e0 + j < E) ? sg[j] + bias[e0 + j] : -INFINITY;
      noaux_kept_experts<LPT, VPL>(ch, e0, E, n_group, topk_group, keep);
    } else {
#pragma unroll
      for (int j = 0; j < VPL; ++j) keep[j] = true;
    }
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      const int e = e0 + j;
      const float r = (e < E) ? router_weights[(size_t)tok * E + e] : 0.f;
      g[j] = (e < E) ? g_rw[(size_t)tok * E + e] : 0.f;
      keep[j] = keep[j] && (e < E);
      if (keep[j]) S += sg[j] + bias[e];
      dot = fmaf(g[j], r, dot);
    }
#pragma unroll
    for (int o = LPT / 2; o > 0; o >>= 1) {
      S += __shfl_xor_sync(0xffffffffu, S, o);
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
    }
#pragma unroll
    for (int j = 0; j < VPL; ++j)
      if (keep[j]) ds[j] = (g[j] - dot) / S;
  }
  if (g_tw) {
    // w_k = scaling * s_k / D, D = sum_k s_k + 1e-20 (K > 1 and norm) else w_k = scaling * s_k
    const bool norm = (K > 1) && norm_topk;
    float D = 0.f, gw = 0.f;
    if (norm) {
      for (int k = 0; k < K; ++k) {
        const int id = (int)topk_ids[(size_t)tok * K + k];
        const float x = logits[(size_t)tok * E + id];
        D += 1.f / (1.f + expf(-x));
        gw = fmaf(g_tw[(size_t)tok * K + k], topk_weights[(size_t)tok * K + k], gw);
      }
      D += 1e-20f;
    }
    for (int k = 0; k < K; ++k) {
      const int id = (int)topk_ids[(size_t)tok * K + k];
      if (id >= e0 && id < e0 + VPL) {
        const float gk = g_tw[(size_t)tok * K + k];
        const float v = norm ? (scaling * gk - gw) / D : scaling * gk;
#pragma unroll
        for (int j = 0; j < VPL; ++j)
          if (id == e0 + j) ds[j] += v;
      }
    }
  }
  if (active) {
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      const int e = e0 + j;
      if (e < E) grad_logits[(size_t)token * E + e] = ds[j] * sg[j] * (1.f - sg[j]);
    }
  }
}

}  // namespace xtb

// =====================================================================================================
// C-ABI
// =====================================================================================================
using namespace xtb;

extern "C" int xtb_gate_logits(const void* x_bf16, const float* w_f32, const float* bias_f32, float* logits, int T,
                               int H, int E, xtb_stream_t stream) {
  XTB_CHECK_ARG(w_f32 && (T == 0 || (x_bf16 && logits)), "xtb_gate_logits: null pointer");
  XTB_CHECK_ARG(T >= 0 && H > 0 && E > 0, "xtb_gate_logits: bad shape T=%d H=%d E=%d", T, H, E);
  if (T == 0) return XTB_OK;
  XTB_ENSURE_CTX(x_bf16);
  cudaStream_t st = as_stream(stream);
  const auto* x = static_cast<const __nv_bfloat16*>(x_bf16);
  const size_t w_smem = (size_t)E * H * sizeof(float);
  if (E <= 16 && H % 256 == 0 && w_smem <= 200 * 1024) {
    const int blocks = min(sm_count(), (T + 63) / 64);
    auto* kernel = E <= 8 ? gate_logits_small_kernel<8, 4> : gate_logits_small_kernel<16, 2>;
    XTB_LAUNCH(kernel, dim3(blocks), dim3(512), w_smem, st, true, x, w_f32, bias_f32, logits, T, H, E);
  } else {
    dim3 grid((E + 63) / 64, (T + 63) / 64);
    // A = x [T,H] (sam=H, sak=1), B(k,n) = w[n,k] (sbk=1, sbn=H)
    XTB_LAUNCH(sgemm_strided_kernel<__nv_bfloat16, float>, grid, dim3(256), 0, st, false, x, H, 1, w_f32, 1, H, logits, E,
               1, bias_f32, T, E, H);
  }
  return XTB_OK;
}

// One block per SM while the block's grad_logits slice (tokens x 16 floats at most) stays under the 48 KB of dynamic shared
// memory a launch gets without opting in; more blocks beyond that (the partial sums scale with the block count).
static int gate_bwd_blocks(int T) {
  constexpr int kMaxTokensPerBlock = 48 * 1024 / (16 * (int)sizeof(float));
  const int by_sm = max(1, min(sm_count(), (T + 15) / 16));
  return max(by_sm, (T + kMaxTokensPerBlock - 1) / kMaxTokensPerBlock);
}

extern "C" size_t xtb_gate_logits_bwd_workspace_bytes(int T, int H, int E) {
  if (E <= 16 && H % 8 == 0) return (size_t)gate_bwd_blocks(T) * E * H * sizeof(float);
  return 16;
}

extern "C" int xtb_gate_logits_bwd(const float* grad_logits, const void* x_bf16, const float* w_f32, float* grad_w,
                                   void* grad_x_bf16, float* grad_bias, int T, int H, int E, void* workspace,
                                   xtb_stream_t stream) {
  XTB_CHECK_ARG(w_f32 && grad_w && (T == 0 || (grad_logits && x_bf16 && grad_x_bf16)), "xtb_gate_logits_bwd: null pointer");
  XTB_CHECK_ARG(T >= 0 && H > 0 && E > 0, "xtb_gate_logits_bwd: bad shape");
  XTB_ENSURE_CTX(w_f32);
  cudaStream_t st = as_stream(stream);
  if (T == 0) {  // an empty micro-batch: the sums over no tokens
    XTB_CUDA(cudaMemsetAsync(grad_w, 0, (size_t)E * H * sizeof(float), st));
    if (grad_bias) XTB_CUDA(cudaMemsetAsync(grad_bias, 0, (size_t)E * sizeof(float), st));
    return XTB_OK;
  }
  const auto* x = static_cast<const __nv_bfloat16*>(x_bf16);
  auto* gx = static_cast<__nv_bfloat16*>(grad_x_bf16);
  if (E <= 16 && H % 8 == 0) {
    XTB_CHECK_ARG(workspace, "xtb_gate_logits_bwd: workspace required");
    const int blocks = gate_bwd_blocks(T);
    const int tpb = (T + blocks - 1) / blocks;
    float* partial = static_cast<float*>(workspace);
    const int cap = E <= 8 ? 512 : 256;  // threads: one per 4 columns, bounded by the kernels' launch bounds
    const int threads = (H / 4 >= cap) ? cap : ((H / 4 + 31) / 32) * 32;
    const int ew = E <= 8 ? 8 : 16;  // logits per token the kernel holds
    XTB_LAUNCH(ew == 8 ? gate_bwd_small_kernel<8> : gate_bwd_small_kernel<16>, dim3(blocks), dim3(threads),
               (size_t)tpb * ew * sizeof(float), st, true, grad_logits, x, w_f32, partial, gx, T, H, E, tpb);
    const int64_t n = (int64_t)E * H;
    XTB_LAUNCH(reduce_partial_rows_kernel<8>, dim3((unsigned)((n + 31) / 32)), dim3(256), 0, st, true,
               (const float*)partial, grad_w, blocks, n);
  } else {
    // grad_x[T,H] = gl[T,E] @ w[E,H]:  A = gl (sam=E, sak=1), B(k=e, n=h) = w[e,h] (sbk=H, sbn=1)
    dim3 g1((H + 63) / 64, (T + 63) / 64);
    XTB_LAUNCH(sgemm_strided_kernel<float, __nv_bfloat16>, g1, dim3(256), 0, st, false, grad_logits, E, 1, w_f32, H, 1, gx,
               H, 1, nullptr, T, H, E);
    // grad_w[e,h] = sum_t gl[t,e] x[t,h]:  A(m=h, k=t) = x[t,h] (sam=1, sak=H), B(k=t, n=e) = gl[t,e]
    // (sbk=E, sbn=1), C(m=h, n=e) -> grad_w[e*H + h] (scm=1, scn=H)
    dim3 g2((E + 63) / 64, (H + 63) / 64);
    XTB_LAUNCH(sgemm_strided_kernel<__nv_bfloat16, float>, g2, dim3(256), 0, st, false, x, 1, H, grad_logits, E, 1, grad_w,
               1, H, nullptr, H, E, T);
  }
  if (grad_bias) {
    XTB_LAUNCH(colsum_kernel, dim3(E), dim3(256), 0, st, false, grad_logits, grad_bias, T, E);
  }
  return XTB_OK;
}

template <int LPT, int VPL>
static int launch_router_greedy(const float* logits, int T, int E, int K, int scoring, int norm, float scaling,
                                float* rw, float* tw, int64_t* ids, int32_t* ids32, int64_t* tpe, void* dispatch_ws,
                                const int64_t* replay_ids, int64_t replay_stride, cudaStream_t st) {
  constexpr int kThreads = (LPT * 32 > 256) ? LPT * 32 : 256;
  const int tokens_per_block = kThreads / LPT;
  const int blocks = (T + tokens_per_block - 1) / tokens_per_block;
  int* counts = nullptr;
  int* estart = nullptr;
  unsigned* ticket = nullptr;
  size_t smem = (size_t)E * sizeof(int);
  if (dispatch_ws) {
    PermuteWorkspace w = carve_permute_workspace(dispatch_ws, E);
    counts = w.counts;
    estart = w.expert_start;
    ticket = w.ticket;
    smem += (size_t)(tokens_per_block / kChunkTokens) * E * sizeof(int);
  } else {
    XTB_CUDA(cudaMemsetAsync(tpe, 0, sizeof(int64_t) * E, st));
  }
  XTB_LAUNCH(replay_ids ? router_greedy_kernel<LPT, VPL, true> : router_greedy_kernel<LPT, VPL>, dim3(blocks),
             dim3(kThreads), smem, st, true, logits, T, E, K, scoring, norm, scaling, rw, tw, ids, ids32,
             reinterpret_cast<unsigned long long*>(tpe), counts, estart, ticket, n_chunks_of(T), replay_ids,
             replay_stride);
  return XTB_OK;
}

template <int LPT, int VPL>
static int launch_router_greedy_bwd(const float* rw, const float* tw, const int64_t* ids, const float* g_tw,
                                    const float* g_rw, const float* g_direct, int T, int E, int K, int scoring,
                                    int norm, float scaling, float* gl, cudaStream_t st) {
  const int tokens_per_block = 256 / LPT;
  const int blocks = (T + tokens_per_block - 1) / tokens_per_block;
  XTB_LAUNCH(router_greedy_bwd_kernel<LPT, VPL>, dim3(blocks), dim3(256), 0, st, true, rw, tw, ids, g_tw, g_rw, g_direct,
             T, E, K, scoring, norm, scaling, gl);
  return XTB_OK;
}

#define XTB_ROUTER_DISPATCH(FN, ...)                                      \
  if (E <= 8) return FN<1, 8>(__VA_ARGS__);                               \
  if (E <= 16) return FN<2, 8>(__VA_ARGS__);                              \
  if (E <= 32) return FN<4, 8>(__VA_ARGS__);                              \
  if (E <= 64) return FN<8, 8>(__VA_ARGS__);                              \
  if (E <= 128) return FN<16, 8>(__VA_ARGS__);                            \
  if (E <= 256) return FN<32, 8>(__VA_ARGS__);                            \
  if (E <= 512) return FN<32, 16>(__VA_ARGS__);                           \
  return fail(XTB_ERR_INVALID, "router: E=%d > 512 not supported", E);

template <int LPT, int VPL>
static int launch_router_noaux_bwd(const float* logits, const float* bias, const float* rw, const float* tw,
                                   const int64_t* ids, const float* g_tw, const float* g_rw, int T, int E, int K,
                                   int n_group, int topk_group, int norm, float scaling, float* gl, cudaStream_t st) {
  const int tokens_per_block = 256 / LPT;
  const int blocks = (T + tokens_per_block - 1) / tokens_per_block;
  XTB_LAUNCH(router_noaux_bwd_kernel<LPT, VPL>, dim3(blocks), dim3(256), 0, st, true, logits, bias, rw, tw, ids,
             g_tw, g_rw, T, E, K, n_group, topk_group, norm, scaling, gl);
  return XTB_OK;
}

static int router_greedy_impl(const float* logits, int T, int E, int K, int scoring, int norm_topk_prob, float scaling,
                              float* router_weights, float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32,
                              int64_t* tokens_per_expert, void* dispatch_ws, xtb_stream_t stream,
                              const int64_t* replay_ids = nullptr, int64_t replay_stride = 0) {
  XTB_CHECK_ARG(logits && router_weights && topk_weights && topk_ids && tokens_per_expert,
                "xtb_router_greedy: null pointer");
  XTB_CHECK_ARG(T >= 0 && E > 0 && K > 0 && K <= E && K <= 8, "xtb_router_greedy: bad shape T=%d E=%d K=%d (K<=8)", T,
                E, K);
  XTB_ENSURE_CTX(logits);
  cudaStream_t st = as_stream(stream);
  if (T == 0) {
    XTB_CUDA(cudaMemsetAsync(tokens_per_expert, 0, sizeof(int64_t) * E, st));
    return XTB_OK;
  }
  XTB_ROUTER_DISPATCH(launch_router_greedy, logits, T, E, K, scoring, norm_topk_prob, scaling, router_weights,
                      topk_weights, topk_ids, topk_ids_i32, tokens_per_expert, dispatch_ws, replay_ids, replay_stride,
                      st)
}

extern "C" int xtb_router_greedy(const float* logits, int T, int E, int K, int scoring, int norm_topk_prob,
                                 float scaling, float* router_weights, float* topk_weights, int64_t* topk_ids,
                                 int32_t* topk_ids_i32, int64_t* tokens_per_expert, xtb_stream_t stream) {
  return router_greedy_impl(logits, T, E, K, scoring, norm_topk_prob, scaling, router_weights, topk_weights, topk_ids,
                            topk_ids_i32, tokens_per_expert, nullptr, stream);
}

extern "C" int xtb_router_greedy_dispatch(const float* logits, int T, int E, int K, int scoring, int norm_topk_prob,
                                          float scaling, float* router_weights, float* topk_weights,
                                          int64_t* topk_ids, int32_t* topk_ids_i32, int64_t* tokens_per_expert,
                                          void* dispatch_workspace, xtb_stream_t stream) {
  XTB_CHECK_ARG(dispatch_workspace && topk_ids_i32, "xtb_router_greedy_dispatch: workspace and topk_ids_i32 required");
  return router_greedy_impl(logits, T, E, K, scoring, norm_topk_prob, scaling, router_weights, topk_weights, topk_ids,
                            topk_ids_i32, tokens_per_expert, dispatch_workspace, stream);
}

extern "C" int xtb_router_greedy_replay(const float* logits, const int64_t* replay_ids, int64_t replay_row_stride,
                                        int T, int E, int K, int scoring, int norm_topk_prob, float scaling,
                                        float* router_weights, float* topk_weights, int64_t* topk_ids,
                                        int32_t* topk_ids_i32, int64_t* tokens_per_expert, void* dispatch_workspace,
                                        xtb_stream_t stream) {
  XTB_CHECK_ARG(tokens_per_expert && (T == 0 || replay_ids), "xtb_router_greedy_replay: null pointer");
  XTB_CHECK_ARG(T >= 0 && E > 0 && K > 0 && replay_row_stride >= K,
                "xtb_router_greedy_replay: bad shape T=%d E=%d K=%d replay_row_stride=%lld", T, E, K,
                (long long)replay_row_stride);
  if (T == 0) {  // an empty micro-batch: no token arrays to address, only the counts to clear
    XTB_ENSURE_CTX(tokens_per_expert);
    XTB_CUDA(cudaMemsetAsync(tokens_per_expert, 0, sizeof(int64_t) * E, as_stream(stream)));
    return XTB_OK;
  }
  XTB_CHECK_ARG(!dispatch_workspace || topk_ids_i32, "xtb_router_greedy_replay: the workspace needs topk_ids_i32");
  return router_greedy_impl(logits, T, E, K, scoring, norm_topk_prob, scaling, router_weights, topk_weights, topk_ids,
                            topk_ids_i32, tokens_per_expert, dispatch_workspace, stream, replay_ids, replay_row_stride);
}

extern "C" int xtb_router_greedy_bwd(const float* router_weights, const float* topk_weights,
                                     const int64_t* topk_ids, const float* grad_topk_weights,
                                     const float* grad_router_weights, const float* grad_logits_direct, int T,
                                     int E, int K, int scoring, int norm_topk_prob, float scaling,
                                     float* grad_logits, xtb_stream_t stream) {
  XTB_CHECK_ARG(router_weights && topk_weights && topk_ids && grad_logits, "xtb_router_greedy_bwd: null pointer");
  XTB_CHECK_ARG(T >= 0 && E > 0 && K > 0 && K <= E, "xtb_router_greedy_bwd: bad shape");
  XTB_ENSURE_CTX(router_weights);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  XTB_ROUTER_DISPATCH(launch_router_greedy_bwd, router_weights, topk_weights, topk_ids, grad_topk_weights,
                      grad_router_weights, grad_logits_direct, T, E, K, scoring, norm_topk_prob, scaling,
                      grad_logits, st)
}

// The no-aux router's group geometry, for the forward and the backward alike.  The forward holds E / 32 experts per
// lane, so a group lies whole inside one lane or spans a power-of-two number of lanes; a group mask scores each group
// by its top two experts, so its groups need at least two.
static int check_noaux_groups(const char* who, int E, int n_group, int topk_group) {
  XTB_CHECK_ARG(E % 32 == 0 && E <= 512, "%s: E=%d must be a multiple of 32 and <= 512", who, E);
  XTB_CHECK_ARG(n_group >= 1 && n_group <= 32 && E % n_group == 0 && topk_group >= 1 && topk_group <= n_group,
                "%s: bad n_group=%d / topk_group=%d for E=%d", who, n_group, topk_group, E);
  const int gs = E / n_group;
  XTB_CHECK_ARG((gs & (gs - 1)) == 0 && gs % (E / 32) == 0,
                "%s: group size %d must be a power of two and a multiple of E/32=%d", who, gs, E / 32);
  XTB_CHECK_ARG(n_group == topk_group || gs >= 2,
                "%s: a group mask (topk_group=%d < n_group=%d) needs at least 2 experts per group, got %d", who,
                topk_group, n_group, gs);
  return XTB_OK;
}

static int router_noaux_impl(const float* logits, const float* e_score_correction_bias, int T, int E, int K,
                             int n_group, int topk_group, int norm_topk_prob, float scaling, float* router_weights,
                             float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32,
                             float* tokens_per_expert_f32, const int64_t* replay_ids, int64_t replay_stride,
                             xtb_stream_t stream) {
  XTB_CHECK_ARG(logits && e_score_correction_bias && router_weights && topk_weights && topk_ids &&
                    tokens_per_expert_f32,
                "xtb_router_noaux: null pointer");
  XTB_CHECK_ARG(T >= 0 && E > 0 && K > 0 && K <= 32 && K <= E, "xtb_router_noaux: bad T/E/K");
  if (const int rc = check_noaux_groups("xtb_router_noaux", E, n_group, topk_group)) return rc;
  XTB_ENSURE_CTX(logits);
  cudaStream_t st = as_stream(stream);
  XTB_CUDA(cudaMemsetAsync(tokens_per_expert_f32, 0, sizeof(float) * E, st));
  if (T == 0) return XTB_OK;
  const int blocks = (T + 7) / 8;
  const bool replay = replay_ids != nullptr;
  decltype(&router_noaux_kernel<1>) kernel;
  switch (E / 32) {
    case 1: kernel = replay ? router_noaux_kernel<1, true> : router_noaux_kernel<1>; break;
    case 2: kernel = replay ? router_noaux_kernel<2, true> : router_noaux_kernel<2>; break;
    case 4: kernel = replay ? router_noaux_kernel<4, true> : router_noaux_kernel<4>; break;
    case 8: kernel = replay ? router_noaux_kernel<8, true> : router_noaux_kernel<8>; break;
    case 16: kernel = replay ? router_noaux_kernel<16, true> : router_noaux_kernel<16>; break;
    default: return fail(XTB_ERR_INVALID, "xtb_router_noaux: E/32=%d unsupported (1,2,4,8,16)", E / 32);
  }
  XTB_LAUNCH(kernel, dim3(blocks), dim3(256), E * sizeof(int), st, true, logits, e_score_correction_bias, T, E, K, n_group,
             topk_group, norm_topk_prob, scaling, router_weights, topk_weights, topk_ids, topk_ids_i32,
             tokens_per_expert_f32, replay_ids, replay_stride);
  return XTB_OK;
}

extern "C" int xtb_router_noaux(const float* logits, const float* e_score_correction_bias, int T, int E, int K,
                                int n_group, int topk_group, int norm_topk_prob, float scaling,
                                float* router_weights, float* topk_weights, int64_t* topk_ids,
                                int32_t* topk_ids_i32, float* tokens_per_expert_f32, xtb_stream_t stream) {
  return router_noaux_impl(logits, e_score_correction_bias, T, E, K, n_group, topk_group, norm_topk_prob, scaling,
                           router_weights, topk_weights, topk_ids, topk_ids_i32, tokens_per_expert_f32, nullptr, 0,
                           stream);
}

extern "C" int xtb_router_noaux_replay(const float* logits, const float* e_score_correction_bias,
                                       const int64_t* replay_ids, int64_t replay_row_stride, int T, int E, int K,
                                       int n_group, int topk_group, int norm_topk_prob, float scaling,
                                       float* router_weights, float* topk_weights, int64_t* topk_ids,
                                       int32_t* topk_ids_i32, float* tokens_per_expert_f32, xtb_stream_t stream) {
  XTB_CHECK_ARG(tokens_per_expert_f32 && (T == 0 || replay_ids), "xtb_router_noaux_replay: null pointer");
  XTB_CHECK_ARG(T >= 0 && E > 0 && K > 0 && replay_row_stride >= K,
                "xtb_router_noaux_replay: bad shape T=%d E=%d K=%d replay_row_stride=%lld", T, E, K,
                (long long)replay_row_stride);
  if (T == 0) {  // an empty micro-batch: no token arrays to address, only the counts to clear
    XTB_ENSURE_CTX(tokens_per_expert_f32);
    XTB_CUDA(cudaMemsetAsync(tokens_per_expert_f32, 0, sizeof(float) * E, as_stream(stream)));
    return XTB_OK;
  }
  return router_noaux_impl(logits, e_score_correction_bias, T, E, K, n_group, topk_group, norm_topk_prob, scaling,
                           router_weights, topk_weights, topk_ids, topk_ids_i32, tokens_per_expert_f32, replay_ids,
                           replay_row_stride, stream);
}

extern "C" int xtb_router_noaux_bwd(const float* logits, const float* e_score_correction_bias,
                                    const float* router_weights, const float* topk_weights, const int64_t* topk_ids,
                                    const float* grad_topk_weights, const float* grad_router_weights, int T, int E,
                                    int K, int group_spec, int norm_topk_prob, float scaling, float* grad_logits,
                                    xtb_stream_t stream) {
  XTB_CHECK_ARG(logits && e_score_correction_bias && router_weights && topk_weights && topk_ids && grad_logits,
                "xtb_router_noaux_bwd: null pointer");
  XTB_CHECK_ARG(T >= 0 && E > 0 && K > 0 && K <= E, "xtb_router_noaux_bwd: bad shape T=%d E=%d K=%d", T, E, K);
  // group_spec = XTB_NOAUX_GROUP_SPEC(n_group, topk_group); 0: no group mask
  const int n_group = group_spec ? (group_spec & 0xFF) : 1;
  const int topk_group = group_spec ? (group_spec >> 8) : 1;
  if (group_spec) {  // a group mask, in the forward's geometry
    XTB_CHECK_ARG(topk_group < n_group, "xtb_router_noaux_bwd: group_spec %d is not a group mask (n_group=%d, "
                  "topk_group=%d)", group_spec, n_group, topk_group);
    if (const int rc = check_noaux_groups("xtb_router_noaux_bwd", E, n_group, topk_group)) return rc;
  }
  XTB_ENSURE_CTX(logits);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  XTB_ROUTER_DISPATCH(launch_router_noaux_bwd, logits, e_score_correction_bias, router_weights, topk_weights, topk_ids,
                      grad_topk_weights, grad_router_weights, T, E, K, n_group, topk_group, norm_topk_prob, scaling,
                      grad_logits, st)
}

extern "C" int xtb_router_gate_bwd(const float* router_weights, const float* topk_weights, const int64_t* topk_ids,
                                   const float* grad_topk_weights, const float* grad_router_weights,
                                   const float* grad_logits_direct, const void* x_bf16, const float* w_f32, float* grad_w,
                                   void* grad_x_bf16, int T, int H, int E, int K, int scoring, int norm_topk_prob,
                                   float scaling, void* workspace, xtb_stream_t stream) {
  XTB_CHECK_ARG(w_f32 && grad_w && (T == 0 || (router_weights && topk_weights && topk_ids && x_bf16 && grad_x_bf16 && workspace)),
                "xtb_router_gate_bwd: null pointer");
  XTB_CHECK_ARG(T >= 0 && H > 0 && E > 0 && K > 0 && K <= E, "xtb_router_gate_bwd: bad shape");
  if (T == 0) {  // an empty micro-batch: the sum over no tokens
    XTB_ENSURE_CTX(w_f32);
    XTB_CUDA(cudaMemsetAsync(grad_w, 0, (size_t)E * H * sizeof(float), as_stream(stream)));
    return XTB_OK;
  }
  XTB_CHECK_ARG(E <= 8 && H % 8 == 0,
                "xtb_router_gate_bwd: supports E <= 8 and H %% 8 == 0 (got E=%d H=%d); use xtb_router_greedy_bwd + "
                "xtb_gate_logits_bwd",
                E, H);
  XTB_ENSURE_CTX(x_bf16);
  cudaStream_t st = as_stream(stream);
  const int blocks = gate_bwd_blocks(T);
  const int tpb = (T + blocks - 1) / blocks;
  float* partial = static_cast<float*>(workspace);
  const int threads = (H / 4 >= 512) ? 512 : ((H / 4 + 31) / 32) * 32;
  const auto* x = static_cast<const __nv_bfloat16*>(x_bf16);
  auto* gx = static_cast<__nv_bfloat16*>(grad_x_bf16);
  const size_t smem = (size_t)tpb * 8 * sizeof(float);
  XTB_LAUNCH(router_gate_bwd_kernel, dim3(blocks), dim3(threads), smem, st, true, router_weights, topk_weights, topk_ids,
             grad_topk_weights, grad_router_weights, grad_logits_direct, K, scoring, norm_topk_prob, scaling, x, w_f32,
             partial, gx, T, H, E, tpb);
  const int64_t n = (int64_t)E * H;
  XTB_LAUNCH(reduce_partial_rows_kernel<8>, dim3((unsigned)((n + 31) / 32)), dim3(256), 0, st, true, (const float*)partial, grad_w,
             blocks, n);
  return XTB_OK;
}
