// a1 (MoEGate.forward, moe_decoder_layer.py:120-141) on the tensor cores, fused with the greedy router and the dispatch
// bucketing into one launch (xtb_gate_route_dispatch: the default of the fused layer for E <= 8; fused against two calls
// has not been measured on H100).  tests/test_gpu_router_edges.py pins its logits against float64 and its routing and
// bucketing bit for bit against the router run on those logits; the fragment mapping is modelled lane by lane on CPU
// (tests/test_gate_mma_mapping_cpu.py).
//
// logits[T,E] = float(x[T,H]) @ float(w[E,H])^T for E <= 8.  The CUDA-core kernel (route.cu) is bound by shared-
// memory bandwidth (every FMA needs a W operand from smem) and by a chain of dependent x loads; here
//   * the fp32 gate weight is split ONCE per CTA into three bf16 planes hi+mid+lo (24 mantissa bits: the split is
//     exact up to the last fp32 ulp), kept in shared memory in B-fragment order, and
//   * x (bf16, exact) streams from global memory straight into A fragments of mma.sync.m16n8k16 (bf16 x bf16
//     products are exact in fp32; fp32 accumulation),
// so per 32 columns a warp issues 2 x LDG.128, 3 x LDS.128 (conflict free) and 6 HMMAs for 16 tokens.
// This is HBM/L2-streaming work, not GEMM-shaped work: mma.sync (not wgmma) is the right tool — N = 8.
//
// K ordering trick: inside a 32-column block, lane (g = lane/4, t = lane%4) owns columns t*8 .. t*8+7 of rows g and
// g+8.  MMA step s in {0,1} takes the lane's elements 4s..4s+3 as logical k = {2t, 2t+1, 2t+8, 2t+9}.  A and B use the
// same (bijective) column permutation, so the dot product is unchanged, every lane's 16 bytes are one contiguous
// LDG.128, and a B fragment is simply 8 consecutive bf16 of one expert's row.
#pragma once
#include "common.cuh"
#include "dispatch_scan.cuh"
#include "greedy_router.cuh"

namespace xtb {

__device__ __forceinline__ void mma_bf16_16x8x16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                 uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Splits the fp32 gate weight [E,H] (E <= 8, rows >= E are zero) into three bf16 planes in B-fragment order:
// s_planes[(p * H/32 + step) * 32 + lane] = 8 consecutive bf16 of plane p, expert lane/4, columns step*32 + (lane%4)*8.
__device__ __forceinline__ void fill_gate_planes(uint4* s_planes, const float* __restrict__ w, int H, int E) {
  const int n_steps = H / 32;
  constexpr int FB = 4;  // fragment slots whose weight loads are in flight together (the loop is a chain of L2 round trips otherwise)
  for (int idx0 = threadIdx.x; idx0 < n_steps * 32; idx0 += blockDim.x * FB) {
    float4 wa[FB], wb[FB];
#pragma unroll
    for (int f = 0; f < FB; ++f) {
      const int idx = idx0 + f * blockDim.x;
      const int ln = idx & 31, step = idx >> 5;
      const int g = ln >> 2, t = ln & 3;
      wa[f] = wb[f] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < n_steps * 32 && g < E) {
        // the lane's 8 consecutive weights as two 16-byte loads (one 32-byte sector, fully used)
        const float4* src = reinterpret_cast<const float4*>(w + (size_t)g * H + step * 32 + t * 8);
        wa[f] = __ldg(src);
        wb[f] = __ldg(src + 1);
      }
    }
#pragma unroll
    for (int f = 0; f < FB; ++f) {
      const int idx = idx0 + f * blockDim.x;
      if (idx >= n_steps * 32) break;
      const int ln = idx & 31, step = idx >> 5;
      uint32_t hi[4], mid[4], lo[4];
      const float wv[8] = {wa[f].x, wa[f].y, wa[f].z, wa[f].w, wb[f].x, wb[f].y, wb[f].z, wb[f].w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[2], r[2];
        uint32_t ph[2], pm[2], pl[2];
#pragma unroll
        for (int z = 0; z < 2; ++z) {
          v[z] = wv[2 * q + z];
          ph[z] = float_to_bf16_bits(v[z]);
          r[z] = v[z] - bf16_bits_to_float(ph[z]);   // exact
          pm[z] = float_to_bf16_bits(r[z]);
          r[z] = r[z] - bf16_bits_to_float(pm[z]);   // exact
          pl[z] = float_to_bf16_bits(r[z]);
        }
        hi[q] = ph[0] | (ph[1] << 16);
        mid[q] = pm[0] | (pm[1] << 16);
        lo[q] = pl[0] | (pl[1] << 16);
      }
      s_planes[(0 * n_steps + step) * 32 + ln] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
      s_planes[(1 * n_steps + step) * 32 + ln] = make_uint4(mid[0], mid[1], mid[2], mid[3]);
      s_planes[(2 * n_steps + step) * 32 + ln] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
  }
}

// Ask L2 for the rows of one token chunk ahead of their use (the plane fill / the previous chunk's epilogue run meanwhile).
__device__ __forceinline__ void prefetch_chunk_l2(const __nv_bfloat16* x, int row0, int n_rows, int T, int H) {
  const int lines_per_row = H / 64;  // 128-byte lines
  const int rows = min(n_rows, T - row0);
  for (int i = threadIdx.x; i < rows * lines_per_row; i += blockDim.x) {
    const int r = i / lines_per_row, l = i - r * lines_per_row;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(x + (size_t)(row0 + r) * H + l * 64));
  }
}

constexpr int kGateTokens = 32;   // tokens per CTA iteration (2 groups of 16)
constexpr int kGateKQ = 4;        // K split: warps (w >> 1) own H/4 columns each
constexpr int kGateBatch = 8;     // 32-column steps whose loads are in flight together

// ---- gate + greedy router + dispatch bucketing in ONE launch (xtb_gate_route_dispatch) -------------------------------
// The tensor-core gate produces the logits of one 32-token block = one histogram chunk of the dispatch
// (dispatch_scan.cuh: kChunkTokens == 32) in shared memory; routing those 32 tokens there (one thread per token, E <= 8:
// greedy_route_token<1, 8>) and counting the chunk's expert histogram with ballots removes the separate router launch
// (12.7 us per layer at C2, all latency) and the logits round trip.  The last block scans the chunk histograms exactly
// like the router kernel does.  REPLAY: the per-token step is greedy_replay_token on the rows of replay_ids (row stride
// replay_stride elements) instead of greedy_route_token (xtb_gate_route_replay_dispatch).
template <bool REPLAY = false>
__global__ void __launch_bounds__(256) gate_route_mma_kernel(
    const __nv_bfloat16* __restrict__ x, const float* __restrict__ w, float* __restrict__ logits, int T, int H, int E,
    int K, int scoring, int norm_topk, float scaling, float* __restrict__ router_weights,
    float* __restrict__ topk_weights, int64_t* __restrict__ topk_ids, int32_t* __restrict__ topk_ids_i32,
    unsigned long long* __restrict__ tokens_per_expert, int* __restrict__ chunk_counts, int* __restrict__ expert_start,
    unsigned* __restrict__ ticket, int n_chunks, const int64_t* __restrict__ replay_ids = nullptr,
    int64_t replay_stride = 0) {
  extern __shared__ uint4 s_planes[];
  __shared__ float s_red[2][kGateKQ][16][8];
  __shared__ float s_logit[kGateTokens][8];
  __shared__ int s_scratch[8];
  const int n_steps = H / 32;
  // The gate weight is a parameter: no kernel of this library that can precede this one in a stream writes it (the
  // programmatic launch only lets a predecessor that itself signals launch_dependents be overtaken, i.e. one of ours), so the
  // plane fill — a third of this kernel's time when it waited for its loads — runs while the predecessor drains.  x is the
  // predecessor's output: everything that touches it comes after the wait.
  pdl_trigger();
  fill_gate_planes(s_planes, w, H, E);
  pdl_wait();
  if ((int)blockIdx.x < n_chunks) prefetch_chunk_l2(x, blockIdx.x * kGateTokens, kGateTokens, T, H);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tg = warp & 1, kq = warp >> 1;
  const int g = lane >> 2, t = lane & 3;
  const int q_steps = n_steps / kGateKQ;
  const int step0 = kq * q_steps;

  for (int blk = blockIdx.x; blk < n_chunks; blk += gridDim.x) {
    if (blk + (int)gridDim.x < n_chunks) prefetch_chunk_l2(x, (blk + gridDim.x) * kGateTokens, kGateTokens, T, H);
    const int row0 = blk * kGateTokens + tg * 16;
    const int ra = min(row0 + g, T - 1), rb = min(row0 + g + 8, T - 1);
    const __nv_bfloat16* pa = x + (size_t)ra * H + (size_t)step0 * 32 + t * 8;
    const __nv_bfloat16* pb = x + (size_t)rb * H + (size_t)step0 * 32 + t * 8;
    float c[4] = {0.f, 0.f, 0.f, 0.f};
    for (int s0 = 0; s0 < q_steps; s0 += kGateBatch) {
      uint4 va[kGateBatch], vb[kGateBatch];
#pragma unroll
      for (int b = 0; b < kGateBatch; ++b) {
        if (s0 + b < q_steps) {
          va[b] = ld_stream_16(pa + (s0 + b) * 32);
          vb[b] = ld_stream_16(pb + (s0 + b) * 32);
        }
      }
#pragma unroll
      for (int b = 0; b < kGateBatch; ++b) {
        if (s0 + b < q_steps) {
          const int step = step0 + s0 + b;
#pragma unroll
          for (int p = 2; p >= 0; --p) {  // smallest plane first
            const uint4 wf = s_planes[(p * n_steps + step) * 32 + lane];
            mma_bf16_16x8x16(c, va[b].x, vb[b].x, va[b].y, vb[b].y, wf.x, wf.y);
            mma_bf16_16x8x16(c, va[b].z, vb[b].z, va[b].w, vb[b].w, wf.z, wf.w);
          }
        }
      }
    }
    // ---- reduce the K quarters; c0,c1 = (token g, experts 2t,2t+1), c2,c3 = (token g+8, same) -------------
    s_red[tg][kq][g][2 * t] = c[0];
    s_red[tg][kq][g][2 * t + 1] = c[1];
    s_red[tg][kq][g + 8][2 * t] = c[2];
    s_red[tg][kq][g + 8][2 * t + 1] = c[3];
    __syncthreads();
    {  // 256 threads = 32 tokens x 8 experts
      const int tok = threadIdx.x >> 3, e = threadIdx.x & 7;
      const int tgi = tok >> 4, r = tok & 15;
      float sacc = s_red[tgi][0][r][e];
#pragma unroll
      for (int q = 1; q < kGateKQ; ++q) sacc += s_red[tgi][q][r][e];
      s_logit[tok][e] = sacc;
      const int token = blk * kGateTokens + tok;
      if (token < T && e < E) logits[(size_t)token * E + e] = sacc;
    }
    __syncthreads();
    if (warp == 0) {  // one lane per token of the chunk
      const int token = blk * kGateTokens + lane;
      const bool active = token < T;
      float pr[8], wv[8];
      int se[8];
      if constexpr (REPLAY)
        greedy_replay_token<1, 8>(s_logit[lane], replay_ids + (int64_t)min(token, T - 1) * replay_stride, 0, E, K,
                                  scoring, norm_topk, scaling, pr, wv, se);
      else
        greedy_route_token<1, 8>(s_logit[lane], 0, E, K, scoring, norm_topk, scaling, pr, wv, se);
      if (active) {
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (j < E) router_weights[(size_t)token * E + j] = pr[j];
        for (int k = 0; k < K; ++k) {
          topk_weights[(size_t)token * K + k] = wv[k];
          topk_ids[(size_t)token * K + k] = (int64_t)se[k];
          topk_ids_i32[(size_t)token * K + k] = se[k];
        }
      }
      // chunk histogram by ballots (no atomics): counts[blk][e] = #(token, k) of this chunk routed to e
      int cnt_mine = 0;  // lane e accumulates expert e
      for (int k = 0; k < K; ++k) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const unsigned b = __ballot_sync(0xffffffffu, active && se[k] == e);
          if (lane == e) cnt_mine += __popc(b);
        }
      }
      if (lane < E) chunk_counts[(size_t)blk * E + lane] = cnt_mine;
    }
    __syncthreads();
  }
  scan_counts_last_block(chunk_counts, expert_start, tokens_per_expert, ticket, n_chunks, E, s_scratch);
}

// Launches gate_route_mma_kernel<REPLAY>.  Each instantiation is made in its own translation unit (gate_mma.cu: routing,
// gate_route_replay.cu: replay): compiled next to the replay kernel, the routing kernel's code changes.
template <bool REPLAY>
int launch_gate_route_mma(const __nv_bfloat16* x, const float* w, float* logits, int T, int H, int E, int K, int scoring,
                          int norm, float scaling, float* rw, float* tw, int64_t* ids, int32_t* ids32, int64_t* tpe,
                          void* dispatch_ws, cudaStream_t st, const int64_t* replay_ids, int64_t replay_stride) {
  const size_t smem = (size_t)3 * (H / 32) * 32 * sizeof(uint4);
  if (E > 8 || K > 8 || H % 128 != 0 || smem > 200 * 1024) return -1;
  PermuteWorkspace pw = carve_permute_workspace(dispatch_ws, E);
  const int n_chunks = n_chunks_of(T);
  const int blocks = max(1, min(2 * sm_count(), n_chunks));
  XTB_LAUNCH(gate_route_mma_kernel<REPLAY>, dim3(blocks), dim3(256), smem, st, true, x, w, logits, T, H, E, K, scoring,
             norm, scaling, rw, tw, ids, ids32, reinterpret_cast<unsigned long long*>(tpe), pw.counts, pw.expert_start,
             pw.ticket, n_chunks, replay_ids, replay_stride);
  return XTB_OK;
}

}  // namespace xtb
