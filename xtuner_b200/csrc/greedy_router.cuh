// The greedy router's per-token arithmetic, forward, routing replay and backward.  The standalone router kernels
// (route.cu) and the fused gate + route (gate_mma.cuh) and router + gate backward (route.cu) kernels all call these
// bodies, so they route and differentiate every token the same way, bit for bit.
//
// LPT lanes cooperate on one token; each lane holds VPL consecutive experts e = e0 + j (e0 = lane-in-group * VPL).
// With LPT = 1 every shuffle loop below is empty and one thread routes its token alone.
#pragma once
#include "common.cuh"

namespace xtb {

// (value desc, index asc) arg-max over the LPT lanes of a token.
template <int LPT>
__device__ __forceinline__ void group_argmax(float& best_v, int& best_e) {
#pragma unroll
  for (int o = LPT / 2; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best_v, o);
    const int oe = __shfl_xor_sync(0xffffffffu, best_e, o);
    if (ov > best_v || (ov == best_v && oe < best_e)) {
      best_v = ov;
      best_e = oe;
    }
  }
}

// Forward of one token from its logits row lg[0, E).  Softmax follows torch's CUDA formulation (max, exp(x-max), sum,
// divide) in fp32.  Top-k = K rounds of (value desc, index asc) arg-max over the group: the order torch.topk(sorted=True)
// returns on tie-free rows.  Out: p[j] = probability of expert e0 + j (what router_weights holds); sel_e[k], sel_w[k] for
// k < K <= 8 = the k-th expert and its weight (renormalised and scaled), the same on every lane of the group.
template <int LPT, int VPL>
__device__ __forceinline__ void greedy_route_token(const float* lg, int e0, int E, int K, int scoring, int norm_topk,
                                                   float scaling, float (&p)[VPL], float (&sel_w)[8], int (&sel_e)[8]) {
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    p[j] = (e0 + j < E) ? lg[e0 + j] : -INFINITY;
    m = fmaxf(m, p[j]);
  }
  if (scoring == XTB_SCORE_SOFTMAX) {
#pragma unroll
    for (int o = LPT / 2; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      p[j] = (e0 + j < E) ? expf(p[j] - m) : 0.f;
      s += p[j];
    }
#pragma unroll
    for (int o = LPT / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
#pragma unroll
    for (int j = 0; j < VPL; ++j) p[j] = p[j] / s;
  } else {
#pragma unroll
    for (int j = 0; j < VPL; ++j) p[j] = (e0 + j < E) ? 1.f / (1.f + expf(-p[j])) : -INFINITY;
  }

  unsigned taken = 0;  // bit j set: p[j] already selected
  unsigned used = 0;   // bit e set: expert e < 32 already selected (the same on every lane of the group)
  float sum = 0.f;
  for (int k = 0; k < K; ++k) {
    float bv = -INFINITY;
    int be = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      if (!((taken >> j) & 1u) && e0 + j < E && (p[j] > bv)) {
        bv = p[j];
        be = e0 + j;
      }
    }
    group_argmax<LPT>(bv, be);
    if (be < 0 || be >= E) {  // only reachable with NaN rows: the lowest index not selected yet, which is at most
                              // k < K <= min(E, 8) and so tracked by `used`.
      be = __ffs(~used) - 1;
      bv = 0.f;
    }
    if (be >= e0 && be < e0 + VPL) taken |= 1u << (be - e0);
    if (be < 32) used |= 1u << be;
    sel_w[k] = bv;
    sel_e[k] = be;
    sum += bv;
  }
  // unrolled: as a loop over k < K this read-modify-write of the stack arrays makes ptxas spill in <32, 8>
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k < K) {
      float wv = sel_w[k];
      if (norm_topk) wv = wv / sum;
      if (scaling != 1.0f) wv = wv * scaling;
      sel_w[k] = wv;
    }
  }
}

// Routing replay (greedy.py:74-78, `routing_weights.gather(dim=1, index=rollout_routed_experts)`): the experts are the
// K given ids ids[0, K) instead of a top-k.  The scores are greedy_route_token's own code with K = 0 (no selection), so
// they are the same bits as routing; each weight is gathered across the group with the reduction greedy_route_token_bwd
// uses (the one lane holding the expert contributes p, the others 0), then the weights are summed in k order and
// renormalised and scaled as in greedy_route_token.  The ids come from outside the program (rollout workers), so they
// are checked, never trusted: an id outside [0, E) becomes expert 0 in sel_e and makes every weight of the token NaN.
// Duplicate ids are gathered twice, as gather does.  Out: as greedy_route_token.
template <int LPT, int VPL>
__device__ __forceinline__ void greedy_replay_token(const float* lg, const int64_t* __restrict__ ids, int e0, int E,
                                                    int K, int scoring, int norm_topk, float scaling, float (&p)[VPL],
                                                    float (&sel_w)[8], int (&sel_e)[8]) {
  greedy_route_token<LPT, VPL>(lg, e0, E, 0, scoring, norm_topk, scaling, p, sel_w, sel_e);
  float sum = 0.f;
  bool bad = false;
  // unrolled, so that sel_w / sel_e stay in registers
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k < K) {
      const int64_t raw = ids[k];
      const bool ok = raw >= 0 && raw < E;
      const int id = ok ? (int)raw : 0;
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < VPL; ++j)
        if (e0 + j == id) v = p[j];
#pragma unroll
      for (int o = LPT / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      bad |= !ok;
      sel_w[k] = v;
      sel_e[k] = id;
      sum += v;
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k < K) {
      float wv = sel_w[k];
      if (norm_topk) wv = wv / sum;
      if (scaling != 1.0f) wv = wv * scaling;
      sel_w[k] = bad ? __int_as_float(0x7fffffff) : wv;  // NaN
    }
  }
}

// Backward of token tok through the router's three differentiable outputs (see xtb_router_greedy_bwd): the topk_weights
// route (selected sum s and dot = sum_k g_k * v_k / s), the router_weights route, the softmax or sigmoid Jacobian, plus
// g_direct.  Each gradient may be NULL (treated as 0).  Out: gl[j] = grad_logits of expert e0 + j, 0 for e0 + j >= E.
template <int LPT, int VPL>
__device__ __forceinline__ void greedy_route_token_bwd(const float* __restrict__ router_weights,
                                                       const float* __restrict__ topk_weights,
                                                       const int64_t* __restrict__ topk_ids,
                                                       const float* __restrict__ g_tw, const float* __restrict__ g_rw,
                                                       const float* __restrict__ g_direct, int tok, int e0, int E,
                                                       int K, int scoring, int norm_topk, float scaling,
                                                       float (&gl)[VPL]) {
  float p[VPL], gp[VPL];
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int e = e0 + j;
    p[j] = (e < E) ? router_weights[(size_t)tok * E + e] : 0.f;
    gp[j] = (e < E && g_rw) ? g_rw[(size_t)tok * E + e] : 0.f;
  }
  if (g_tw) {
    float s = 0.f, dot = 0.f;
    for (int k = 0; k < K; ++k) {
      const int id = (int)topk_ids[(size_t)tok * K + k];
      const float g = g_tw[(size_t)tok * K + k];
      const float twk = topk_weights[(size_t)tok * K + k];
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < VPL; ++j)
        if (e0 + j == id) v = p[j];
#pragma unroll
      for (int o = LPT / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      s += v;
      dot += g * (scaling != 1.0f ? twk / scaling : twk);  // twk/scaling == v_k/s when norm_topk
    }
    for (int k = 0; k < K; ++k) {
      const int id = (int)topk_ids[(size_t)tok * K + k];
      const float g = g_tw[(size_t)tok * K + k];
      const float gv = norm_topk ? scaling * (g - dot) / s : scaling * g;
#pragma unroll
      for (int j = 0; j < VPL; ++j)
        if (e0 + j == id) gp[j] += gv;
    }
  }
  if (scoring == XTB_SCORE_SOFTMAX) {
    float d = 0.f;
#pragma unroll
    for (int j = 0; j < VPL; ++j) d = fmaf(gp[j], p[j], d);
#pragma unroll
    for (int o = LPT / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
#pragma unroll
    for (int j = 0; j < VPL; ++j) gl[j] = p[j] * (gp[j] - d);
  } else {
#pragma unroll
    for (int j = 0; j < VPL; ++j) gl[j] = gp[j] * p[j] * (1.f - p[j]);
  }
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int e = e0 + j;
    gl[j] = (e < E) ? gl[j] + (g_direct ? g_direct[(size_t)tok * E + e] : 0.f) : 0.f;
  }
}

}  // namespace xtb
