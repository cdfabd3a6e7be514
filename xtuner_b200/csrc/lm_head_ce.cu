// lm_head projection fused with the cross-entropy loss (xtb_lm_head_ce, DESIGN.md §10), and the same projection split
// around the label log-probability for any per-token loss of it (xtb_lm_head_logprob / _bwd, DESIGN.md §13).
//
// xtb_lm_head_ce, one call, for T rows of hidden states h[T, H] against the head weight w[V, H]:
//   1. ce_set_rows_kernel   tokens_per_expert = {T} in the workspace: the one-group tile list of the GEMMs below
//   2. the NT grouped GEMM with the EPI_CE epilogue (group_gemm.cu): z = bf16(h . w^T) into the caller's [T, V] buffer, and
//      per row and vocab tile the pair (max, sum exp(z - max)) of the rounded values
//   3. ce_row_kernel        per row: logsumexp from the tile pairs in a fixed order, ce_t, and (need_grad) G over z in place
//   4. ce_loss_kernel       loss = sum_t ce_t * w_t in a fixed order (one CTA, no float atomics)
//   5. (need_grad) dh = G . w and dW = G^T . h on the existing NN / TN grouped-GEMM entries with one group
// xtb_lm_head_logprob runs 1 and 2, then logprob_row_kernel (logp_t and the row's (max, log sum) from the tile pairs and
// one logit); xtb_lm_head_logprob_bwd runs 1, logprob_grad_row_kernel (G over z in place from dL/dlogp_t) and 5.  Steps 3
// and the two logprob row kernels share row_max_sum and grad_row_in_place, so both paths round identically.
#include "common.cuh"

namespace xtb {

constexpr int kRowThreads = 256;
constexpr int kLossThreads = 1024;
constexpr size_t kWsHeader = 256;  // tokens_per_expert {T}, then the tile pairs

__global__ void ce_set_rows_kernel(int64_t* tokens_per_expert, int64_t T) {
  pdl_sync();
  *tokens_per_expert = T;
}

// Block-wide reductions in a fixed order: xor butterfly inside each warp (every lane ends with the same value), then the
// warps' results in warp order.  Ends with a barrier, so the block may reuse `red` and anything it read before.
template <int NT, bool MAX>
__device__ __forceinline__ float block_reduce(float v, float* red) {
  v = MAX ? warp_max(v) : warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int i = 1; i < NT / 32; ++i) r = MAX ? fmaxf(r, red[i]) : r + red[i];
  __syncthreads();
  return r;
}

// Row t's (max, sum exp(z - max)) over its tile pairs p[0..n_vt): the max, then the pairs' sums rescaled to it, each
// reduced in a fixed order.
template <int NT>
__device__ __forceinline__ float2 row_max_sum(const float2* __restrict__ p, int n_vt, float* red) {
  float m = __int_as_float(0xff800000);
  for (int i = threadIdx.x; i < n_vt; i += NT) m = fmaxf(m, p[i].x);
  m = block_reduce<NT, true>(m, red);
  float s = 0.f;
  for (int i = threadIdx.x; i < n_vt; i += NT) {
    const float2 q = p[i];
    s += q.y * expf(q.x - m);
  }
  s = block_reduce<NT, false>(s, red);
  return make_float2(m, s);
}

// G over row z[0..8*n16) in place: G_v = bf16(exp(lsm_v) * w - [v == lab] * w) with lsm_v = (z_v - m) - logsum, rounded
// in that order (multiply, then subtract; no contraction).
template <int NT>
__device__ __forceinline__ void grad_row_in_place(uint4* __restrict__ row, int n16, float m, float logsum, float w,
                                                  int64_t lab) {
  auto grad = [&](float zv, int64_t col) {
    const float g = __fmul_rn(expf(__fsub_rn(__fsub_rn(zv, m), logsum)), w);
    return col == lab ? __fsub_rn(g, w) : g;
  };
  constexpr int U = 4;  // 16-byte chunks in flight per thread
  for (int i0 = threadIdx.x; i0 < n16; i0 += U * NT) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * NT;
      if (i < n16) v[u] = row[i];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = i0 + u * NT;
      if (i >= n16) break;
      uint32_t* e = reinterpret_cast<uint32_t*>(&v[u]);
      const int64_t col = (int64_t)i * 8;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float lo, hi;
        unpack_bf16x2(e[k], lo, hi);
        e[k] = pack_bf16x2(grad(lo, col + 2 * k), grad(hi, col + 2 * k + 1));
      }
      row[i] = v[u];
    }
  }
}

// One CTA per row t.  With lsm_v = (z_v - max) - log(sum exp(z - max)) (torch's log_softmax in fp32):
//   ce_t = -lsm_label;  G_v = bf16(exp(lsm_v) * w_t - [v == label] * w_t)   (torch's log_softmax_backward of the
//   nll gradient -w_t at the label).  An ignored row has ce_t = 0 and G = 0; a label outside [0, V) that is not
//   ignore_index gives ce_t = NaN and a NaN row of G.
__global__ void __launch_bounds__(kRowThreads) ce_row_kernel(__nv_bfloat16* __restrict__ z, const float2* __restrict__ part,
                                                            int n_vt, const int64_t* __restrict__ labels,
                                                            int64_t ignore_index, const float* __restrict__ loss_weight,
                                                            int V, int need_grad, float* __restrict__ row_ce) {
  __shared__ float red[kRowThreads / 32];
  pdl_sync();
  const int64_t t = blockIdx.x;
  const int64_t lab = labels[t];
  uint4* row = reinterpret_cast<uint4*>(z + t * (int64_t)V);
  const int n16 = V / 8;  // 16-byte chunks of the row
  if (lab == ignore_index) {
    if (threadIdx.x == 0) row_ce[t] = 0.f;
    if (need_grad)
      for (int i = threadIdx.x; i < n16; i += kRowThreads) row[i] = make_uint4(0, 0, 0, 0);
    return;
  }
  const bool bad = lab < 0 || lab >= V;
  // z at the label, read before any thread overwrites the row (the reductions below end with barriers)
  const float z_lab = (threadIdx.x == 0 && !bad) ? __bfloat162float(z[t * (int64_t)V + lab]) : 0.f;

  const float2 ms = row_max_sum<kRowThreads>(part + t * (int64_t)n_vt, n_vt, red);
  const float m = ms.x;
  const float logsum = bad ? __int_as_float(0x7fc00000) : logf(ms.y);
  if (threadIdx.x == 0) row_ce[t] = -__fsub_rn(__fsub_rn(z_lab, m), logsum);
  if (!need_grad) return;
  grad_row_in_place<kRowThreads>(row, n16, m, logsum, loss_weight[t], lab);
}

// One CTA per row t, the forward of ce_row_kernel for the clipped label lab = max(label_t, 0), reading only the row's
// tile pairs and z[t, lab]:  logp_t = lsm_lab (so -logp_t is ce_row_kernel's ce_t for the same label, bit for bit);
// row_stats[t] = (max, log sum) when row_stats is not null.  lab >= V gives NaN in both logp_t and the log sum.
__global__ void __launch_bounds__(kRowThreads) logprob_row_kernel(const __nv_bfloat16* __restrict__ z,
                                                                 const float2* __restrict__ part, int n_vt,
                                                                 const int64_t* __restrict__ labels, int V,
                                                                 float* __restrict__ logp, float2* __restrict__ row_stats) {
  __shared__ float red[kRowThreads / 32];
  pdl_sync();
  const int64_t t = blockIdx.x;
  const int64_t lab = max(labels[t], (int64_t)0);
  const bool bad = lab >= V;
  const float z_lab = (threadIdx.x == 0 && !bad) ? __bfloat162float(z[t * (int64_t)V + lab]) : 0.f;
  const float2 ms = row_max_sum<kRowThreads>(part + t * (int64_t)n_vt, n_vt, red);
  const float logsum = bad ? __int_as_float(0x7fc00000) : logf(ms.y);
  if (threadIdx.x == 0) {
    logp[t] = __fsub_rn(__fsub_rn(z_lab, ms.x), logsum);
    if (row_stats) row_stats[t] = make_float2(ms.x, logsum);
  }
}

// One CTA per row t: G over z in place from c_t = grad_logp[t], the log_softmax backward of gather's scatter of c_t to
// the clipped label: G_v = [v == lab] * c_t - exp(lsm_v) * c_t, computed as ce_row_kernel computes its G with
// w = -c_t (equal values; exact negations).
__global__ void __launch_bounds__(kRowThreads) logprob_grad_row_kernel(__nv_bfloat16* __restrict__ z,
                                                                      const float2* __restrict__ row_stats,
                                                                      const int64_t* __restrict__ labels,
                                                                      const float* __restrict__ grad_logp, int V) {
  pdl_sync();
  const int64_t t = blockIdx.x;
  const float2 st = row_stats[t];
  grad_row_in_place<kRowThreads>(reinterpret_cast<uint4*>(z + t * (int64_t)V), V / 8, st.x, st.y, -grad_logp[t],
                                 max(labels[t], (int64_t)0));
}

__global__ void __launch_bounds__(kLossThreads) ce_loss_kernel(const float* __restrict__ row_ce,
                                                              const float* __restrict__ loss_weight, int64_t T,
                                                              float* __restrict__ loss) {
  __shared__ float red[kLossThreads / 32];
  pdl_sync();
  float s = 0.f;
  for (int64_t t = threadIdx.x; t < T; t += kLossThreads) s += __fmul_rn(row_ce[t], loss_weight[t]);
  s = block_reduce<kLossThreads, false>(s, red);
  if (threadIdx.x == 0) *loss = s;
}

}  // namespace xtb

using namespace xtb;

extern "C" size_t xtb_lm_head_ce_workspace_bytes(int64_t T, int V) {
  if (T < 0 || V <= 0 || V % 128) return 0;
  return kWsHeader + (size_t)T * lm_head_ce_vocab_tiles(V) * sizeof(float2);
}

extern "C" int xtb_lm_head_ce(const void* h, const void* w, const int64_t* labels, const float* loss_weight, int64_t T,
                              int H, int V, int64_t ignore_index, int need_grad, void* z_or_G, void* workspace,
                              float* row_ce, float* loss, void* dh, void* dW, xtb_stream_t stream) {
  XTB_CHECK_ARG(h && w && labels && loss_weight && z_or_G && workspace && row_ce && loss, "xtb_lm_head_ce: null pointer");
  XTB_CHECK_ARG(!need_grad || (dh && dW), "xtb_lm_head_ce: null pointer (dh and dW are required with need_grad)");
  XTB_CHECK_ARG(T >= 0 && T < (1ll << 31), "xtb_lm_head_ce: bad T=%lld", (long long)T);
  XTB_CHECK_ARG(H > 0 && V > 0 && H % 128 == 0 && V % 128 == 0, "xtb_lm_head_ce: H=%d and V=%d must be multiples of 128",
                H, V);
  const uintptr_t align = reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(w) |
                          reinterpret_cast<uintptr_t>(z_or_G) | reinterpret_cast<uintptr_t>(workspace) |
                          reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(dW);
  XTB_CHECK_ARG((align & 15) == 0, "xtb_lm_head_ce: h, w, z_or_G, workspace, dh and dW must be 16-byte aligned");
  XTB_CHECK_ARG((reinterpret_cast<uintptr_t>(labels) & 7) == 0 && (reinterpret_cast<uintptr_t>(loss_weight) & 3) == 0 &&
                    (reinterpret_cast<uintptr_t>(row_ce) & 3) == 0 && (reinterpret_cast<uintptr_t>(loss) & 3) == 0,
                "xtb_lm_head_ce: labels, loss_weight, row_ce and loss must be aligned to their element size");
  XTB_ENSURE_CTX(h);
  cudaStream_t st = as_stream(stream);
  if (T == 0) {
    XTB_CUDA(cudaMemsetAsync(loss, 0, sizeof(float), st));
    if (need_grad) XTB_CUDA(cudaMemsetAsync(dW, 0, (size_t)V * H * 2, st));
    return XTB_OK;
  }
  int64_t* tpe = static_cast<int64_t*>(workspace);
  float2* part = reinterpret_cast<float2*>(static_cast<uint8_t*>(workspace) + kWsHeader);
  XTB_LAUNCH(ce_set_rows_kernel, dim3(1), dim3(32), 0, st, true, tpe, T);
  int rc = lm_head_logits_ce(h, w, tpe, T, H, V, z_or_G, part, st);
  if (rc) return rc;
  XTB_LAUNCH(ce_row_kernel, dim3((unsigned)T), dim3(kRowThreads), 0, st, true, static_cast<__nv_bfloat16*>(z_or_G),
             static_cast<const float2*>(part), lm_head_ce_vocab_tiles(V), labels, ignore_index, loss_weight, V,
             need_grad, row_ce);
  XTB_LAUNCH(ce_loss_kernel, dim3(1), dim3(kLossThreads), 0, st, true, static_cast<const float*>(row_ce), loss_weight,
             T, loss);
  if (!need_grad) return XTB_OK;
  if ((rc = xtb_group_gemm_nn(z_or_G, w, tpe, T, V, H, 1, dh, stream))) return rc;
  return xtb_group_gemm_tn(z_or_G, h, tpe, T, V, H, 1, dW, stream);
}

extern "C" size_t xtb_lm_head_logprob_workspace_bytes(int64_t T, int V) { return xtb_lm_head_ce_workspace_bytes(T, V); }

extern "C" int xtb_lm_head_logprob(const void* h, const void* w, const int64_t* labels, int64_t T, int H, int V, void* z,
                                   void* workspace, float* logp, float* row_stats, xtb_stream_t stream) {
  XTB_CHECK_ARG(h && w && labels && z && workspace && logp, "xtb_lm_head_logprob: null pointer");
  XTB_CHECK_ARG(T >= 0 && T < (1ll << 31), "xtb_lm_head_logprob: bad T=%lld", (long long)T);
  XTB_CHECK_ARG(H > 0 && V > 0 && H % 128 == 0 && V % 128 == 0,
                "xtb_lm_head_logprob: H=%d and V=%d must be multiples of 128", H, V);
  const uintptr_t align = reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(z) |
                          reinterpret_cast<uintptr_t>(workspace);
  XTB_CHECK_ARG((align & 15) == 0, "xtb_lm_head_logprob: h, w, z and workspace must be 16-byte aligned");
  XTB_CHECK_ARG((reinterpret_cast<uintptr_t>(labels) & 7) == 0 && (reinterpret_cast<uintptr_t>(logp) & 3) == 0 &&
                    (reinterpret_cast<uintptr_t>(row_stats) & 7) == 0,
                "xtb_lm_head_logprob: labels and row_stats must be 8-byte aligned, logp 4-byte aligned");
  XTB_ENSURE_CTX(h);
  if (T == 0) return XTB_OK;
  cudaStream_t st = as_stream(stream);
  int64_t* tpe = static_cast<int64_t*>(workspace);
  float2* part = reinterpret_cast<float2*>(static_cast<uint8_t*>(workspace) + kWsHeader);
  XTB_LAUNCH(ce_set_rows_kernel, dim3(1), dim3(32), 0, st, true, tpe, T);
  const int rc = lm_head_logits_ce(h, w, tpe, T, H, V, z, part, st);
  if (rc) return rc;
  XTB_LAUNCH(logprob_row_kernel, dim3((unsigned)T), dim3(kRowThreads), 0, st, true,
             static_cast<const __nv_bfloat16*>(z), static_cast<const float2*>(part), lm_head_ce_vocab_tiles(V),
             labels, V, logp, reinterpret_cast<float2*>(row_stats));
  return XTB_OK;
}

extern "C" int xtb_lm_head_logprob_bwd(void* z_or_G, const float* row_stats, const int64_t* labels, const float* grad_logp,
                                       const void* h, const void* w, int64_t T, int H, int V, void* workspace, void* dh,
                                       void* dW, xtb_stream_t stream) {
  XTB_CHECK_ARG(z_or_G && row_stats && labels && grad_logp && h && w && workspace && dh && dW,
                "xtb_lm_head_logprob_bwd: null pointer");
  XTB_CHECK_ARG(T >= 0 && T < (1ll << 31), "xtb_lm_head_logprob_bwd: bad T=%lld", (long long)T);
  XTB_CHECK_ARG(H > 0 && V > 0 && H % 128 == 0 && V % 128 == 0,
                "xtb_lm_head_logprob_bwd: H=%d and V=%d must be multiples of 128", H, V);
  const uintptr_t align = reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(w) |
                          reinterpret_cast<uintptr_t>(z_or_G) | reinterpret_cast<uintptr_t>(workspace) |
                          reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(dW);
  XTB_CHECK_ARG((align & 15) == 0, "xtb_lm_head_logprob_bwd: h, w, z_or_G, workspace, dh and dW must be 16-byte aligned");
  XTB_CHECK_ARG((reinterpret_cast<uintptr_t>(labels) & 7) == 0 && (reinterpret_cast<uintptr_t>(row_stats) & 7) == 0 &&
                    (reinterpret_cast<uintptr_t>(grad_logp) & 3) == 0,
                "xtb_lm_head_logprob_bwd: labels and row_stats must be 8-byte aligned, grad_logp 4-byte aligned");
  XTB_ENSURE_CTX(h);
  cudaStream_t st = as_stream(stream);
  if (T == 0) {
    XTB_CUDA(cudaMemsetAsync(dW, 0, (size_t)V * H * 2, st));
    return XTB_OK;
  }
  int64_t* tpe = static_cast<int64_t*>(workspace);
  XTB_LAUNCH(ce_set_rows_kernel, dim3(1), dim3(32), 0, st, true, tpe, T);
  XTB_LAUNCH(logprob_grad_row_kernel, dim3((unsigned)T), dim3(kRowThreads), 0, st, true,
             static_cast<__nv_bfloat16*>(z_or_G), reinterpret_cast<const float2*>(row_stats), labels, grad_logp,
             V);
  int rc;
  if ((rc = xtb_group_gemm_nn(z_or_G, w, tpe, T, V, H, 1, dh, stream))) return rc;
  return xtb_group_gemm_tn(z_or_G, h, tpe, T, V, H, 1, dW, stream);
}
