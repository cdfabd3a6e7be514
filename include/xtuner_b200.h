/*
 * xtuner_b200.h — C-ABI of the H100-native (sm_90a) MoE hot path for XTuner V1.
 *
 * Drop-in boundary (SURVEY.md §8b).  Every entry point takes raw DEVICE pointers, plain sizes and a
 * cudaStream_t (passed as void*); no torch types, no allocation inside (workspaces are passed in, sized
 * by the matching *_workspace_bytes call); returns 0 on success, non-zero on failure, with a
 * thread-local message available from xtb_last_error().  Kernels are enqueued on the given stream and
 * never synchronise the host.  There is NO CPU fallback: without a CUDA device every compute entry
 * point fails.
 *
 * Each entry cites the reference interface (InternLM/xtuner @ b934f46, paths relative to the reference
 * root) it replaces.  The reference-side bindings are shown in INTEGRATION.md.
 *
 * Conventions shared by all entries
 *   T  tokens on this rank          H  hidden size           E  routed experts (local)
 *   K  experts per token (top-k)    I  expert intermediate    M = T*K permuted rows
 *   activations / expert weights are bf16 (XTB_BF16); router math is fp32; ids follow the reference's
 *   dtypes (topk_ids int64 out of the router, int32 into permute, tokens_per_expert int64).
 *   "flat index" f = t*K + k (token-major), the order the reference sorts (permute_unpermute.py:214-215).
 */
#ifndef XTUNER_B200_H_
#define XTUNER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XTB_VERSION 100 /* 0.1.0 */

typedef void* xtb_stream_t; /* cudaStream_t */

enum xtb_status {
  XTB_OK = 0,
  XTB_ERR_INVALID = 1,     /* bad argument / unsupported shape */
  XTB_ERR_CUDA = 2,        /* CUDA runtime / driver error (message has the string) */
  XTB_ERR_UNSUPPORTED = 3, /* device is not sm_90 */
};

enum xtb_scoring { XTB_SCORE_SOFTMAX = 0, XTB_SCORE_SIGMOID = 1 };

/* ---- library ---------------------------------------------------------------------------------- */
int xtb_version(void);
const char* xtb_last_error(void);
/* Checks that the current device is sm_90 and resolves the driver entry points (TMA descriptors). */
int xtb_init(void);
/* Number of kernels this library has launched since load / last reset (bench.py "gpu_launches"). */
int64_t xtb_launch_count(void);
void xtb_reset_launch_count(void);

/* ---- a1  MoEGate.forward: module/decoder_layer/moe_decoder_layer.py:120-141 ------------------------
 * logits[T,E] (fp32) = float(x[T,H] bf16) @ float(w[E,H])^T (+ bias[E]), fp32 FMA accumulation.
 * w is fp32 (the reference upcasts the gate weight: `weight.float()`, :140).  bias may be NULL. */
int xtb_gate_logits(const void* x_bf16, const float* w_f32, const float* bias_f32, float* logits, int T, int H,
                    int E, xtb_stream_t stream);
/* backward of a1: grad_w[E,H] (fp32, overwritten) = grad_logits^T @ float(x);
 *                 grad_x[T,H] (bf16, overwritten) = bf16(grad_logits @ w)   (autograd of x.float()). */
size_t xtb_gate_logits_bwd_workspace_bytes(int T, int H, int E);
int xtb_gate_logits_bwd(const float* grad_logits, const void* x_bf16, const float* w_f32, float* grad_w,
                        void* grad_x_bf16, float* grad_bias /*nullable*/, int T, int H, int E, void* workspace,
                        xtb_stream_t stream);

/* ---- a2  GreedyRouter.forward: module/router/greedy.py:64-98 ---------------------------------------
 * router_weights[T,E] = softmax(logits, dim=1) in fp32 (or sigmoid); topk over E (descending);
 * optional renormalisation (`topk_weights /= sum`, :82-83) and scaling (:85-86);
 * tokens_per_expert[E] = histc(topk_ids, bins=E) as int64 (:90).  topk_ids are int64 like torch.topk.
 * topk_ids_i32 (nullable) additionally receives the int32 copy the dispatcher makes
 * (`topk_ids.to(torch.int32)`, module/dispatcher/base.py:396). */
int xtb_router_greedy(const float* logits, int T, int E, int K, int scoring, int norm_topk_prob, float scaling,
                      float* router_weights, float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32,
                      int64_t* tokens_per_expert, xtb_stream_t stream);
/* a2 + the index half of a4 in ONE launch: same outputs as xtb_router_greedy, and additionally fills
 * `dispatch_workspace` (xtb_moe_permute_workspace_bytes(T,K,E) bytes) with the per-chunk histograms and
 * their scan, so that xtb_moe_permute_prepared() can gather rows without a counting pass.  Replaces the
 * reference's second histogram (`torch.histc` in dispatcher/base.py:398) and the sort of
 * ops/moe/cuda/permute_unpermute.py:215.  topk_ids_i32 is required. */
int xtb_router_greedy_dispatch(const float* logits, int T, int E, int K, int scoring, int norm_topk_prob,
                               float scaling, float* router_weights, float* topk_weights, int64_t* topk_ids,
                               int32_t* topk_ids_i32, int64_t* tokens_per_expert, void* dispatch_workspace,
                               xtb_stream_t stream);
/* a1 + a2 + the index half of a4 in ONE launch (csrc/gate_mma.cu) — what the fused layer calls.  Gate logits on the
 * tensor cores (fp32 weight as three bf16 planes, exact products, fp32 accumulation), then the per-token code of
 * xtb_router_greedy_dispatch itself (csrc/greedy_router.cuh) on the 32-token block that is still in shared memory, then
 * the chunk histograms and their scan: the outputs of xtb_gate_logits (no bias) followed by xtb_router_greedy_dispatch,
 * one kernel instead of two and no logits round trip.  The logits equal float64 on exact inputs and stay within the bound of
 * tests/router_reference.py otherwise; every other output, the dispatch workspace included, is bit-equal on an H100 to
 * xtb_router_greedy_dispatch run on those logits (tests/test_gpu_router_edges.py).  E <= 8, K <= 8, H % 128 == 0,
 * H <= 4224; XTB_ERR_INVALID otherwise (use the two calls). */
int xtb_gate_route_dispatch(const void* x_bf16, const float* w_f32, int T, int H, int E, int K, int scoring,
                            int norm_topk_prob, float scaling, float* logits, float* router_weights,
                            float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32, int64_t* tokens_per_expert,
                            void* dispatch_workspace, xtb_stream_t stream);
/* backward of a2 through its three differentiable outputs (SURVEY.md Appendix B "three routes"):
 * grad_logits[T,E] = d(topk_weights)·grad_topk_weights + d(router_weights)·grad_router_weights
 *                    (+ grad_logits_direct if not NULL).  Either grad input may be NULL (treated as 0). */
int xtb_router_greedy_bwd(const float* router_weights, const float* topk_weights, const int64_t* topk_ids,
                          const float* grad_topk_weights, const float* grad_router_weights,
                          const float* grad_logits_direct, int T, int E, int K, int scoring, int norm_topk_prob,
                          float scaling, float* grad_logits, xtb_stream_t stream);

/* backward of a2 and of a1 in ONE launch — what the fused layer calls; bit-equal on an H100 to xtb_router_greedy_bwd +
 * xtb_gate_logits_bwd (tests/test_gpu_router_edges.py): grad_logits is computed per token in the prologue of the
 * gate backward by the per-token code of xtb_router_greedy_bwd itself (csrc/greedy_router.cuh) and never written to
 * memory; grad_w / grad_x as xtb_gate_logits_bwd (no bias).  workspace: xtb_gate_logits_bwd_workspace_bytes(T, H, E).
 * E <= 8, H % 8 == 0; XTB_ERR_INVALID otherwise (use the two calls). */
int xtb_router_gate_bwd(const float* router_weights, const float* topk_weights, const int64_t* topk_ids,
                        const float* grad_topk_weights, const float* grad_router_weights,
                        const float* grad_logits_direct, const void* x_bf16, const float* w_f32, float* grad_w,
                        void* grad_x_bf16, int T, int H, int E, int K, int scoring, int norm_topk_prob, float scaling,
                        void* workspace, xtb_stream_t stream);

/* ---- a2' NoAuxRouter.forward: module/router/noaux_router.py:78-150 (DeepSeek-V3 style) --------------
 * sigmoid scores; choice scores = scores + bias; group-limited routing (top-2 sum per group, keep
 * topk_group groups); topk on masked choice scores; weights gathered from the UNBIASED scores, renormalised
 * with +1e-20 and scaled; router_weights = masked choice scores / row sum; tokens_per_expert as FLOAT32
 * (the reference calls histc on `topk_ids.float()`, :137-142). */
int xtb_router_noaux(const float* logits, const float* e_score_correction_bias, int T, int E, int K, int n_group,
                     int topk_group, int norm_topk_prob, float scaling, float* router_weights,
                     float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32, float* tokens_per_expert_f32,
                     xtb_stream_t stream);

/* backward of a2' (what autograd does to noaux_router.py:80-134; closed form in oracle/moe_oracle.py
 * noaux_router_bwd).  Inputs are the forward's inputs and outputs, and its group geometry as
 * group_spec = XTB_NOAUX_GROUP_SPEC(n_group, topk_group): 0 when n_group == topk_group (no group mask), otherwise
 * n_group | topk_group << 8.  The kept-group mask is recomputed from logits and bias: a kept expert's router weight may
 * be exactly 0, so router_weights != 0 does not identify it.  Either grad may be NULL. */
#define XTB_NOAUX_GROUP_SPEC(n_group, topk_group) \
  ((n_group) == (topk_group) ? 0 : ((n_group) | ((topk_group) << 8)))
int xtb_router_noaux_bwd(const float* logits, const float* e_score_correction_bias, const float* router_weights,
                         const float* topk_weights, const int64_t* topk_ids, const float* grad_topk_weights,
                         const float* grad_router_weights, int T, int E, int K, int group_spec,
                         int norm_topk_prob, float scaling, float* grad_logits, xtb_stream_t stream);

/* ---- a4  permute: ops/moe/protocol.py:15-23, ops/moe/cuda/permute_unpermute.py:92-143,205-219 -------
 * Stable sort of the flat [T*K] expert ids; permuted[r] = x[sorted_indices[r] / K].
 *   row_id_map[f]      (int32, [T*K])  = permuted row of flat index f  (opaque handle for unpermute)
 *   sorted_indices[r]  (int64, [T*K], nullable) = flat index held by row r (== the in-tree fallback's
 *                      `row_id_map`, permute_unpermute.py:215)
 *   tokens_per_expert  (int64, [E], nullable)   = histogram of ids (dispatcher/base.py:398)
 * ids outside [0,E) are invalid (the dropless path never produces them).  row_bytes = H * sizeof(elt),
 * must be a multiple of 16. */
/* The workspace (ticket | expert_start[E] | per-chunk counts) must be ZERO-FILLED ONCE after it is allocated: the last CTA
 * of every call that uses it resets the ticket, so each call leaves it ready for the next and no memset runs on the hot
 * path (a memset node between two kernels would also cut the programmatic dependent launch between them).  One
 * workspace per stream. */
size_t xtb_moe_permute_workspace_bytes(int T, int K, int E);
int xtb_moe_permute(const void* x, const int32_t* ids, int T, int K, int E, int64_t row_bytes, void* permuted,
                    int32_t* row_id_map, int64_t* sorted_indices, int64_t* tokens_per_expert, void* workspace,
                    xtb_stream_t stream);
/* Row gather of a4 against a workspace prepared by xtb_router_greedy_dispatch (same T, K, E, ids). */
int xtb_moe_permute_prepared(const void* x, const int32_t* ids, int T, int K, int E, int64_t row_bytes,
                             void* permuted, int32_t* row_id_map, int64_t* sorted_indices,
                             const void* prepared_workspace, xtb_stream_t stream);

/* ---- a5  unpermute: ops/moe/protocol.py:26-30, permute_unpermute.py:146-192,222-248 ----------------
 * out[t] = bf16( sum_k fp32(probs[t,k]) * fp32(y[row_id_map[t*K+k]]) ), fp32 accumulation in k order.
 * probs == NULL: plain sum (this is also permute's backward, :129-143). */
int xtb_moe_unpermute(const void* y_bf16, const int32_t* row_id_map, const float* probs, int T, int K, int H,
                      void* out_bf16, xtb_stream_t stream);
/* a5 fused with MoEDecoderLayer._post_moe_forward (module/decoder_layer/moe_decoder_layer.py:696-705):
 *   out[t] = bf16( bf16( bf16(sum_k p*y) * hidden_factor ) + residual[t] )   (each eager op's bf16 rounding
 * kept).  residual may be NULL (then only the factor is applied); hidden_factor == 1 skips that rounding. */
int xtb_moe_combine(const void* y_bf16, const int32_t* row_id_map, const float* probs, const void* residual_bf16,
                    float hidden_factor, int T, int K, int H, void* out_bf16, xtb_stream_t stream);
/* backward of a5 (`moe::unpermute_bwd`, permute_unpermute.py:64-76,177-192):
 *   act_grad[r]      (bf16 [T*K,H]) = bf16( fp32(grad_out[t]) * probs[t,k] ),  r = row_id_map[t*K+k]
 *   prob_grad[t,k]   (fp32 [T,K])   = sum_h fp32(grad_out[t,h]) * fp32(y_fwd[r,h])     (nullable) */
int xtb_moe_unpermute_bwd(const void* grad_out_bf16, const void* y_fwd_bf16, const int32_t* row_id_map,
                          const float* probs, int T, int K, int H, void* act_grad_bf16, float* prob_grad,
                          xtb_stream_t stream);

/* ---- a6/a7  grouped expert GEMMs: ops/moe/protocol.py:6-12, ops/moe/cuda/group_gemm.py:8-37 ----------
 * wgmma kernels, fp32 accumulation in registers, bf16 in/out.  tokens_per_expert is a DEVICE int64
 * [E] tensor (never read on the host); rows of x are sorted by expert (group e owns rows
 * [cumsum[e-1], cumsum[e]) ).  M_total = rows of x (sum of tokens_per_expert).
 *
 *  xtb_group_gemm_nt : out[M_total,N]   = x[M_total,Kd] @ w[e][N,Kd]^T      (m_grouped_gemm trans_b=True)
 *  xtb_group_gemm_nn : out[M_total,Kd]  = dy[M_total,N] @ w[e][N,Kd]        (m_grouped_gemm trans_b=False, dX)
 *  xtb_group_gemm_tn : dw[E,N,Kd]       = dy[rows e]^T[N,rows] @ x[rows e][rows,Kd]   (k_grouped_gemm, dW;
 *                      an expert with zero rows gets a zero matrix)
 * Constraints: N % 128 == 0, Kd % 128 == 0.  w is [E,N,Kd] contiguous. */
int xtb_group_gemm_nt(const void* x, const void* w, const int64_t* tokens_per_expert, int64_t M_total, int N,
                      int Kd, int E, void* out, xtb_stream_t stream);
/* a6+a8 fused (MoEBlock.forward, moe_decoder_layer.py:196-200): h[M,2I] = x . w13[e]^T as above AND
 * a[M,I] = bf16( bf16(silu(h[:, :I])) * h[:, I:] ) from the same accumulators (the SwiGLU is applied in the
 * GEMM epilogue on the bf16-rounded h, so results equal the unfused pair).  I % 64 == 0. */
int xtb_group_gemm_nt_swiglu(const void* x, const void* w13, const int64_t* tokens_per_expert, int64_t M_total,
                             int I, int Kd, int E, void* h_out, void* a_out, xtb_stream_t stream);
int xtb_group_gemm_nn(const void* dy, const void* w, const int64_t* tokens_per_expert, int64_t M_total, int N,
                      int Kd, int E, void* out, xtb_stream_t stream);
int xtb_group_gemm_tn(const void* dy, const void* x, const int64_t* tokens_per_expert, int64_t M_total, int N,
                      int Kd, int E, void* dw, xtb_stream_t stream);
/* both weight gradients of the expert MLP (GroupedLinear.backward of fused_w2 and fused_w1w3, moe_group_linear.py:162-173
 * through ops/moe/cuda/group_gemm.py:25-37) in ONE launch: dw_a = xtb_group_gemm_tn(dy_a, x_a, N_a, Kd_a) and
 * dw_b = xtb_group_gemm_tn(dy_b, x_b, N_b, Kd_b) over the same tokens_per_expert — identical bits, one persistent tile list
 * over both products (fills the partly empty last wave each product has alone).  Shapes the CTA-pair kernel does not
 * take (not multiples of 256) run as the two separate launches. */
int xtb_group_gemm_tn_pair(const void* dy_a, const void* x_a, int N_a, int Kd_a, void* dw_a, const void* dy_b,
                           const void* x_b, int N_b, int Kd_b, void* dw_b, const int64_t* tokens_per_expert,
                           int64_t M_total, int E, xtb_stream_t stream);
/* ---- f4  lm_head + cross-entropy: loss/ce_loss.py LMHeadLossContext.loss_fn (mode "eager"; "chunk" runs it per chunk)
 * For T rows of h[T,H] (bf16), head weight w[V,H] (bf16, no bias), labels[T] (int64) and loss_weight[T] (fp32):
 *   z        = bf16(h . w^T), fp32 accumulation                                   ([T,V] bf16, in z_or_G)
 *   lsm      = (z - max) - log(sum exp(z - max))  per row, fp32
 *   row_ce[t]= -lsm[t, labels[t]]  (fp32 [T]);  0 where labels[t] == ignore_index
 *   *loss    = sum_t row_ce[t] * loss_weight[t]  (fp32 scalar, fixed summation order: identical bits run to run;
 *              exactly 0 when every row is ignored)
 * need_grad != 0 additionally (the backward of the above for a loss gradient of 1):
 *   G        = bf16(exp(lsm) * loss_weight[t] - [v == labels[t]] * loss_weight[t]), written OVER z in z_or_G
 *              (ignored rows: exactly 0)
 *   dh[T,H]  = bf16(G . w)      (xtb_group_gemm_nn with one group)
 *   dW[V,H]  = bf16(G^T . h)    (xtb_group_gemm_tn with one group)
 * need_grad == 0 leaves z in z_or_G; dh and dW may then be NULL.
 * A label outside [0, V) that is not ignore_index does not fault: that row's row_ce is NaN (so is the loss, and with
 * need_grad that row of G).
 * V % 128 == 0, H % 128 == 0, T < 2^31 (T*V may exceed 2^31: all row offsets are 64-bit).  workspace:
 * xtb_lm_head_ce_workspace_bytes(T, V) bytes, 16-byte aligned, no initialisation needed. */
size_t xtb_lm_head_ce_workspace_bytes(int64_t T, int V);
int xtb_lm_head_ce(const void* h, const void* w, const int64_t* labels, const float* loss_weight, int64_t T, int H, int V,
                   int64_t ignore_index, int need_grad, void* z_or_G, void* workspace, float* row_ce, float* loss, void* dh,
                   void* dW, xtb_stream_t stream);
/* ---- a8  native_swiglu: ops/act_fn.py:7-9 ---------------------------------------------------------
 * out[m, j] = bf16( bf16(silu(h[m, j])) * h[m, I + j] ),  h is [M, 2I] bf16 (gate | up).  I % 8 == 0; every pointer of
 * both entries 16-byte aligned. */
int xtb_swiglu(const void* h_bf16, void* out_bf16, int64_t M, int I, xtb_stream_t stream);
/* autograd of the two eager ops (silu, mul) with their bf16 roundings:
 *   grad_h[m, I + j] = bf16(g * s),  s = bf16(silu(x1));  d_s = bf16(g * x2);
 *   grad_h[m, j]     = bf16( d_s * sigmoid(x1) * (1 + x1 * (1 - sigmoid(x1))) )
 * I / 8 <= 23170 (the row split's 32-bit reciprocal). */
int xtb_swiglu_bwd(const void* grad_out_bf16, const void* h_bf16, void* grad_h_bf16, int64_t M, int I,
                   xtb_stream_t stream);

/* ==== the step either side of the path (SURVEY.md §8f-3) =================================================
 * post_attention_layernorm (module/decoder_layer/moe_decoder_layer.py:664-679; F.rms_norm via
 * ops/rms_norm/__init__.py:8-11) fused with its neighbours.
 *
 * xtb_rmsnorm_gate: x = bf16(float(h) * rsqrt(mean(h^2)+eps) * norm_w); rstd[T] saved for backward; when
 * gate_w is not NULL also logits[T,E] = float(x) @ gate_w^T (a1) in the same pass (E <= 8, (E+1)*H*4 <= 200 KiB). */
int xtb_rmsnorm_gate(const void* h_bf16, const float* norm_w_f32, const float* gate_w_f32, float eps, int T, int H,
                     int E, void* x_out_bf16, float* rstd_out, float* logits, xtb_stream_t stream);
/* Backward chain of the MoE half's input side in one kernel:
 *   g_x = bf16( bf16(sum_k g_xperm[row_id_map[t*K+k]]) + g_x_gate )      (permute backward + autograd's add;
 *                                                                         g_x_gate may be NULL)
 *   g_h = bf16( rmsnorm_backward(g_x; h, rstd, norm_w) ) (+ g_res, the residual branch's gradient, if not NULL)
 *   g_norm_w[H] = sum_t float(g_x) * h * rstd   (NULL to skip; needs the workspace) */
size_t xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(int T, int H);
int xtb_moe_dispatch_bwd_rmsnorm(const void* g_xperm_bf16, const int32_t* row_id_map, const void* g_x_gate_bf16,
                                 const void* h_bf16, const float* rstd, const float* norm_w_f32,
                                 const void* g_res_bf16, int T, int K, int H, void* g_h_bf16, float* g_norm_w,
                                 void* workspace, xtb_stream_t stream);

/* q_norm / k_norm and the rotary embedding in front of the attention (MultiHeadAttention.forward,
 * module/attention/mha.py:353-363: RMSNorm = F.rms_norm, ops/rms_norm/__init__.py:8-11, then
 * apply_rotary_pos_emb_cuda, ops/rotary_emb.py:18-49), one kernel each way for q and k together.
 *   q [T, Hq, D], k [T, Hkv, D] bf16 with any token / head stride (elements, multiples of 8) and the D axis contiguous;
 *   cos, sin [T, D] bf16 contiguous (all D columns are read); w_q, w_k [D] fp32, or both NULL for qk_norm=False.
 *   half = D/2, D in {64, 128, 256} (XTB_ERR_INVALID otherwise); pointers 16-byte aligned.
 * Forward, per (token, head) row x:
 *   rstd  = rsqrtf(mean(x^2) + eps) in fp32, written to rstd_q [T, Hq] / rstd_k [T, Hkv]   (norm only)
 *   n_i   = bf16((x_i rstd) w_i)                 (n = x without the norm)
 *   r_i   = -n_{i+half} for i < half, n_{i-half} otherwise                        (rotate_half)
 *   out_i = bf16( bf16(n_i cos_i) + bf16(r_i sin_i) )  into contiguous out_q [T, Hq, D], out_k [T, Hkv, D]
 * Backward, g = grad of out (same stride rules as q / k):
 *   gn_i  = bf16( bf16(g_i cos_i) + bf16(g_{i+half} sin_{i+half}) )   for i < half
 *   gn_i  = bf16( bf16(g_i cos_i) - bf16(g_{i-half} sin_{i-half}) )   for i >= half   (autograd's roundings)
 *   dx    = bf16( (w gn - x c) rstd ),  c = (sum_i w_i gn_i x_i) rstd^2 / D           (dx = gn without the norm)
 *   dw    [2D] fp32 = [dw_q | dw_k], dw_q = sum over (t, h) of gn x rstd, summed in a fixed order (identical bits run to
 *         run); NULL to skip, needs xtb_qk_norm_rope_bwd_workspace_bytes(T, D) bytes of workspace.  cos and sin get no
 *         gradient.  dx_q / dx_k are contiguous [T, Hq, D] / [T, Hkv, D].
 * T = 0 is a no-op (the backward then writes dw = 0).  Byte offsets are 64-bit: T * H * D may exceed 2^31. */
int xtb_qk_norm_rope(const void* q_bf16, int64_t q_stride_t, int64_t q_stride_h, const void* k_bf16, int64_t k_stride_t,
                     int64_t k_stride_h, const void* cos_bf16, const void* sin_bf16, const float* w_q_f32,
                     const float* w_k_f32, float eps, int T, int Hq, int Hkv, int D, void* out_q_bf16, void* out_k_bf16,
                     float* rstd_q, float* rstd_k, xtb_stream_t stream);
size_t xtb_qk_norm_rope_bwd_workspace_bytes(int T, int D);
int xtb_qk_norm_rope_bwd(const void* g_q_bf16, int64_t g_q_stride_t, int64_t g_q_stride_h, const void* g_k_bf16,
                         int64_t g_k_stride_t, int64_t g_k_stride_h, const void* q_bf16, int64_t q_stride_t,
                         int64_t q_stride_h, const void* k_bf16, int64_t k_stride_t, int64_t k_stride_h,
                         const void* cos_bf16, const void* sin_bf16, const float* w_q_f32, const float* w_k_f32,
                         const float* rstd_q, const float* rstd_k, int T, int Hq, int Hkv, int D, void* dx_q_bf16,
                         void* dx_k_bf16, float* dw, void* workspace, xtb_stream_t stream);

/* ==== fp8 tile-wise quantisation (row a15, config 5) ============================================================
 * e4m3, scale = clamp(amax, 1e-12) / 448 (xtuner/v1/float8/float8_utils.py:6-32, fsdp_utils.py:75-116,195-223,
 * triton_kernels/per_tile_quant.py:61-100).  Bit-exact on an H100 against reference-made golden vectors
 * (tests/test_gpu_fp8.py), and against the oracle and the reference's own functions on every bf16 value in
 * [-448, 448], all-zero blocks, fp32 and bf16 weights and NaN / inf inputs (tests/test_gpu_fp8_edges.py): a NaN makes
 * its tile's or block's scale and bytes NaN, an inf gives an inf scale.  x must be 8-byte aligned, q and scales 4-byte
 * aligned; nw <= 65535.  Nothing on the bf16 default path calls these; `plugin.install_fp8_cast()` rebinds the
 * reference's FSDP fp8 all-gather cast (`WeightWithDynamicTilewiseFloat8CastTensor.fsdp_pre_all_gather`,
 * fsdp_utils.py:379-409) and its scale precompute to them.  There is no fp8 grouped GEMM here yet. */
int xtb_fp8_per_tile_quant(const void* x_bf16, void* q_e4m3, float* scales /*[M, K/128]*/, int64_t M, int64_t K,
                           xtb_stream_t stream);
int xtb_fp8_block_scales(const void* w, int w_is_f32, int64_t nw, int dout, int din,
                         float* scales /*[nw, dout/128, din/128]*/, xtb_stream_t stream);
int xtb_fp8_block_cast(const void* w, int w_is_f32, int64_t nw, int dout, int din, const float* scales, void* q_e4m3,
                       xtb_stream_t stream);

/* ==== peer-memory (NVLink / NVSwitch) exchange steps ===================================================
 * "peer pointer arrays" are DEVICE arrays of `world` base addresses of a symmetric allocation (same size on
 * every rank, all mapped into every rank: torch.distributed._symmetric_memory or CUDA IPC on the host side). */

/* Rendezvous of all ranks on `stream`: rank r sets slot [channel*world + r] of every peer's signal pad
 * (uint32 array, zero-initialised, >= (channel+1)*world entries) and waits for every peer's mark in its own. */
int xtb_peer_barrier(void* const* signal_pad_ptrs_dev, int rank, int world, int channel, xtb_stream_t stream);

/* a12  ulysses_all_to_all: xtuner/v1/ops/comm/all_to_all.py:6-51 (call sites module/attention/mha.py:373-390,
 * 421-427).  Every rank PULLS its share of every peer's input straight into the final output layout — the
 * reference's contiguous/movedim before and tensor_split/cat after the NCCL all-to-all (all_to_all.py:35-50)
 * disappear into the addressing.  Rows are indexed (o, x, m) with n_o*n_x*n_m rows of row_bytes each:
 *   src byte offset in peer s's buffer = src_base + o*src_stride_o + x*src_stride_x + m*src_stride_m
 *   dst byte offset in `out`           = s*dst_peer_stride + o*dst_stride_o + x*dst_stride_x + m*dst_stride_m
 * (all multiples of 16).  The host helper xtuner_b200.comm.a2a_plan derives them from (shape, scatter_dim,
 * gather_dim, world, rank).  Callers order it after an xtb_peer_barrier ("inputs are ready"). */
int xtb_a2a_pull(void* const* peer_in_ptrs_dev, void* out, int rank, int world, int64_t n_o, int64_t n_x,
                 int64_t n_m, int64_t row_bytes, int64_t src_stride_o, int64_t src_stride_x, int64_t src_stride_m,
                 int64_t src_base, int64_t dst_stride_o, int64_t dst_stride_x, int64_t dst_stride_m,
                 int64_t dst_peer_stride, xtb_stream_t stream);

/* a14  FSDP all-gather of a flat parameter shard (torch FSDP2 all-gather at model/base.py:714-721, applied per
 * decoder layer model/moe/moe.py:1197-1217), fused with MixedPrecisionPolicy's fp32->bf16 cast
 * (moe.py:1193-1195): rank r writes bf16(local_in[0:n]) at element offset r*n of EVERY rank's output buffer.
 * in_is_f32 = 0: the shard is already bf16 (plain all-gather).  n_local_elems % 8 == 0. */
int xtb_allgather_push(const void* local_in, void* const* peer_out_ptrs_dev, int rank, int world,
                       int64_t n_local_elems, int in_is_f32, xtb_stream_t stream);

/* a14  FSDP reduce-scatter of bf16 gradients (reduce_dtype bf16, config/fsdp.py:36-37) with fp32 accumulation:
 * out[i] = scale * sum_{r=0..world-1} float(in_r[rank*n + i]) in rank order (deterministic), stored as bf16 or
 * fp32.  `scale` carries the data-parallel averaging (1/world) FSDP applies. */
int xtb_reduce_scatter_pull(void* const* peer_in_ptrs_dev, void* out, int rank, int world, int64_t n_local_elems,
                            float scale, int out_is_f32, xtb_stream_t stream);

/* a16  Averaging of the replicated (non-expert) gradients (MoE.scale_and_reduce_grad, model/moe/moe.py:1338-1390: grads /=
 * group size, then one coalesced all-reduce): one-shot all-reduce over peer memory, out[i] = scale * sum_r in_r[i] in fp32,
 * summed in rank order on every rank (bit-identical results on all ranks).  in_r = rank r's flat fp32 buffer in symmetric
 * memory; `out` may be local memory.  n_elems % 4 == 0.  Callers order it between two xtb_peer_barrier calls. */
int xtb_allreduce_pull_f32(void* const* peer_in_ptrs_dev, void* out, int rank, int world, int64_t n_elems, float scale,
                           xtb_stream_t stream);

/* Batch of device-to-device copies between (peer-mapped) addresses on the copy engines — the FSDP engine's XTB_FSDP_DMA
 * mode moves the gathered parameters / gradient slices with it so that no SM is taken from the GEMMs it runs under.
 * All three arrays are HOST arrays of length n; entries with nbytes == 0 or dst == src are skipped.  Every entry is
 * checked before anything is enqueued: a batch with a bad entry is refused without copying any entry. */
int xtb_peer_memcpy_batch(void* const* dst_ptrs_host, const void* const* src_ptrs_host, const int64_t* nbytes_host, int n,
                          xtb_stream_t stream);

/* a10  Expert-parallel token exchange with device-side split sizes (replaces torch_all2all.py:91-114 counts all-to-all +
 * host read + variable-split NCCL all-to-all, and the re-sort by local expert :485-495).  A staging buffer (symmetric
 * memory) = [int32 cnt[E] header, padded to hdr_bytes][rows].  Callers order the calls with xtb_peer_barrier.
 *
 * xtb_ep_write_header: header[e] = (int32) tokens_per_expert[e] of this rank's dispatch (rows sorted by GLOBAL expert).
 * xtb_ep_pull_to_experts: rank `rank` owns experts [rank*E/world, (rank+1)*E/world); pulls their rows from every peer's
 *   source-major staging buffer into `out` grouped by (local expert, source rank), source order kept.  First use of a layer:
 *   cnt_all_in = NULL, the counts are read from the peers' headers and the full table is written to cnt_all_out
 *   [world][E]; later uses (backward of the return trip) pass cnt_all_in.  tokens_per_expert_local[E/world] (int64) and
 *   status[2] = {rows received, 1 if > cap_rows} are optional.  Rows beyond cap_rows are not transferred.
 * xtb_ep_pull_to_sources: the way back — this rank's m_rows permuted rows are fetched from the owners' expert-major
 *   staging buffers (same addressing, inverted). */
int xtb_ep_write_header(const int64_t* tokens_per_expert, void* header, int E, xtb_stream_t stream);
/* host-only (no CUDA call): the (peer rank, row) every output row of the two pull kernels is fetched from, computed with the
 * kernels' own addressing functions from a HOST copy of cnt_all — what the CPU tests check against the reference order. */
int xtb_ep_plan(const int32_t* cnt_all, int rank, int world, int E, int32_t* to_experts, int64_t max_rows_e,
                int32_t* to_sources, int64_t max_rows_s, int64_t* n_rows_e, int64_t* n_rows_s);
int xtb_ep_pull_to_experts(void* const* peer_ptrs_dev, const int32_t* cnt_all_in, int32_t* cnt_all_out, void* out,
                           int64_t* tokens_per_expert_local, int32_t* status, int rank, int world, int E, int64_t row_bytes,
                           int64_t hdr_bytes, int64_t cap_rows, xtb_stream_t stream);
int xtb_ep_pull_to_sources(void* const* peer_ptrs_dev, const int32_t* cnt_all, void* out, int rank, int world, int E,
                           int64_t row_bytes, int64_t hdr_bytes, int64_t cap_rows, int64_t m_rows, xtb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* XTUNER_B200_H_ */
