// xtb_gate_route_replay_dispatch: the gate + route + bucketing kernel of gate_mma.cuh with the routing replay step
// (greedy_replay_token).  Its own translation unit: instantiated next to the routing kernel, it changes that kernel's code.
#include "gate_mma.cuh"

using namespace xtb;

extern "C" int xtb_gate_route_replay_dispatch(const void* x_bf16, const float* w_f32, const int64_t* replay_ids,
                                              int64_t replay_row_stride, int T, int H, int E, int K, int scoring,
                                              int norm_topk_prob, float scaling, float* logits, float* router_weights,
                                              float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32,
                                              int64_t* tokens_per_expert, void* dispatch_workspace,
                                              xtb_stream_t stream) {
  XTB_CHECK_ARG(w_f32 && tokens_per_expert && (T == 0 || (x_bf16 && replay_ids && logits && router_weights &&
                                                            topk_weights && topk_ids && topk_ids_i32 && dispatch_workspace)),
                "xtb_gate_route_replay_dispatch: null pointer");
  XTB_CHECK_ARG(T >= 0 && H > 0 && E > 0 && K > 0 && K <= E && replay_row_stride >= K,
                "xtb_gate_route_replay_dispatch: bad shape T=%d H=%d E=%d K=%d stride=%lld", T, H, E, K,
                (long long)replay_row_stride);
  XTB_CHECK_ARG(E <= 8 && K <= 8 && H % 128 == 0 && (size_t)48 * H <= 200 * 1024,
                "xtb_gate_route_replay_dispatch: supports E <= 8, H %% 128 == 0, H <= 4224 (got E=%d H=%d); use "
                "xtb_gate_logits + xtb_router_greedy_replay",
                E, H);
  XTB_ENSURE_CTX(w_f32);
  cudaStream_t st = as_stream(stream);
  if (T == 0) {  // an empty micro-batch: no token arrays to address, only the counts to clear
    XTB_CUDA(cudaMemsetAsync(tokens_per_expert, 0, sizeof(int64_t) * E, st));
    return XTB_OK;
  }
  const int rc = launch_gate_route_mma<true>(static_cast<const __nv_bfloat16*>(x_bf16), w_f32, logits, T, H, E, K,
                                             scoring, norm_topk_prob, scaling, router_weights, topk_weights, topk_ids,
                                             topk_ids_i32, tokens_per_expert, dispatch_workspace, st, replay_ids,
                                             replay_row_stride);
  return rc < 0 ? fail(XTB_ERR_INVALID, "xtb_gate_route_replay_dispatch: unsupported shape") : rc;
}
