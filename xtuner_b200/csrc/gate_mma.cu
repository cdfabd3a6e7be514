// a1 + a2 + the index half of a4 in one launch (xtb_gate_route_dispatch); the kernel is in gate_mma.cuh.
#include "gate_mma.cuh"

using namespace xtb;

extern "C" int xtb_gate_route_dispatch(const void* x_bf16, const float* w_f32, int T, int H, int E, int K, int scoring,
                                       int norm_topk_prob, float scaling, float* logits, float* router_weights,
                                       float* topk_weights, int64_t* topk_ids, int32_t* topk_ids_i32,
                                       int64_t* tokens_per_expert, void* dispatch_workspace, xtb_stream_t stream) {
  XTB_CHECK_ARG(x_bf16 && w_f32 && logits && router_weights && topk_weights && topk_ids && topk_ids_i32 &&
                    tokens_per_expert && dispatch_workspace,
                "xtb_gate_route_dispatch: null pointer");
  XTB_CHECK_ARG(T >= 0 && H > 0 && E > 0 && K > 0 && K <= E, "xtb_gate_route_dispatch: bad shape T=%d H=%d E=%d K=%d", T,
                H, E, K);
  XTB_CHECK_ARG(E <= 8 && K <= 8 && H % 128 == 0 && (size_t)48 * H <= 200 * 1024,
                "xtb_gate_route_dispatch: supports E <= 8, H %% 128 == 0, H <= 4224 (got E=%d H=%d); use xtb_gate_logits + "
                "xtb_router_greedy_dispatch",
                E, H);
  XTB_ENSURE_CTX(x_bf16);
  cudaStream_t st = as_stream(stream);
  if (T == 0) {
    XTB_CUDA(cudaMemsetAsync(tokens_per_expert, 0, sizeof(int64_t) * E, st));
    return XTB_OK;
  }
  const int rc = launch_gate_route_mma<false>(static_cast<const __nv_bfloat16*>(x_bf16), w_f32, logits, T, H, E, K,
                                              scoring, norm_topk_prob, scaling, router_weights, topk_weights, topk_ids,
                                              topk_ids_i32, tokens_per_expert, dispatch_workspace, st, nullptr, 0);
  return rc < 0 ? fail(XTB_ERR_INVALID, "xtb_gate_route_dispatch: unsupported shape") : rc;
}
