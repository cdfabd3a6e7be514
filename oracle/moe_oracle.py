"""CPU oracle for the XTuner-V1 MoE hot path.  **TEST INFRASTRUCTURE — NOT PRODUCT CODE.**

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this module.  The product path (``xtuner_b200``) never routes through it and raises if
its CUDA library is missing.

What it is: a restatement, function by function, of the reference's eager algorithm for the path
(SURVEY.md §8a rows a1-a9), written with plain ``torch`` CPU tensor ops because the reference *is* eager
PyTorch: bf16 roundings, fp32 promotions and autograd semantics are then the reference's own by
construction.  Integer/index work (routing ids, histogram, stable order) is exact.  Every function cites
the reference ``file:line`` it follows (paths relative to ``/root/reference``).

Parity pinning: ``tests/golden/make_golden.py`` runs the *reference's own code* (imported from
``/root/reference`` in the authoring container) on seeded inputs and commits the results under
``tests/golden/*.pt``; ``tests/test_oracle_golden.py`` checks this oracle against those vectors and against
the reference's only exact known-answer test for the path (``tests/module/dispatcher/test_noep.py:19-87``).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------------------
# a1  MoEGate.forward  — xtuner/v1/module/decoder_layer/moe_decoder_layer.py:120-141
# --------------------------------------------------------------------------------------------------


def gate_logits(hidden_states: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``router_compute_dtype == "float32"`` branch (moe_decoder_layer.py:138-140):
    ``F.linear(x.float(), W.float(), bias.float())`` on the ``[T, H]`` view of the activations."""
    x = hidden_states.reshape(-1, hidden_states.shape[-1])
    b = bias.float() if bias is not None else None
    return F.linear(x.float(), weight.float(), b)


# --------------------------------------------------------------------------------------------------
# a2  GreedyRouter.forward — xtuner/v1/module/router/greedy.py:64-98
# --------------------------------------------------------------------------------------------------


def tokens_per_expert_hist(topk_ids: torch.Tensor, n_experts: int) -> torch.Tensor:
    """``torch.histc(topk_ids, bins=E, min=0, max=E)`` (greedy.py:90, dispatcher/base.py:398).
    On CUDA histc keeps the int64 dtype of ``topk_ids``; integer bincount is the same arithmetic."""
    return torch.bincount(topk_ids.reshape(-1).to(torch.int64), minlength=n_experts)[:n_experts].to(torch.int64)


def greedy_router(
    logits: torch.Tensor,
    top_k: int,
    norm_topk_prob: bool = True,
    router_scaling_factor: float = 1.0,
    scoring_func: str = "softmax",
) -> Dict[str, torch.Tensor]:
    n_experts = logits.shape[1]
    if scoring_func == "sigmoid":
        routing_weights = logits.sigmoid()  # greedy.py:71
    else:
        routing_weights = F.softmax(logits, dim=1, dtype=torch.float)  # greedy.py:73
    topk_weights, topk_ids = torch.topk(routing_weights, top_k, dim=-1)  # greedy.py:80 (sorted desc)
    if norm_topk_prob:
        topk_weights = topk_weights / topk_weights.sum(dim=-1, keepdim=True)  # greedy.py:82-83 (in-place there)
    if router_scaling_factor != 1.0:
        topk_weights = topk_weights * router_scaling_factor  # greedy.py:85-86
    return {
        "logits": logits,
        "router_weights": routing_weights,
        "topk_weights": topk_weights,
        "topk_ids": topk_ids,
        "topkens_per_expert": tokens_per_expert_hist(topk_ids, n_experts),  # greedy.py:90 (key spelled as there)
    }


# --------------------------------------------------------------------------------------------------
# a2' NoAuxRouter.forward — xtuner/v1/module/router/noaux_router.py:78-150
# --------------------------------------------------------------------------------------------------


def noaux_router(
    logits: torch.Tensor,
    e_score_correction_bias: torch.Tensor,
    top_k: int,
    n_group: int,
    topk_group: int,
    router_scaling_factor: float,
    norm_topk_prob: bool = True,
) -> Dict[str, torch.Tensor]:
    n_tok, n_experts = logits.shape
    scores = logits.sigmoid()  # :80
    scores_for_choice = scores + e_score_correction_bias.unsqueeze(0)  # :85
    if n_group != topk_group:  # :91-113
        group_scores = scores_for_choice.view(n_tok, n_group, -1).topk(2, dim=-1)[0].sum(dim=-1)
        group_idx = torch.topk(group_scores, k=topk_group, dim=-1, sorted=False)[1]
        group_mask = torch.zeros_like(group_scores)
        group_mask.scatter_(1, group_idx, 1)
        score_mask = group_mask.unsqueeze(-1).expand(n_tok, n_group, n_experts // n_group).reshape(n_tok, -1)
        scores_for_choice = scores_for_choice.masked_fill(~score_mask.bool(), 0.0)
    _, topk_ids = torch.topk(scores_for_choice, k=top_k, dim=-1)  # :117
    topk_weight = scores.gather(dim=1, index=topk_ids)  # :125 (unbiased scores)
    router_weights = scores_for_choice / torch.sum(scores_for_choice, dim=-1, keepdim=True)  # :129
    if top_k > 1 and norm_topk_prob:  # :131-133
        topk_weight = topk_weight / (topk_weight.sum(dim=-1, keepdim=True) + 1e-20)
    topk_weight = topk_weight * router_scaling_factor  # :134
    # :137-142 histc on the float view of the ids -> float32 counts
    tpe = tokens_per_expert_hist(topk_ids, n_experts).to(torch.float32)
    return {
        "logits": logits,
        "router_weights": router_weights,
        "topk_weights": topk_weight,
        "topk_ids": topk_ids,
        "topkens_per_expert": tpe,
    }


def noaux_kept_experts(scores_for_choice: torch.Tensor, n_group: int, topk_group: int) -> torch.Tensor:
    """bool [T, E]: the experts whose group ``noaux_router`` keeps (noaux_router.py:91-113), all True when
    ``n_group == topk_group``.  Group score = largest + second largest choice score of the group; groups tied on the
    score are taken lowest index first (what the CUDA kernels do; ``topk(sorted=False)`` leaves the order open)."""
    n_tok, n_experts = scores_for_choice.shape
    if n_group == topk_group:
        return torch.ones_like(scores_for_choice, dtype=torch.bool)
    group_scores = scores_for_choice.view(n_tok, n_group, -1).topk(2, dim=-1)[0].sum(dim=-1)
    order = torch.sort(group_scores, dim=-1, descending=True, stable=True)[1]
    group_mask = torch.zeros_like(group_scores, dtype=torch.bool)
    group_mask.scatter_(1, order[:, :topk_group], True)
    return group_mask.repeat_interleave(n_experts // n_group, dim=1)


def noaux_router_bwd(
    logits: torch.Tensor,
    e_score_correction_bias: torch.Tensor,
    router_weights: torch.Tensor,
    topk_weights: torch.Tensor,
    topk_ids: torch.Tensor,
    grad_topk_weights: Optional[torch.Tensor],
    grad_router_weights: Optional[torch.Tensor],
    has_group_mask: bool,
    router_scaling_factor: float,
    norm_topk_prob: bool = True,
    n_group: Optional[int] = None,
    topk_group: Optional[int] = None,
) -> torch.Tensor:
    """Closed form of what autograd does to ``noaux_router`` (noaux_router.py:80,85,113,125-134): the restatement the
    CUDA backward follows.  With ``n_group`` and ``topk_group`` the group mask is recomputed from logits and bias
    (:func:`noaux_kept_experts`), as the CUDA backward does.  Without them it is read back as ``router_weights != 0``
    (masked choice scores are exactly 0.0 after ``masked_fill``, :113).  That read-back cannot tell a masked expert from
    a kept one whose choice score is exactly 0 (router weight 0, gradient (g - dot) / S), so it raises on such rows
    instead of dropping that gradient."""
    s = torch.sigmoid(logits)
    ds = torch.zeros_like(s)
    if grad_router_weights is not None:
        ch = s + e_score_correction_bias.unsqueeze(0)
        if not has_group_mask:
            mask = torch.ones_like(s, dtype=torch.bool)
        elif n_group is not None and topk_group is not None:
            mask = noaux_kept_experts(ch, n_group, topk_group)
        else:
            mask = router_weights != 0
            if bool(((ch == 0) & ~mask).any()):
                raise ValueError("noaux_router_bwd: a choice score is exactly 0, so router_weights != 0 does not give "
                                 "the group mask; pass n_group and topk_group")
        c = torch.where(mask, s + e_score_correction_bias.unsqueeze(0), torch.zeros_like(s))
        S = c.sum(dim=-1, keepdim=True)
        dot = (grad_router_weights * router_weights).sum(dim=-1, keepdim=True)
        ds = ds + torch.where(mask, (grad_router_weights - dot) / S, torch.zeros_like(s))
    if grad_topk_weights is not None:
        K = topk_ids.shape[1]
        sk = s.gather(1, topk_ids)
        if K > 1 and norm_topk_prob:
            D = sk.sum(dim=-1, keepdim=True) + 1e-20
            gw = (grad_topk_weights * topk_weights).sum(dim=-1, keepdim=True)
            dsk = (router_scaling_factor * grad_topk_weights - gw) / D
        else:
            dsk = router_scaling_factor * grad_topk_weights
        ds = ds.scatter_add(1, topk_ids, dsk)
    return ds * s * (1.0 - s)


# --------------------------------------------------------------------------------------------------
# a4  permute — xtuner/v1/ops/moe/cuda/permute_unpermute.py:205-219 (in-tree torch fallback)
# --------------------------------------------------------------------------------------------------


def permute(input_act: torch.Tensor, indices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Stable sort of the token-major flattened expert ids (flat index ``f = t*K + k``); permuted row
    ``r`` holds token ``sorted_indices[r] // K``.  Returns ``(permuted, sorted_indices)``."""
    topk = 1 if indices.dim() == 1 else indices.size(1)
    flatten_indices = indices.reshape(-1)
    sorted_indices = torch.argsort(flatten_indices, stable=True)  # :215
    permuted_tokens = input_act.index_select(0, sorted_indices // topk)  # :217
    return permuted_tokens, sorted_indices


# --------------------------------------------------------------------------------------------------
# a5  unpermute — xtuner/v1/ops/moe/cuda/permute_unpermute.py:222-248
# --------------------------------------------------------------------------------------------------


def unpermute(input_act: torch.Tensor, row_id_map: torch.Tensor, probs: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``out[t] = dtype( sum_k fp32(probs[t,k]) * act[pos(t,k)] )``; ``row_id_map`` is the
    ``sorted_indices`` returned by :func:`permute` (row -> flat index)."""
    assert row_id_map.numel() == input_act.size(0)  # :227
    if probs is not None:
        num_unpermuted_tokens = probs.numel()
        topk = probs.size(1)
    else:
        num_unpermuted_tokens = input_act.size(0)
        topk = 1
    unpermuted = torch.zeros([num_unpermuted_tokens, input_act.shape[-1]], dtype=input_act.dtype)
    unpermuted = unpermuted.index_put((row_id_map,), input_act, accumulate=False)  # :243 (in-place there)
    unpermuted = unpermuted.reshape(-1, topk, input_act.size(-1))
    if probs is not None:
        unpermuted = unpermuted * probs.unsqueeze(-1)  # :245-246 bf16 * fp32 -> fp32
    unpermuted = unpermuted.sum(dim=1)  # :247
    return unpermuted.to(input_act.dtype)  # :248


# --------------------------------------------------------------------------------------------------
# a6/a7  grouped GEMM — semantic definition used by the reference's own test
#        tests/ops/test_grouped_gemm_triton.py:6-23 (== ops/moe/cuda/triton_kernels/utils.py:79-88)
# --------------------------------------------------------------------------------------------------


def group_gemm(x: torch.Tensor, w: torch.Tensor, tokens_per_expert: torch.Tensor) -> torch.Tensor:
    """``out[rows of expert e] = x[rows of e] @ w[e].T`` with ``w`` of shape ``[E, dout, din]``;
    fp32 accumulation, output rounded to the input dtype (one rounding)."""
    outs: List[torch.Tensor] = []
    start = 0
    for i, n in enumerate(tokens_per_expert.tolist()):
        n = int(n)
        outs.append(torch.matmul(x[start : start + n], w[i].T))
        start += n
    return torch.cat(outs) if outs else x.new_zeros((0, w.shape[1]))


def group_gemm_fp32acc(x: torch.Tensor, w: torch.Tensor, tokens_per_expert: torch.Tensor) -> torch.Tensor:
    """Same product with an explicit fp32 accumulate + single rounding (order-independent yardstick
    for tensor-core kernels, whose summation order differs from the CPU's)."""
    outs, start = [], 0
    for i, n in enumerate(tokens_per_expert.tolist()):
        n = int(n)
        outs.append((x[start : start + n].float() @ w[i].float().T).to(x.dtype))
        start += n
    return torch.cat(outs) if outs else x.new_zeros((0, w.shape[1]))


# --------------------------------------------------------------------------------------------------
# a8  native_swiglu — xtuner/v1/ops/act_fn.py:7-9
# --------------------------------------------------------------------------------------------------


def swiglu(fused_x: torch.Tensor) -> torch.Tensor:
    x1, x2 = torch.chunk(fused_x, 2, dim=-1)
    return F.silu(x1) * x2


# --------------------------------------------------------------------------------------------------
# MoEBlock.forward — moe_decoder_layer.py:196-200 ; GroupedLinear.forward — moe_group_linear.py:162-165
# --------------------------------------------------------------------------------------------------


def experts_forward(
    x_perm: torch.Tensor,
    w13: torch.Tensor,
    w2: torch.Tensor,
    tokens_per_expert: torch.Tensor,
    n_experts: int,
) -> torch.Tensor:
    """``w13`` is the flat ``[E*2I, H]`` parameter, ``w2`` the flat ``[E*H, I]`` parameter
    (moe_group_linear.py:110-114); viewed ``[E, out, in]`` before the grouped GEMM (:163-164)."""
    hidden = x_perm.shape[-1]
    w13v = w13.view(n_experts, -1, hidden)
    inter = w13v.shape[1] // 2
    w2v = w2.view(n_experts, hidden, inter)
    gate_up = group_gemm(x_perm, w13v, tokens_per_expert)
    act = swiglu(gate_up)
    return group_gemm(act, w2v, tokens_per_expert)


# --------------------------------------------------------------------------------------------------
# a3/a9  NaiveDispatcher + MoEDecoderLayer._forward (MoE half) — dispatcher/base.py:378-454,
#        moe_decoder_layer.py:392-488, _post_moe_forward :696-705
# --------------------------------------------------------------------------------------------------


def moe_layer_forward(
    hidden_states: torch.Tensor,  # [T, H] (already post-attention-layernormed), bf16 or fp32
    gate_weight: torch.Tensor,  # [E, H]
    w13: torch.Tensor,  # [E*2I, H]
    w2: torch.Tensor,  # [E*H, I]
    top_k: int,
    norm_topk_prob: bool = True,
    router_scaling_factor: float = 1.0,
    hidden_factor: float = 1.0,
    residual: Optional[torch.Tensor] = None,
    scoring_func: str = "softmax",
) -> Dict[str, torch.Tensor]:
    n_experts = gate_weight.shape[0]
    logits = gate_logits(hidden_states, gate_weight)  # a1
    router = greedy_router(logits, top_k, norm_topk_prob, router_scaling_factor, scoring_func)  # a2
    topk_ids = router["topk_ids"]
    # dispatch_postprocess: base.py:394-398
    x_perm, row_id_map = permute(hidden_states, topk_ids.to(torch.int32))
    tokens_per_expert = tokens_per_expert_hist(topk_ids, n_experts)
    # experts: moe_decoder_layer.py:432-436
    y_perm = experts_forward(x_perm, w13, w2, tokens_per_expert, n_experts)
    # combine_preprocess: base.py:429-433
    combined = unpermute(y_perm, row_id_map, probs=router["topk_weights"])
    out = combined * hidden_factor  # _post_moe_forward :705
    if residual is not None:
        out = out + residual
    return {
        "hidden_states": out,
        "combined": combined,
        "x_perm": x_perm,
        "y_perm": y_perm,
        "row_id_map": row_id_map,
        "tokens_per_expert": tokens_per_expert,
        **{f"router.{k}": v for k, v in router.items()},
    }


# --------------------------------------------------------------------------------------------------
# aux losses that consume router outputs — loss/moe_loss.py:121-170 (balancing), :242-289 (z-loss)
# single-rank restatement (no all-reduce), used only to define "loss parity" for the path
# --------------------------------------------------------------------------------------------------


def balancing_loss(router_weights: torch.Tensor, tokens_per_expert: torch.Tensor, top_k: int, alpha: float = 0.001) -> torch.Tensor:
    n_tok, n_experts = router_weights.shape
    tpe = tokens_per_expert.to(router_weights.dtype)
    mean_w = router_weights.mean(dim=0)
    return alpha * (n_experts / (n_tok * top_k)) * (tpe * mean_w).sum()


def z_loss(logits: torch.Tensor, alpha: float = 0.001) -> torch.Tensor:
    return alpha * (torch.logsumexp(logits.float(), dim=-1) ** 2).mean()


# --------------------------------------------------------------------------------------------------
# a12 ulysses_all_to_all — xtuner/v1/ops/comm/all_to_all.py:6-51, single-process simulation
# --------------------------------------------------------------------------------------------------


def ulysses_all_to_all_sim(inputs: List[torch.Tensor], scatter_dim: int, gather_dim: int) -> List[torch.Tensor]:
    """Given the per-rank inputs of one ``ulysses_all_to_all`` call (``len(inputs) == sp``), return the
    per-rank outputs.  Restates :30-51: split ``scatter_dim`` into ``sp`` equal parts, part ``j`` goes
    to rank ``j``; each rank concatenates what it received, in source-rank order, along ``gather_dim``."""
    world = len(inputs)
    chunks = [torch.tensor_split(x.contiguous(), world, dim=scatter_dim) for x in inputs]
    return [torch.cat([chunks[src][dst] for src in range(world)], dim=gather_dim).contiguous() for dst in range(world)]


# --------------------------------------------------------------------------------------------------
# a15  fp8 (e4m3) tile-wise quantisation used by the fp8 FSDP hooks / grouped GEMM (config 5).
# CUDA kernels for these are NOT built yet; the restatements pin the arithmetic for the next round.
#   EPS, saturating cast ........ xtuner/v1/float8/float8_utils.py:6, :16-32
#   128x128 weight block scales . xtuner/v1/float8/fsdp_utils.py:75-116 (dout >= 128 branch)
#   block cast with given scales  xtuner/v1/float8/fsdp_utils.py:195-223
#   1x128 activation tiles ...... xtuner/v1/float8/triton_kernels/per_tile_quant.py:145-155 (torch reference there)
# --------------------------------------------------------------------------------------------------
FP8_EPS = 1e-12
FP8_DTYPE = torch.float8_e4m3fn


def to_fp8_saturated(x: torch.Tensor, float8_dtype: torch.dtype = FP8_DTYPE) -> torch.Tensor:
    max_value = torch.finfo(float8_dtype).max
    return x.clamp(min=-max_value, max=max_value).to(float8_dtype)


def per_block_fp8_scales(w: torch.Tensor, block_size: int = 128, float8_dtype: torch.dtype = FP8_DTYPE) -> torch.Tensor:
    """``w`` [nw, dout, din] with dout, din multiples of 128 -> scales [nw, dout/128, din/128] (fp32);
    scale = clamp(amax, EPS) / 448 computed through float64 (fsdp_utils.py:106-110)."""
    nw, dout, din = w.shape
    blocks = w.view(nw, dout // block_size, block_size, din // block_size, block_size).transpose(2, 3).reshape(-1, block_size * block_size)
    amax = blocks.abs().amax(-1, True).to(torch.float64)
    scales = (torch.clamp(amax, min=FP8_EPS) / torch.finfo(float8_dtype).max).to(torch.float32)
    return scales.view(nw, dout // block_size, din // block_size).contiguous()


def cast_to_per_block_fp8(w2d: torch.Tensor, scales: torch.Tensor, block_size: int = 128, float8_dtype: torch.dtype = FP8_DTYPE) -> torch.Tensor:
    """``w2d`` [dout, din] (dout >= 128) and its [dout/128, din/128] scales -> e4m3 tensor of the same shape."""
    dout, din = w2d.shape
    t = w2d.view(dout // block_size, block_size, din // block_size, block_size).transpose(1, 2).reshape(-1, block_size * block_size)
    q = to_fp8_saturated(t.to(torch.float32) / scales.reshape(-1, 1), float8_dtype)
    return q.view(dout // block_size, din // block_size, block_size, block_size).transpose(1, 2).reshape(dout, din)


def per_tile_quant(x: torch.Tensor, eps: float = FP8_EPS, float8_dtype: torch.dtype = FP8_DTYPE) -> Tuple[torch.Tensor, torch.Tensor]:
    """activations [M, K] (K % 128 == 0) -> (e4m3 [M, K], scales [M, K/128] fp32), one scale per 1x128 tile."""
    seq, dim = x.shape
    t = x.reshape(-1, 128)
    amax = t.abs().amax(-1, True).to(torch.float64)
    scales = (torch.clamp(amax, min=eps) / torch.finfo(float8_dtype).max).to(torch.float32)
    q = to_fp8_saturated(t.float() / scales, float8_dtype)
    return q.view(seq, dim), scales.view(seq, -1)
