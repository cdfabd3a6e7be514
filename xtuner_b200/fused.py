"""Fused MoE layer: the whole MoE half of ``MoEDecoderLayer._forward`` (reference
``module/decoder_layer/moe_decoder_layer.py:392-488`` + ``_post_moe_forward`` :696-705) as ONE autograd node
that drives the C-ABI kernels directly:

forward   gate GEMM (fp32) -> router (softmax/top-k/renorm/histogram) -> bucket+gather (dispatch)
          -> grouped GEMM w13 with the SwiGLU in its epilogue -> grouped GEMM w2
          -> combine (x prob, sum over k) + hidden_factor + residual in one pass
backward  combine-bwd -> dX/dW grouped GEMMs (w2) -> SwiGLU-bwd -> dX/dW grouped GEMMs (w13)
          -> router-bwd (three gradient routes) -> gate-bwd -> dispatch-bwd fused with the gate-grad add

``recompute`` trades time for memory in the expert half (see :data:`RECOMPUTE`): the node keeps fewer of its four
``[T*K, .]`` intermediates and rebuilds them in the backward from ``x`` and the routing it keeps anyway.  Every kernel
on that path is deterministic, so the gradients are the saved path's, bit for bit.

One Python frame and ~20 kernel launches per layer instead of ~40 dispatcher/custom-op calls: the path is
launch-bound in eager mode otherwise.  Numerics are identical to composing
``xtuner_b200.ops`` (same kernels); the per-op bf16 roundings of the reference are kept (see kernel notes).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor, nn

from . import _capi, ops
from ._capi import check, current_stream, ptr
from .router import SCORING, replay_ids_arg

# Where the next expert-weight gradients are written: a callable returning ``(g_w13_buffer, g_w2_buffer)`` (bf16, same
# numel as the weights) or None.  The FSDP engine (fsdp_experts.py) points this at its symmetric gradient buffers so the
# dW grouped GEMMs write straight into the memory the reduce-scatter pulls from (no copy-in).
GRAD_SINK = None


def _weight_grad_buffers(w13: Tensor, w2: Tensor):
    sink = GRAD_SINK() if GRAD_SINK is not None else None
    if sink is not None:
        b13, b2 = sink
        if (b13.numel() == w13.numel() and b2.numel() == w2.numel() and b13.dtype == w13.dtype and b2.dtype == w2.dtype
                and b13.device == w13.device and b13.is_contiguous() and b2.is_contiguous()):
            return b13.view_as(w13), b2.view_as(w2)
    return torch.empty_like(w13), torch.empty_like(w2)


def _gate_route(lib, x, gate_w, T, H, E, K, scoring, norm, scaling, st, replay=None):
    """(logits, rw, tw, ids, ids32, tpe, ws): gate, greedy router and dispatch bucketing into the permute workspace ``ws``.
    One launch (xtb_gate_route_dispatch: gate on the tensor cores) where E <= 8, K <= 8, H % 128 == 0 and H <= 4096, the
    gate and the router as two calls otherwise (their A/B at the shapes both take has not been repeated on H100).  With
    ``replay`` (rollout-routed experts, int64 [T, K]) the replay entries of the same two paths gather the weights at those
    ids instead of a top-k."""
    dev = x.device
    logits = torch.empty((T, E), dtype=torch.float32, device=dev)
    rw = torch.empty((T, E), dtype=torch.float32, device=dev)
    tw = torch.empty((T, K), dtype=torch.float32, device=dev)
    ids = torch.empty((T, K), dtype=torch.int64, device=dev)
    ids32 = torch.empty((T, K), dtype=torch.int32, device=dev)
    tpe = torch.empty((E,), dtype=torch.int64, device=dev)
    ws = ops.permute_workspace(T, K, E, dev)
    one_launch = E <= 8 and K <= 8 and H % 128 == 0 and H <= 4096
    if replay is not None:
        rp, stride = replay_ids_arg(replay, T, K, dev)
        if one_launch:
            _k(lib, "xtb_gate_route_replay_dispatch", ptr(x), ptr(gate_w), ptr(rp), stride, T, H, E, K, scoring, int(norm),
               float(scaling), ptr(logits), ptr(rw), ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), ptr(ws), st)
        else:
            _k(lib, "xtb_gate_logits", ptr(x), ptr(gate_w), None, ptr(logits), T, H, E, st)
            _k(lib, "xtb_router_greedy_replay", ptr(logits), ptr(rp), stride, T, E, K, scoring, int(norm), float(scaling),
               ptr(rw), ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), ptr(ws), st)
    elif one_launch:
        _k(lib, "xtb_gate_route_dispatch", ptr(x), ptr(gate_w), T, H, E, K, scoring, int(norm), float(scaling),
           ptr(logits), ptr(rw), ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), ptr(ws), st)
    else:
        _k(lib, "xtb_gate_logits", ptr(x), ptr(gate_w), None, ptr(logits), T, H, E, st)
        _k(lib, "xtb_router_greedy_dispatch", ptr(logits), T, E, K, scoring, int(norm), float(scaling), ptr(rw), ptr(tw),
           ptr(ids), ptr(ids32), ptr(tpe), ptr(ws), st)
    return logits, rw, tw, ids, ids32, tpe, ws


def _router_gate_bwd(lib, rw, tw, ids, g_tw, g_rw, g_lg, x, gate_w, T, H, E, K, scoring, norm, scaling, st):
    """(grad_gate_w, grad_x_gate): router backward followed by the gate backward, in one launch (xtb_router_gate_bwd: the
    router backward in the prologue of the gate backward) where E <= 8 and H % 8 == 0, in two otherwise."""
    dev = x.device
    g_gate_w = torch.empty_like(gate_w)
    g_x_gate = torch.empty((T, H), dtype=torch.bfloat16, device=dev)
    wsb = ops._scratch("gate_bwd", int(lib.xtb_gate_logits_bwd_workspace_bytes(T, H, E)), dev)
    g_rw_c = None if g_rw is None else g_rw.contiguous()
    g_lg_c = None if g_lg is None else g_lg.contiguous()
    if E <= 8 and H % 8 == 0:
        _k(lib, "xtb_router_gate_bwd", ptr(rw), ptr(tw), ptr(ids), ptr(g_tw), ptr(g_rw_c), ptr(g_lg_c), ptr(x), ptr(gate_w),
           ptr(g_gate_w), ptr(g_x_gate), T, H, E, K, scoring, int(norm), float(scaling), ptr(wsb), st)
        return g_gate_w, g_x_gate
    g_l = torch.empty((T, E), dtype=torch.float32, device=dev)
    _k(lib, "xtb_router_greedy_bwd", ptr(rw), ptr(tw), ptr(ids), ptr(g_tw), ptr(g_rw_c), ptr(g_lg_c), T, E, K, scoring,
       int(norm), float(scaling), ptr(g_l), st)
    _k(lib, "xtb_gate_logits_bwd", ptr(g_l), ptr(x), ptr(gate_w), ptr(g_gate_w), ptr(g_x_gate), None, T, H, E, ptr(wsb), st)
    return g_gate_w, g_x_gate


def _no_tokens(ctx, x: Tensor, gate_w: Tensor, K: int):
    """Forward outputs of a node given no tokens (T = 0), with no launch: the kernels take no null pointers, and an empty
    tensor has none.  Its backward returns empty / zero gradients (:func:`_no_token_grads`)."""
    ctx.no_tokens = True
    E, dev = gate_w.shape[0], x.device
    ids = torch.empty((0, K), dtype=torch.int64, device=dev)
    tpe = torch.zeros((E,), dtype=torch.int64, device=dev)
    ctx.mark_non_differentiable(ids, tpe)
    lg = torch.empty((0, E), dtype=torch.float32, device=dev)
    return torch.empty_like(x), lg, lg.clone(), ids, tpe


def _no_token_grads(gate_w: Tensor, w13: Tensor, w2: Tensor):
    """(g_gate_w, g_w13, g_w2) of a node given no tokens: zeros, the expert ones in the GRAD_SINK buffers if set."""
    g_w13, g_w2 = _weight_grad_buffers(w13, w2)
    return torch.zeros_like(gate_w), g_w13.zero_(), g_w2.zero_()


# What a fused node may recompute in its backward instead of saving from its forward (the user's memory-for-time choice):
#   None       save x_perm, h, a and y (the default)
#   "act"      save neither x_perm nor a: x_perm is permuted again from x after the dX GEMM of w13, a comes out of the
#              SwiGLU backward (xtb_swiglu_bwd_act); no GEMM runs again
#   "experts"  save none of the four: the backward first reruns the permute and both expert GEMMs of the forward
RECOMPUTE = (None, "act", "experts")


def _check_recompute(entry: str, recompute) -> None:
    if recompute not in RECOMPUTE:
        raise ValueError(f"{entry}: recompute must be None, 'act' or 'experts' (got {recompute!r})")


# Optional profiling: when a list, every kernel call is bracketed by CUDA events on the current stream
# and (name, start, end) is appended.  bench.py uses this to time kernels inside the timed region.
PROFILE: Optional[list] = None


def _k(lib, name: str, *args) -> None:
    if PROFILE is None:
        check(getattr(lib, name)(*args), name)
        return
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    check(getattr(lib, name)(*args), name)
    e.record()
    PROFILE.append((name, s, e))


def _moe_forward(ctx, lib, st, x, residual, gate_w, w13, w2, K, norm, scaling, hidden_factor, scoring, replay,
                 recompute):
    """Gate and route through the combine, ``out = moe(x) * hidden_factor + residual``, for both nodes.  Returns the
    node's outputs ``(out, logits, rw, ids, tpe)`` and the 14 tensors :func:`_moe_backward` reads, in that order; those
    ``recompute`` rebuilds in the backward are None, and so is the last one, ids32, when nothing is rebuilt."""
    T, H = x.shape
    E = gate_w.shape[0]
    I = w2.shape[-1]
    M = T * K
    dev = x.device
    bf = torch.bfloat16
    logits, rw, tw, ids, ids32, tpe, ws = _gate_route(lib, x, gate_w, T, H, E, K, scoring, norm, scaling, st, replay)

    x_perm = torch.empty((M, H), dtype=bf, device=dev)
    row_id_map = torch.empty((M,), dtype=torch.int32, device=dev)
    _k(lib, "xtb_moe_permute_prepared", ptr(x), ptr(ids32), T, K, E, H * 2, ptr(x_perm), ptr(row_id_map), None, ptr(ws), st)

    h = torch.empty((M, 2 * I), dtype=bf, device=dev)
    a = torch.empty((M, I), dtype=bf, device=dev)
    _k(lib, "xtb_group_gemm_nt_swiglu", ptr(x_perm), ptr(w13), ptr(tpe), M, I, H, E, ptr(h), ptr(a), st)

    y = torch.empty((M, H), dtype=bf, device=dev)
    _k(lib, "xtb_group_gemm_nt", ptr(a), ptr(w2), ptr(tpe), M, H, I, E, ptr(y), st)

    out = torch.empty((T, H), dtype=bf, device=dev)
    _k(lib, "xtb_moe_combine", ptr(y), ptr(row_id_map), ptr(tw), ptr(residual), float(hidden_factor), T, K, H, ptr(out), st)

    ctx.mark_non_differentiable(ids, tpe)
    if recompute == "act":
        x_perm = a = None
    elif recompute == "experts":
        x_perm = h = a = y = None
    else:
        ids32 = None
    return (out, logits, rw, ids, tpe), (x, gate_w, w13, w2, rw, tw, ids, row_id_map, tpe, x_perm, h, a, y, ids32)


def _permute_again(lib, x, ids32, T, K, E, H, st):
    """x_perm of the forward, from x and its int32 expert ids: the permute is a stable counting sort, so every row lands
    where the forward put it.  The row map it writes again is not needed (the saved one is the same)."""
    x_perm = torch.empty((T * K, H), dtype=torch.bfloat16, device=x.device)
    row_id_map = torch.empty((T * K,), dtype=torch.int32, device=x.device)
    _k(lib, "xtb_moe_permute", ptr(x), ptr(ids32), T, K, E, H * 2, ptr(x_perm), ptr(row_id_map), None, None,
       ptr(ops.permute_workspace(T, K, E, x.device)), st)
    return x_perm


def _moe_backward(lib, st, saved, cfg, recompute, g_out, g_logits, g_rw):
    """From the combine backward through the router and gate backward, for both nodes: ``saved`` holds the 14 tensors
    of :func:`_moe_forward` under the same ``recompute``, ``cfg`` starts with (K, norm, scaling, hidden_factor, scoring),
    ``g_out`` is contiguous.  Returns ``(g_xp, g_x_gate, g_gate_w, g_w13, g_w2)``; the node's last launch sums each
    token's K rows of g_xp and adds g_x_gate."""
    x, gate_w, w13, w2, rw, tw, ids, row_id_map, tpe, x_perm, h, a, y, ids32 = saved
    K, norm, scaling, hidden_factor, scoring = cfg[:5]
    T, H = x.shape
    E = gate_w.shape[0]
    I = w2.shape[-1]
    M = T * K
    dev = x.device
    bf, f32 = torch.bfloat16, torch.float32
    if recompute == "experts":  # the forward's expert half again, up to y
        x_perm = _permute_again(lib, x, ids32, T, K, E, H, st)
        h = torch.empty((M, 2 * I), dtype=bf, device=dev)
        a = torch.empty((M, I), dtype=bf, device=dev)
        _k(lib, "xtb_group_gemm_nt_swiglu", ptr(x_perm), ptr(w13), ptr(tpe), M, I, H, E, ptr(h), ptr(a), st)
        y = torch.empty((M, H), dtype=bf, device=dev)
        _k(lib, "xtb_group_gemm_nt", ptr(a), ptr(w2), ptr(tpe), M, H, I, E, ptr(y), st)
    g_comb = g_out if hidden_factor == 1.0 else (g_out * hidden_factor)

    g_y = torch.empty((M, H), dtype=bf, device=dev)
    g_tw = torch.empty((T, K), dtype=f32, device=dev)
    _k(lib, "xtb_moe_unpermute_bwd", ptr(g_comb), ptr(y), ptr(row_id_map), ptr(tw), T, K, H, ptr(g_y), ptr(g_tw), st)
    y = None  # a rebuilt y is freed here; a saved one lives on in ctx

    g_w13, g_w2 = _weight_grad_buffers(w13, w2)
    g_a = torch.empty((M, I), dtype=bf, device=dev)
    _k(lib, "xtb_group_gemm_nn", ptr(g_y), ptr(w2), ptr(tpe), M, H, I, E, ptr(g_a), st)
    g_h = torch.empty((M, 2 * I), dtype=bf, device=dev)
    if recompute == "act":
        a = torch.empty((M, I), dtype=bf, device=dev)
        _k(lib, "xtb_swiglu_bwd_act", ptr(g_a), ptr(h), ptr(g_h), ptr(a), M, I, st)
    else:
        _k(lib, "xtb_swiglu_bwd", ptr(g_a), ptr(h), ptr(g_h), M, I, st)
    h = None  # a rebuilt h is freed here

    g_xp = torch.empty((M, H), dtype=bf, device=dev)
    _k(lib, "xtb_group_gemm_nn", ptr(g_h), ptr(w13), ptr(tpe), M, 2 * I, H, E, ptr(g_xp), st)
    if recompute == "act":  # only now: x_perm is not held across the two dX GEMMs
        x_perm = _permute_again(lib, x, ids32, T, K, E, H, st)
    # both weight gradients in one launch: one tile list over the two products fills the persistent schedule's last wave
    _k(lib, "xtb_group_gemm_tn_pair", ptr(g_y), ptr(a), H, I, ptr(g_w2), ptr(g_h), ptr(x_perm), 2 * I, H, ptr(g_w13),
       ptr(tpe), M, E, st)

    g_gate_w, g_x_gate = _router_gate_bwd(lib, rw, tw, ids, g_tw, g_rw, g_logits, x, gate_w, T, H, E, K, scoring, norm,
                                          scaling, st)
    return g_xp, g_x_gate, g_gate_w, g_w13, g_w2


_ROW_ID_MAP = 7  # where row_id_map sits among the 14 tensors of _moe_forward: the node's last launch reads it


class FusedMoEFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, residual: Optional[Tensor], gate_w: Tensor, w13: Tensor, w2: Tensor, top_k: int,
                norm_topk_prob: bool, scaling: float, hidden_factor: float, scoring: int,
                rollout_routed_experts: Optional[Tensor] = None, recompute: Optional[str] = None):
        lib = _capi.ensure_init()
        st = current_stream()
        if x.shape[0] == 0:
            ctx.save_for_backward(gate_w, w13, w2)
            ctx.has_res = residual is not None
            return _no_tokens(ctx, x, gate_w, top_k)
        outputs, saved = _moe_forward(ctx, lib, st, x, residual, gate_w, w13, w2, top_k, norm_topk_prob, scaling,
                                      hidden_factor, scoring, rollout_routed_experts, recompute)
        ctx.save_for_backward(*saved)
        ctx.cfg = (top_k, norm_topk_prob, scaling, hidden_factor, scoring, residual is not None)
        ctx.recompute = recompute
        return outputs

    @staticmethod
    def backward(ctx, g_out, g_logits, g_rw, _g_ids, _g_tpe):
        if getattr(ctx, "no_tokens", False):
            return (torch.empty_like(g_out), g_out if ctx.has_res else None, *_no_token_grads(*ctx.saved_tensors),
                    None, None, None, None, None, None, None)
        lib = _capi.ensure_init()
        st = current_stream()
        saved = ctx.saved_tensors
        K, has_res = ctx.cfg[0], ctx.cfg[5]
        g_out = g_out.contiguous()
        g_xp, g_x_gate, g_gate_w, g_w13, g_w2 = _moe_backward(lib, st, saved, ctx.cfg, ctx.recompute, g_out, g_logits,
                                                              g_rw)

        # dispatch backward (sum of the K copies' grads) fused with "+ gate-path grad" (autograd's add)
        T, H = g_x_gate.shape
        g_x = torch.empty_like(g_x_gate)
        _k(lib, "xtb_moe_combine", ptr(g_xp), ptr(saved[_ROW_ID_MAP]), None, ptr(g_x_gate), 1.0, T, K, H, ptr(g_x), st)
        return g_x, g_out if has_res else None, g_gate_w, g_w13, g_w2, None, None, None, None, None, None, None


class FusedMoEBlockFunction(torch.autograd.Function):
    """MoE half of the decoder layer INCLUDING its RMSNorm and residual
    (``_pre_moe_forward``'s post_attention_layernorm + gate, the dispatcher/experts, ``_post_moe_forward``;
    moe_decoder_layer.py:664-705): ``out = moe(rms_norm(h)) * hidden_factor + h`` as one autograd node."""

    @staticmethod
    def forward(ctx, h: Tensor, norm_w: Tensor, eps: float, gate_w: Tensor, w13: Tensor, w2: Tensor, top_k: int,
                norm_topk_prob: bool, scaling: float, hidden_factor: float, scoring: int,
                rollout_routed_experts: Optional[Tensor] = None, recompute: Optional[str] = None):
        lib = _capi.ensure_init()
        st = current_stream()
        T, H = h.shape
        if T == 0:
            ctx.save_for_backward(norm_w, gate_w, w13, w2)
            return _no_tokens(ctx, h, gate_w, top_k)
        E = gate_w.shape[0]
        x = torch.empty((T, H), dtype=torch.bfloat16, device=h.device)
        rstd = torch.empty((T,), dtype=torch.float32, device=h.device)
        # the norm as its own streaming kernel: folding the gate into it (xtb_rmsnorm_gate with gate_w) is not used by
        # the fused layer (not measured on H100)
        _k(lib, "xtb_rmsnorm_gate", ptr(h), ptr(norm_w), None, float(eps), T, H, E, ptr(x), ptr(rstd), None, st)
        outputs, saved = _moe_forward(ctx, lib, st, x, h, gate_w, w13, w2, top_k, norm_topk_prob, scaling, hidden_factor,
                                      scoring, rollout_routed_experts, recompute)
        ctx.save_for_backward(h, norm_w, rstd, *saved)
        ctx.cfg = (top_k, norm_topk_prob, scaling, hidden_factor, scoring)
        ctx.recompute = recompute
        return outputs

    @staticmethod
    def backward(ctx, g_out, g_logits, g_rw, _g_ids, _g_tpe):
        if getattr(ctx, "no_tokens", False):
            norm_w, gate_w, w13, w2 = ctx.saved_tensors
            g_norm_w = torch.zeros_like(norm_w) if ctx.needs_input_grad[1] else None
            return (torch.empty_like(g_out), g_norm_w, None, *_no_token_grads(gate_w, w13, w2), None, None, None, None,
                    None, None, None)
        lib = _capi.ensure_init()
        st = current_stream()
        h, norm_w, rstd, *saved = ctx.saved_tensors
        K = ctx.cfg[0]
        g_out = g_out.contiguous()
        g_xp, g_x_gate, g_gate_w, g_w13, g_w2 = _moe_backward(lib, st, saved, ctx.cfg, ctx.recompute, g_out, g_logits,
                                                              g_rw)

        T, H = h.shape
        g_h = torch.empty_like(g_x_gate)
        g_norm_w = wsn = None
        if ctx.needs_input_grad[1]:
            g_norm_w = torch.empty_like(norm_w)
            wsn = ops._scratch("norm_bwd", int(lib.xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(T, H)), h.device)
        _k(lib, "xtb_moe_dispatch_bwd_rmsnorm", ptr(g_xp), ptr(saved[_ROW_ID_MAP]), ptr(g_x_gate), ptr(h), ptr(rstd),
           ptr(norm_w), ptr(g_out), T, K, H, ptr(g_h), ptr(g_norm_w), ptr(wsn), st)
        return g_h, g_norm_w, None, g_gate_w, g_w13, g_w2, None, None, None, None, None, None, None


_FUSED_NORM_H = (256, 512, 1024, 2048)


def _fp32_gate(entry: str, x: Tensor, gate_weight: Tensor, w13: Tensor, w2: Tensor) -> Tensor:
    """The gate weight in fp32, once ``entry``'s activations and expert weights have passed its checks."""
    if not x.is_cuda:
        raise _capi.XtbError(f"{entry} needs CUDA tensors (no CPU fallback)")
    if x.dtype != torch.bfloat16 or w13.dtype != torch.bfloat16 or w2.dtype != torch.bfloat16:
        raise TypeError(f"{entry}: activations and expert weights must be bfloat16")
    return gate_weight if gate_weight.dtype == torch.float32 else gate_weight.float()


def _router_results(logits: Tensor, rw: Tensor, ids: Tensor, tpe: Tensor) -> dict:
    """The reference's RouterResults of a fused node (topk_weights stay inside the node)."""
    return {"logits": logits, "router_weights": rw, "topk_weights": None, "topk_ids": ids, "topkens_per_expert": tpe}


def fused_moe_block(h: Tensor, norm_weight: Tensor, eps: float, gate_weight: Tensor, w13: Tensor, w2: Tensor, *, top_k: int,
                    norm_topk_prob: bool = True, router_scaling_factor: float = 1.0, hidden_factor: float = 1.0,
                    scoring_func: str = "softmax", rollout_routed_experts: Optional[Tensor] = None,
                    recompute: Optional[str] = None):
    """``h`` [T,H] bf16 residual stream -> ``moe(rms_norm(h, norm_weight, eps)) * hidden_factor + h``.
    Supported H for the fused backward: 256/512/1024/2048.  ``rollout_routed_experts`` (int64 [T, top_k], on h's device):
    route those experts instead of the router's top-k (RL routing replay).  ``recompute`` (None, "act" or "experts", see
    :data:`RECOMPUTE`): which expert intermediates the backward rebuilds instead of keeping them from the forward; the
    results do not change.  Returns ``(hidden_states, router_results)``."""
    _check_recompute("fused_moe_block", recompute)
    gw = _fp32_gate("fused_moe_block", h, gate_weight, w13, w2)
    shape = h.shape
    if shape[-1] not in _FUSED_NORM_H:
        # the fused norm kernels keep the row slice in registers (xtb_rmsnorm_gate: H in 256/512/1024/2048): compose instead
        x = torch.nn.functional.rms_norm(h, (shape[-1],), norm_weight.to(h.dtype), eps)
        return fused_moe(x, h, gw, w13, w2, top_k=top_k, norm_topk_prob=norm_topk_prob,
                         router_scaling_factor=router_scaling_factor, hidden_factor=hidden_factor, scoring_func=scoring_func,
                         rollout_routed_experts=rollout_routed_experts, recompute=recompute)
    h2 = h.contiguous().view(-1, shape[-1])
    nw = norm_weight if norm_weight.dtype == torch.float32 else norm_weight.float()
    out, *rr = FusedMoEBlockFunction.apply(
        h2, nw.contiguous(), eps, gw.contiguous(), w13.contiguous(), w2.contiguous(), top_k, norm_topk_prob,
        router_scaling_factor, hidden_factor, SCORING[scoring_func], rollout_routed_experts, recompute)
    return out.view(shape), _router_results(*rr)


def fused_moe(x: Tensor, residual: Optional[Tensor], gate_weight: Tensor, w13: Tensor, w2: Tensor, *, top_k: int,
              norm_topk_prob: bool = True, router_scaling_factor: float = 1.0, hidden_factor: float = 1.0,
              scoring_func: str = "softmax", rollout_routed_experts: Optional[Tensor] = None,
              recompute: Optional[str] = None):
    """``x`` [T,H] bf16 (post-attention-layernorm activations), ``residual`` [T,H] bf16 or None,
    ``gate_weight`` [E,H] (used in fp32), ``w13`` [E*2I,H] or [E,2I,H], ``w2`` [E*H,I] or [E,H,I] (bf16),
    ``rollout_routed_experts`` int64 [T, top_k] or None (RL routing replay), ``recompute`` None, "act" or "experts" (both
    as in :func:`fused_moe_block`).  Returns ``(hidden_states, router_results)`` with the reference's RouterResults keys."""
    _check_recompute("fused_moe", recompute)
    gw = _fp32_gate("fused_moe", x, gate_weight, w13, w2)
    shape = x.shape
    x2 = x.contiguous().view(-1, shape[-1])
    res2 = None if residual is None else residual.contiguous().view(-1, shape[-1])
    out, *rr = FusedMoEFunction.apply(
        x2, res2, gw.contiguous(), w13.contiguous(), w2.contiguous(), top_k, norm_topk_prob, router_scaling_factor,
        hidden_factor, SCORING[scoring_func], rollout_routed_experts, recompute)
    return out.view(shape), _router_results(*rr)


def _add_gate_and_experts(mod: nn.Module, hidden_size: int, moe_intermediate_size: int, n_routed_experts: int,
                          num_experts_per_tok: int, norm_topk_prob: bool, router_scaling_factor: float,
                          hidden_factor: float) -> None:
    """The routing settings and the ``gate`` / ``experts`` submodules both fused modules register, named as in
    :class:`xtuner_b200.moe.MoELayer`."""
    from .moe import MoEBlock, MoEGate

    mod.top_k, mod.norm_topk_prob = num_experts_per_tok, norm_topk_prob
    mod.router_scaling_factor, mod.hidden_factor = router_scaling_factor, hidden_factor
    mod.gate = MoEGate(hidden_size=hidden_size, n_routed_experts=n_routed_experts, num_experts_per_tok=num_experts_per_tok,
                       norm_topk_prob=norm_topk_prob, router_scaling_factor=router_scaling_factor)
    mod.experts = MoEBlock(hidden_size=hidden_size, moe_intermediate_size=moe_intermediate_size,
                           n_routed_experts=n_routed_experts)


class FusedMoEBlock(nn.Module):
    """``post_attention_layernorm`` + MoE + residual; parameters named as in the reference's decoder layer:
    ``post_attention_layernorm.weight``, ``gate.weight``, ``experts.fused_w1w3.weight``, ``experts.fused_w2.weight``.
    ``recompute``: as in :func:`fused_moe_block`."""

    def __init__(self, *, hidden_size: int, moe_intermediate_size: int, n_routed_experts: int, num_experts_per_tok: int,
                 rms_norm_eps: float = 1e-6, norm_topk_prob: bool = True, router_scaling_factor: float = 1.0,
                 hidden_factor: float = 1.0, recompute: Optional[str] = None):
        super().__init__()
        _check_recompute("FusedMoEBlock", recompute)
        self.eps = rms_norm_eps
        self.recompute = recompute
        self.post_attention_layernorm = nn.Module()
        self.post_attention_layernorm.weight = nn.Parameter(torch.ones(hidden_size))
        _add_gate_and_experts(self, hidden_size, moe_intermediate_size, n_routed_experts, num_experts_per_tok,
                              norm_topk_prob, router_scaling_factor, hidden_factor)

    def forward(self, hidden_states: Tensor):
        return fused_moe_block(hidden_states, self.post_attention_layernorm.weight, self.eps, self.gate.weight,
                               self.experts.fused_w1w3.weight, self.experts.fused_w2.weight, top_k=self.top_k,
                               norm_topk_prob=self.norm_topk_prob, router_scaling_factor=self.router_scaling_factor,
                               hidden_factor=self.hidden_factor, recompute=self.recompute)


class FusedMoELayer(nn.Module):
    """Same parameters / state-dict keys as :class:`xtuner_b200.moe.MoELayer` (and therefore as the
    reference's ``gate.weight``, ``experts.fused_w1w3.weight``, ``experts.fused_w2.weight``).  ``recompute``: as in
    :func:`fused_moe_block`."""

    def __init__(self, *, hidden_size: int, moe_intermediate_size: int, n_routed_experts: int, num_experts_per_tok: int,
                 norm_topk_prob: bool = True, router_scaling_factor: float = 1.0, hidden_factor: float = 1.0,
                 recompute: Optional[str] = None):
        super().__init__()
        _check_recompute("FusedMoELayer", recompute)
        self.recompute = recompute
        _add_gate_and_experts(self, hidden_size, moe_intermediate_size, n_routed_experts, num_experts_per_tok,
                              norm_topk_prob, router_scaling_factor, hidden_factor)

    def forward(self, hidden_states: Tensor, residual: Tensor | None = None):
        return fused_moe(hidden_states, residual, self.gate.weight, self.experts.fused_w1w3.weight,
                         self.experts.fused_w2.weight, top_k=self.top_k, norm_topk_prob=self.norm_topk_prob,
                         router_scaling_factor=self.router_scaling_factor, hidden_factor=self.hidden_factor,
                         recompute=self.recompute)
