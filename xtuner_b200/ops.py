"""Host-side mirror of the reference's MoE op protocols (``xtuner/v1/ops/moe/protocol.py:6-30``),
backed by the sm_90a C-ABI library.  Same names, argument meaning and error behaviour as the reference's
``xtuner.v1.ops.{permute, unpermute, group_gemm}`` and ``xtuner.v1.ops.act_fn.native_swiglu``:

* autograd-aware (``torch.autograd.Function`` over ``torch.library.custom_op`` kernels with fake
  implementations, the same layering as ``ops/moe/cuda/permute_unpermute.py:18-89``), so they survive
  ``torch.compile(fullgraph=True)`` (``model/moe/moe.py:84-98``);
* ``tokens_per_expert`` stays a device int64 tensor (no host read);
* zero-token inputs still join the autograd graph (``ops/moe/cuda/group_gemm.py:34-36``).

There is no fallback: every op raises if the CUDA library is missing or the tensors are not on an H100.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _capi
from ._capi import check, current_stream, ptr

__all__ = ["permute", "unpermute", "group_gemm", "swiglu", "gate_logits", "permute_workspace", "lm_head_cross_entropy",
           "lm_head_logprobs", "qk_norm_rope", "moe_aux_stats"]


def _require_cuda(*tensors: Tensor) -> None:
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _capi.XtbError(
                "xtuner_b200 ops run on CUDA tensors only (there is no CPU fallback); got a tensor on " + str(t.device)
            )


def _bf16(t: Tensor, name: str) -> None:
    if t.dtype != torch.bfloat16:
        raise TypeError(f"{name} must be bfloat16 (got {t.dtype})")


# per-device cached workspaces (stream-ordered reuse is safe: kernels of one stream execute in order)
_workspaces: dict = {}


def permute_workspace(T: int, K: int, E: int, device) -> Tensor:
    lib = _capi.load()
    need = int(lib.xtb_moe_permute_workspace_bytes(T, K, E))
    key = ("permute", device, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(max(need, 1 << 16), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def _scratch(tag: str, nbytes: int, device) -> Tensor:
    key = (tag, device, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


# ======================================================================================================
# raw kernels as custom ops (fake impls make them traceable)
# ======================================================================================================


@torch.library.custom_op("xtuner_b200::permute", mutates_args=())
def _permute_op(input_act: Tensor, indices: Tensor, n_experts: int) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (permuted [T*K,H], row_id_map int32 [T*K] (flat->row), sorted_indices int64 [T*K] (row->flat),
    tokens_per_expert int64 [E])"""
    lib = _capi.ensure_init()
    T, K = indices.shape
    H = input_act.shape[1]
    dev = input_act.device
    permuted = torch.empty((T * K, H), dtype=input_act.dtype, device=dev)
    row_id_map = torch.empty((T * K,), dtype=torch.int32, device=dev)
    sorted_indices = torch.empty((T * K,), dtype=torch.int64, device=dev)
    tpe = torch.empty((n_experts,), dtype=torch.int64, device=dev)
    ws = permute_workspace(T, K, n_experts, dev)
    check(
        lib.xtb_moe_permute(
            ptr(input_act), ptr(indices), T, K, n_experts, H * input_act.element_size(), ptr(permuted),
            ptr(row_id_map), ptr(sorted_indices), ptr(tpe), ptr(ws), current_stream(),
        ),
        "xtb_moe_permute",
    )
    return permuted, row_id_map, sorted_indices, tpe


@_permute_op.register_fake
def _(input_act, indices, n_experts):
    T, K = indices.shape
    return (
        input_act.new_empty((T * K, input_act.shape[1])),
        indices.new_empty((T * K,), dtype=torch.int32),
        indices.new_empty((T * K,), dtype=torch.int64),
        indices.new_empty((n_experts,), dtype=torch.int64),
    )


@torch.library.custom_op("xtuner_b200::unpermute", mutates_args=())
def _unpermute_op(input_act: Tensor, row_id_map: Tensor, probs: Optional[Tensor], num_tokens: int, topk: int) -> Tensor:
    lib = _capi.ensure_init()
    H = input_act.shape[1]
    out = torch.empty((num_tokens, H), dtype=input_act.dtype, device=input_act.device)
    check(
        lib.xtb_moe_unpermute(ptr(input_act), ptr(row_id_map), ptr(probs), num_tokens, topk, H, ptr(out), current_stream()),
        "xtb_moe_unpermute",
    )
    return out


@_unpermute_op.register_fake
def _(input_act, row_id_map, probs, num_tokens, topk):
    return input_act.new_empty((num_tokens, input_act.shape[1]))


@torch.library.custom_op("xtuner_b200::unpermute_bwd", mutates_args=())
def _unpermute_bwd_op(
    grad_out: Tensor, input_fwd: Tensor, row_id_map: Tensor, probs: Optional[Tensor], topk: int, need_prob_grad: bool
) -> Tuple[Tensor, Tensor]:
    lib = _capi.ensure_init()
    T, H = grad_out.shape
    act_grad = torch.empty_like(input_fwd)
    prob_grad = torch.empty((T, topk), dtype=torch.float32, device=grad_out.device)
    check(
        lib.xtb_moe_unpermute_bwd(
            ptr(grad_out), ptr(input_fwd), ptr(row_id_map), ptr(probs), T, topk, H, ptr(act_grad),
            ptr(prob_grad) if need_prob_grad else None, current_stream(),
        ),
        "xtb_moe_unpermute_bwd",
    )
    return act_grad, prob_grad


@_unpermute_bwd_op.register_fake
def _(grad_out, input_fwd, row_id_map, probs, topk, need_prob_grad):
    return torch.empty_like(input_fwd), grad_out.new_empty((grad_out.shape[0], topk), dtype=torch.float32)


def _gg_call(fn_name: str, a: Tensor, b: Tensor, tpe: Tensor, M: int, N: int, Kd: int, E: int, out: Tensor) -> None:
    lib = _capi.ensure_init()
    check(getattr(lib, fn_name)(ptr(a), ptr(b), ptr(tpe), M, N, Kd, E, ptr(out), current_stream()), fn_name)


@torch.library.custom_op("xtuner_b200::group_gemm_nt", mutates_args=())
def _gg_nt(x: Tensor, w: Tensor, tokens_per_expert: Tensor) -> Tensor:
    E, N, Kd = w.shape
    out = torch.empty((x.shape[0], N), dtype=x.dtype, device=x.device)
    _gg_call("xtb_group_gemm_nt", x, w, tokens_per_expert, x.shape[0], N, Kd, E, out)
    return out


@_gg_nt.register_fake
def _(x, w, tokens_per_expert):
    return x.new_empty((x.shape[0], w.shape[1]))


@torch.library.custom_op("xtuner_b200::group_gemm_nn", mutates_args=())
def _gg_nn(dy: Tensor, w: Tensor, tokens_per_expert: Tensor) -> Tensor:
    E, N, Kd = w.shape
    out = torch.empty((dy.shape[0], Kd), dtype=dy.dtype, device=dy.device)
    _gg_call("xtb_group_gemm_nn", dy, w, tokens_per_expert, dy.shape[0], N, Kd, E, out)
    return out


@_gg_nn.register_fake
def _(dy, w, tokens_per_expert):
    return dy.new_empty((dy.shape[0], w.shape[2]))


@torch.library.custom_op("xtuner_b200::group_gemm_tn", mutates_args=())
def _gg_tn(dy: Tensor, x: Tensor, tokens_per_expert: Tensor) -> Tensor:
    E = tokens_per_expert.shape[0]
    N, Kd = dy.shape[1], x.shape[1]
    dw = torch.empty((E, N, Kd), dtype=x.dtype, device=x.device)
    _gg_call("xtb_group_gemm_tn", dy, x, tokens_per_expert, x.shape[0], N, Kd, E, dw)
    return dw


@_gg_tn.register_fake
def _(dy, x, tokens_per_expert):
    return x.new_empty((tokens_per_expert.shape[0], dy.shape[1], x.shape[1]))


@torch.library.custom_op("xtuner_b200::swiglu", mutates_args=())
def _swiglu_op(h: Tensor) -> Tensor:
    lib = _capi.ensure_init()
    M, twoI = h.shape
    out = torch.empty((M, twoI // 2), dtype=h.dtype, device=h.device)
    check(lib.xtb_swiglu(ptr(h), ptr(out), M, twoI // 2, current_stream()), "xtb_swiglu")
    return out


@_swiglu_op.register_fake
def _(h):
    return h.new_empty((h.shape[0], h.shape[1] // 2))


@torch.library.custom_op("xtuner_b200::swiglu_bwd", mutates_args=())
def _swiglu_bwd_op(grad_out: Tensor, h: Tensor) -> Tensor:
    lib = _capi.ensure_init()
    M, twoI = h.shape
    grad_h = torch.empty_like(h)
    check(lib.xtb_swiglu_bwd(ptr(grad_out), ptr(h), ptr(grad_h), M, twoI // 2, current_stream()), "xtb_swiglu_bwd")
    return grad_h


@_swiglu_bwd_op.register_fake
def _(grad_out, h):
    return torch.empty_like(h)


@torch.library.custom_op("xtuner_b200::gate_logits", mutates_args=())
def _gate_logits_op(x: Tensor, w: Tensor, bias: Optional[Tensor]) -> Tensor:
    lib = _capi.ensure_init()
    T, H = x.shape
    E = w.shape[0]
    logits = torch.empty((T, E), dtype=torch.float32, device=x.device)
    check(lib.xtb_gate_logits(ptr(x), ptr(w), ptr(bias), ptr(logits), T, H, E, current_stream()), "xtb_gate_logits")
    return logits


@_gate_logits_op.register_fake
def _(x, w, bias):
    return x.new_empty((x.shape[0], w.shape[0]), dtype=torch.float32)


@torch.library.custom_op("xtuner_b200::gate_logits_bwd", mutates_args=())
def _gate_logits_bwd_op(grad_logits: Tensor, x: Tensor, w: Tensor, need_bias: bool) -> Tuple[Tensor, Tensor, Tensor]:
    lib = _capi.ensure_init()
    T, H = x.shape
    E = w.shape[0]
    grad_w = torch.empty_like(w)
    grad_x = torch.empty_like(x)
    grad_b = torch.empty((E,), dtype=torch.float32, device=x.device)
    ws = _scratch("gate_bwd", int(lib.xtb_gate_logits_bwd_workspace_bytes(T, H, E)), x.device)
    check(
        lib.xtb_gate_logits_bwd(
            ptr(grad_logits), ptr(x), ptr(w), ptr(grad_w), ptr(grad_x), ptr(grad_b) if need_bias else None, T, H, E,
            ptr(ws), current_stream(),
        ),
        "xtb_gate_logits_bwd",
    )
    return grad_x, grad_w, grad_b


@_gate_logits_bwd_op.register_fake
def _(grad_logits, x, w, need_bias):
    return torch.empty_like(x), torch.empty_like(w), w.new_empty((w.shape[0],))


# ======================================================================================================
# autograd layer + protocol-compatible callables
# ======================================================================================================


class _Permute(torch.autograd.Function):
    """``PermuteMoE_topK`` (permute_unpermute.py:92-143): backward = unpermute without probs."""

    @staticmethod
    def forward(ctx, input_act: Tensor, indices: Tensor, n_experts: int):
        permuted, row_id_map, sorted_indices, tpe = _permute_op(input_act, indices, n_experts)
        ctx.save_for_backward(row_id_map)
        ctx.num_tokens, ctx.topk = indices.shape
        ctx.mark_non_differentiable(row_id_map, sorted_indices, tpe)
        return permuted, row_id_map, sorted_indices, tpe

    @staticmethod
    def backward(ctx, g_perm, _g1, _g2, _g3):
        (row_id_map,) = ctx.saved_tensors
        return _unpermute_op(g_perm.contiguous(), row_id_map, None, ctx.num_tokens, ctx.topk), None, None


class _Unpermute(torch.autograd.Function):
    """``UnpermuteMoE_topK`` (permute_unpermute.py:146-192)."""

    @staticmethod
    def forward(ctx, input_act: Tensor, row_id_map: Tensor, probs: Optional[Tensor]):
        if probs is not None:
            num_tokens, topk = probs.shape
        else:
            num_tokens, topk = input_act.shape[0], 1
        out = _unpermute_op(input_act, row_id_map, probs, num_tokens, topk)
        ctx.save_for_backward(input_act, row_id_map, probs)
        ctx.topk = topk
        return out

    @staticmethod
    def backward(ctx, g_out):
        input_act, row_id_map, probs = ctx.saved_tensors
        need_p = probs is not None and ctx.needs_input_grad[2]
        act_grad, prob_grad = _unpermute_bwd_op(g_out.contiguous(), input_act, row_id_map, probs, ctx.topk, need_p)
        return act_grad, None, (prob_grad if need_p else None)


class _GroupedGemm(torch.autograd.Function):
    """``GroupedGemm`` (ops/moe/cuda/group_gemm.py:8-20): dx via the NN product, dw via the TN product."""

    @staticmethod
    def forward(ctx, x: Tensor, w: Tensor, tokens_per_expert: Tensor):
        out = _gg_nt(x, w, tokens_per_expert)
        ctx.save_for_backward(x, w, tokens_per_expert)
        return out

    @staticmethod
    def backward(ctx, grad_output):
        x, w, tpe = ctx.saved_tensors
        grad_output = grad_output.contiguous()
        dx = _gg_nn(grad_output, w, tpe) if ctx.needs_input_grad[0] else None
        dw = _gg_tn(grad_output, x, tpe) if ctx.needs_input_grad[1] else None
        return dx, dw, None


class _Swiglu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, h: Tensor):
        ctx.save_for_backward(h)
        return _swiglu_op(h)

    @staticmethod
    def backward(ctx, g):
        (h,) = ctx.saved_tensors
        return _swiglu_bwd_op(g.contiguous(), h)


class _GateLogits(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x: Tensor, w: Tensor, bias: Optional[Tensor]):
        ctx.save_for_backward(x, w)
        ctx.has_bias = bias is not None
        return _gate_logits_op(x, w, bias)

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        gx, gw, gb = _gate_logits_bwd_op(g.contiguous(), x, w, ctx.has_bias)
        return gx, gw, (gb if ctx.has_bias else None)


def permute(
    input_act: Tensor,
    indices: Tensor,
    num_topK: int | None = None,
    num_out_tokens: int | None = None,
    num_negative_one_in_indices: int | None = None,
    *,
    n_experts: int | None = None,
    return_extra: bool = False,
):
    """``MoePermuteProtocol`` (ops/moe/protocol.py:15-23).  Returns ``(permuted, row_id_map)``.

    ``row_id_map`` is opaque (flat index -> permuted row, int32) and is only meaningful to
    :func:`unpermute`.  ``n_experts`` bounds the expert ids; when omitted it is taken as
    ``indices.max()+1`` rounded up — pass it to stay free of a device->host sync.
    With ``return_extra`` also returns ``(sorted_indices, tokens_per_expert)``."""
    if num_out_tokens not in (None, 0) or num_negative_one_in_indices not in (None, 0):
        raise NotImplementedError("dropless path only: num_out_tokens / num_negative_one_in_indices must be 0")
    _require_cuda(input_act, indices)
    if not input_act.numel():
        if not return_extra:
            return input_act, None
        # the reference still produces the (all-zero) histogram for an empty batch (dispatcher/base.py:398)
        tpe = None if n_experts is None else torch.zeros(n_experts, dtype=torch.int64, device=input_act.device)
        return input_act, None, None, tpe
    if indices.dtype != torch.int32:
        indices = indices.to(torch.int32)  # permute_unpermute.py:104-105
    if indices.dim() == 1:
        indices = indices.view(-1, 1)
    input_act = input_act.contiguous()
    indices = indices.contiguous()
    if n_experts is None:
        n_experts = int(indices.max().item()) + 1  # host sync: callers on the hot path pass n_experts
    permuted, row_id_map, sorted_indices, tpe = _Permute.apply(input_act, indices, n_experts)
    if return_extra:
        return permuted, row_id_map, sorted_indices, tpe
    return permuted, row_id_map


def unpermute(input_act: Tensor, row_id_map: Tensor, probs: Tensor | None = None) -> Tensor:
    """``MoeUnpermuteProtocol`` (ops/moe/protocol.py:26-30)."""
    _require_cuda(input_act, row_id_map, probs)
    if not input_act.numel():
        return input_act
    _bf16(input_act, "input_act")
    input_act = input_act.contiguous()
    row_id_map = row_id_map.contiguous()
    if probs is not None:
        probs = probs.contiguous()
        if probs.dtype != torch.float32:
            probs = probs.to(torch.float32)  # permute_unpermute.py:160-161
    return _Unpermute.apply(input_act, row_id_map, probs)


def group_gemm(x: Tensor, weights: Tensor, split_sizes: Tensor) -> Tensor:
    """``GroupGemmProtocol`` (ops/moe/protocol.py:6-12): ``weights`` is ``[E, dout, din]``,
    ``split_sizes`` the device int64 ``tokens_per_expert``.

    Shapes are checked on the host before anything is launched (``XtbError``): ``weights`` must be 3-D, ``x`` 2-D with
    ``x.shape[1] == weights.shape[2]``, and ``split_sizes`` 1-D with ``weights.shape[0]`` entries.  That
    ``split_sizes`` sums to ``x.shape[0]`` is not checked: the counts live on the device and reading them would
    synchronise the stream."""
    _require_cuda(x, weights, split_sizes)
    if weights.dim() != 3:
        raise _capi.XtbError(f"group_gemm: weights must be [E, dout, din] (got shape {tuple(weights.shape)})")
    if x.dim() != 2 or x.shape[1] != weights.shape[2]:
        raise _capi.XtbError(f"group_gemm: x must be [M, {weights.shape[2]}] for weights {tuple(weights.shape)} "
                             f"(got {tuple(x.shape)})")
    if split_sizes.dim() != 1 or split_sizes.shape[0] != weights.shape[0]:
        raise _capi.XtbError(f"group_gemm: split_sizes must be 1-D with {weights.shape[0]} entries, one per expert "
                             f"(got shape {tuple(split_sizes.shape)})")
    if x.shape[0] == 0:
        return torch.matmul(x, weights[0].T)  # keep x and w in the graph (group_gemm.py:34-36)
    _bf16(x, "x")
    _bf16(weights, "weights")
    if split_sizes.dtype != torch.int64:
        split_sizes = split_sizes.to(torch.int64)
    return _GroupedGemm.apply(x.contiguous(), weights.contiguous(), split_sizes.contiguous())


def swiglu(fused_x: Tensor, split_dim: int = -1) -> Tensor:
    """``native_swiglu`` (ops/act_fn.py:7-9) for the ``[M, 2I]`` expert activation."""
    _require_cuda(fused_x)
    if split_dim not in (-1, fused_x.dim() - 1):
        raise NotImplementedError("swiglu: only the last dim can be split")
    _bf16(fused_x, "fused_x")
    shape = fused_x.shape
    out = _Swiglu.apply(fused_x.contiguous().view(-1, shape[-1]))
    return out.view(*shape[:-1], shape[-1] // 2)


def gate_logits(hidden_states: Tensor, weight: Tensor, bias: Tensor | None = None) -> Tensor:
    """fp32 gate GEMM of ``MoEGate.forward`` (moe_decoder_layer.py:136-140); ``weight`` is used in fp32."""
    _require_cuda(hidden_states, weight, bias)
    _bf16(hidden_states, "hidden_states")
    x = hidden_states.contiguous().view(-1, hidden_states.shape[-1])
    w = weight if weight.dtype == torch.float32 else weight.float()
    b = None if bias is None else bias.float().contiguous()
    return _GateLogits.apply(x, w.contiguous(), b)


# ======================================================================================================
# lm_head + cross-entropy (f4): what LMHeadLossContext computes in modes "eager" and "chunk"
# ======================================================================================================


def _lm_head_ce_call(h, w, labels, loss_weight, ignore_index, need_grad, z, row_ce, loss, dh, dw) -> None:
    lib = _capi.ensure_init()
    T, H = h.shape
    V = w.shape[0]
    ws = _scratch("lm_head_ce", int(lib.xtb_lm_head_ce_workspace_bytes(T, V)), h.device)
    check(
        lib.xtb_lm_head_ce(
            ptr(h), ptr(w), ptr(labels), ptr(loss_weight), T, H, V, ignore_index, int(need_grad), ptr(z), ptr(ws),
            ptr(row_ce), ptr(loss), ptr(dh), ptr(dw), current_stream(),
        ),
        "xtb_lm_head_ce",
    )


class _LMHeadCrossEntropy(torch.autograd.Function):
    """``ChunkLoss`` (loss/chunk_loss.py) over ``xtb_lm_head_ce``: the gradients are computed in the forward, one row chunk
    at a time (one chunk = eager semantics); chunk losses are added in fp32 and each later chunk's ``dW`` is added into
    the first in bf16, in chunk order.  Backward scales both by ``grad_output`` on the device."""

    @staticmethod
    def forward(ctx, h: Tensor, w: Tensor, labels: Tensor, loss_weight: Tensor, ignore_index: int,
                chunk_size: Optional[int], need_grad: bool):
        T = h.shape[0]
        if T == 0:  # an empty tensor has no address, which the entry rejects; the reference gives 0, empty dh, zero dW
            if need_grad:
                ctx.save_for_backward(torch.empty_like(h), torch.zeros_like(w))
            return torch.zeros((), dtype=torch.float32, device=h.device)
        step = T if chunk_size is None else chunk_size
        z = torch.empty((min(step, T), w.shape[0]), dtype=torch.bfloat16, device=h.device)  # z, then G, of one chunk
        row_ce = torch.empty((T,), dtype=torch.float32, device=h.device)
        dh = torch.empty_like(h) if need_grad else None
        loss = dw = dw_chunk = None
        for s in range(0, T, step):
            n = min(step, T - s)
            loss_c = torch.empty((), dtype=torch.float32, device=h.device)
            dw_c = None
            if need_grad:  # the first chunk writes dW itself, later ones a scratch copy that is added into it
                dw_chunk = torch.empty_like(w) if dw is not None and dw_chunk is None else dw_chunk
                dw_c = torch.empty_like(w) if dw is None else dw_chunk
            _lm_head_ce_call(h[s:s + n], w, labels[s:s + n], loss_weight[s:s + n], ignore_index, need_grad, z[:n],
                             row_ce[s:s + n], loss_c, None if dh is None else dh[s:s + n], dw_c)
            loss = loss_c if loss is None else loss.add_(loss_c)
            if need_grad:
                dw = dw_c if dw is None else dw.add_(dw_c)
        if need_grad:
            ctx.save_for_backward(dh, dw)
        return loss

    @staticmethod
    def backward(ctx, grad_output):
        dh, dw = ctx.saved_tensors
        # unconditional: x1 is exact, so this equals ChunkLoss's `if grad_output != 1` without reading it on the host
        return (dh * grad_output if ctx.needs_input_grad[0] else None,
                dw * grad_output if ctx.needs_input_grad[1] else None, None, None, None, None, None)


def lm_head_cross_entropy(hidden: Tensor, weight: Tensor, labels: Tensor, loss_weight: Tensor, ignore_index: int = -100,
                          chunk_size: int | None = None) -> Tensor:
    """``sum_t CE(hidden[t] . weight^T, labels[t]) * loss_weight[t]`` as ``LMHeadLossContext`` computes it
    (loss/ce_loss.py ``loss_fn``): bf16 logits, fp32 log-softmax, rows with ``labels == ignore_index`` contribute 0.
    ``chunk_size=None`` is mode "eager"; an integer runs mode "chunk" (``ChunkLoss``) over rows of that many.
    ``hidden`` is ``[..., H]`` bf16, ``weight`` ``[V, H]`` bf16 with ``V % 128 == 0`` and ``H % 128 == 0``, ``labels`` and
    ``loss_weight`` hold one entry per row of ``hidden``.  The logits are never returned: one bf16 ``[rows, V]`` buffer per
    chunk holds them and then their gradient.  Gradients are computed in the forward when grad mode is on and ``hidden``
    or ``weight`` requires grad.  A label outside ``[0, V)`` that is not ``ignore_index`` makes the loss NaN."""
    _require_cuda(hidden, weight, labels, loss_weight)
    _bf16(hidden, "hidden")
    _bf16(weight, "weight")
    if weight.dim() != 2 or hidden.shape[-1] != weight.shape[1]:
        raise _capi.XtbError(f"lm_head_cross_entropy: weight must be [V, {hidden.shape[-1]}] (got {tuple(weight.shape)})")
    h = hidden.reshape(-1, hidden.shape[-1]).contiguous()
    lab = labels.reshape(-1).to(torch.int64).contiguous()
    lw = loss_weight.reshape(-1).to(torch.float32).contiguous()
    if lab.numel() != h.shape[0] or lw.numel() != h.shape[0]:
        raise _capi.XtbError(f"lm_head_cross_entropy: {h.shape[0]} rows but {lab.numel()} labels and {lw.numel()} weights")
    if chunk_size is not None and chunk_size <= 0:
        raise ValueError(f"lm_head_cross_entropy: chunk_size must be positive (got {chunk_size})")
    need_grad = torch.is_grad_enabled() and (hidden.requires_grad or weight.requires_grad)
    return _LMHeadCrossEntropy.apply(h, weight.contiguous(), lab, lw, int(ignore_index), chunk_size, need_grad)


# ======================================================================================================
# lm_head label log-probabilities (f5): gather_logprobs(F.linear(h, W).float(), labels) of LogProbContext and
# GRPOLossContext, with the per-token loss of logp left to torch
# ======================================================================================================


def _lm_head_logprob_call(h, w, labels, z, logp, row_stats) -> None:
    lib = _capi.ensure_init()
    T, H = h.shape
    V = w.shape[0]
    ws = _scratch("lm_head_logprob", int(lib.xtb_lm_head_logprob_workspace_bytes(T, V)), h.device)
    check(lib.xtb_lm_head_logprob(ptr(h), ptr(w), ptr(labels), T, H, V, ptr(z), ptr(ws), ptr(logp), ptr(row_stats),
                                  current_stream()), "xtb_lm_head_logprob")


class _LMHeadLogProbs(torch.autograd.Function):
    """One node over all rows: the forward keeps z ([T, V] bf16) and the row statistics, the backward writes G over z from
    ``dL/dlogp`` and returns dh and dW.  G replaces z, so the node can be differentiated once."""

    @staticmethod
    def forward(ctx, h: Tensor, w: Tensor, labels: Tensor):
        T, V = h.shape[0], w.shape[0]
        z = torch.empty((T, V), dtype=torch.bfloat16, device=h.device)
        logp = torch.empty((T,), dtype=torch.float32, device=h.device)
        row_stats = torch.empty((T, 2), dtype=torch.float32, device=h.device)
        if T:  # an empty tensor has no address, which the entries reject
            _lm_head_logprob_call(h, w, labels, z, logp, row_stats)
        ctx.save_for_backward(z, row_stats, labels, h, w)
        ctx.consumed = False
        return logp

    @staticmethod
    def backward(ctx, grad_logp):
        if ctx.consumed:
            raise RuntimeError("lm_head_logprobs: the backward overwrites the saved logits with their gradient, so it runs "
                               "once per forward; recompute the forward instead of backpropagating twice")
        ctx.consumed = True
        z, row_stats, labels, h, w = ctx.saved_tensors
        T, H = h.shape
        V = w.shape[0]
        if T == 0:
            return (torch.empty_like(h) if ctx.needs_input_grad[0] else None,
                    torch.zeros_like(w) if ctx.needs_input_grad[1] else None, None)
        g = grad_logp.to(torch.float32).contiguous()
        dh, dw = torch.empty_like(h), torch.empty_like(w)
        lib = _capi.ensure_init()
        ws = _scratch("lm_head_logprob", int(lib.xtb_lm_head_logprob_workspace_bytes(0, V)), h.device)
        check(lib.xtb_lm_head_logprob_bwd(ptr(z), ptr(row_stats), ptr(labels), ptr(g), ptr(h), ptr(w), T, H, V, ptr(ws),
                                          ptr(dh), ptr(dw), current_stream()), "xtb_lm_head_logprob_bwd")
        return (dh if ctx.needs_input_grad[0] else None, dw if ctx.needs_input_grad[1] else None, None)


def lm_head_logprobs(hidden: Tensor, weight: Tensor, labels: Tensor, chunk_size: int | None = None) -> Tensor:
    """``gather_logprobs(F.linear(hidden, weight).float(), labels)`` (rl/utils/misc.py): the fp32 log-probability of each
    row's label under the bf16 logits, shaped like ``labels``.  Labels are clipped at 0 as there, so an ignored position
    (-100) gets the log-probability of token 0; a label ``>= V`` gives NaN in its row.  ``hidden`` is ``[..., H]`` bf16,
    ``weight`` ``[V, H]`` bf16 with ``V % 128 == 0`` and ``H % 128 == 0``, ``labels`` holds one entry per row.

    Without grad (grad mode off, or neither ``hidden`` nor ``weight`` requires it) the forward runs ``chunk_size`` rows at
    a time (all at once for None) through one reused ``[chunk_size, V]`` bf16 buffer; rows are independent, so the result
    does not depend on ``chunk_size``.  With grad it is one autograd node that keeps the ``[rows, V]`` bf16 logits for its
    backward, which overwrites them: a second backward through the same call raises."""
    _require_cuda(hidden, weight, labels)
    _bf16(hidden, "hidden")
    _bf16(weight, "weight")
    if weight.dim() != 2 or hidden.shape[-1] != weight.shape[1]:
        raise _capi.XtbError(f"lm_head_logprobs: weight must be [V, {hidden.shape[-1]}] (got {tuple(weight.shape)})")
    h = hidden.reshape(-1, hidden.shape[-1]).contiguous()
    lab = labels.reshape(-1).to(torch.int64).contiguous()
    if lab.numel() != h.shape[0]:
        raise _capi.XtbError(f"lm_head_logprobs: {h.shape[0]} rows but {lab.numel()} labels")
    if chunk_size is not None and chunk_size <= 0:
        raise ValueError(f"lm_head_logprobs: chunk_size must be positive (got {chunk_size})")
    w = weight.contiguous()
    if torch.is_grad_enabled() and (hidden.requires_grad or weight.requires_grad):
        return _LMHeadLogProbs.apply(h, w, lab).view(labels.shape)
    T = h.shape[0]
    step = max(T, 1) if chunk_size is None else chunk_size
    z = torch.empty((min(step, T), w.shape[0]), dtype=torch.bfloat16, device=h.device)
    logp = torch.empty((T,), dtype=torch.float32, device=h.device)
    for s in range(0, T, step):
        n = min(step, T - s)
        _lm_head_logprob_call(h[s:s + n], w, lab[s:s + n], z[:n], logp[s:s + n], None)
    return logp.view(labels.shape)


# ======================================================================================================
# q/k RMSNorm + rotary embedding in front of the attention (MultiHeadAttention.forward, mha.py:353-363)
# ======================================================================================================


def _rows(t: Tensor) -> Tuple[int, int]:
    """(token stride, head stride) in elements of a [T, H, D] operand"""
    return t.stride(0), t.stride(1)


@torch.library.custom_op("xtuner_b200::qk_norm_rope", mutates_args=())
def _qk_norm_rope_op(q: Tensor, k: Tensor, cos: Tensor, sin: Tensor, w_q: Optional[Tensor], w_k: Optional[Tensor],
                     eps: float) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (out_q [T, Hq, D], out_k [T, Hkv, D], rstd_q fp32 [T, Hq], rstd_k fp32 [T, Hkv]); the rstd are empty without a
    norm weight"""
    lib = _capi.ensure_init()
    q, k = _strided_rows(q), _strided_rows(k)
    T, Hq, D = q.shape
    Hkv = k.shape[1]
    out_q, out_k = q.new_empty((T, Hq, D)), k.new_empty((T, Hkv, D))
    norm = w_q is not None
    rstd_q = q.new_empty((T, Hq) if norm else (0,), dtype=torch.float32)
    rstd_k = k.new_empty((T, Hkv) if norm else (0,), dtype=torch.float32)
    if T == 0:
        return out_q, out_k, rstd_q, rstd_k
    check(
        lib.xtb_qk_norm_rope(
            ptr(q), *_rows(q), ptr(k), *_rows(k), ptr(cos), ptr(sin), ptr(w_q), ptr(w_k), eps, T, Hq, Hkv, D, ptr(out_q),
            ptr(out_k), ptr(rstd_q) if norm else None, ptr(rstd_k) if norm else None, current_stream(),
        ),
        "xtb_qk_norm_rope",
    )
    return out_q, out_k, rstd_q, rstd_k


@_qk_norm_rope_op.register_fake
def _(q, k, cos, sin, w_q, w_k, eps):
    norm = w_q is not None
    return (q.new_empty(q.shape), k.new_empty(k.shape),
            q.new_empty(q.shape[:2] if norm else (0,), dtype=torch.float32),
            k.new_empty(k.shape[:2] if norm else (0,), dtype=torch.float32))


@torch.library.custom_op("xtuner_b200::qk_norm_rope_bwd", mutates_args=())
def _qk_norm_rope_bwd_op(g_q: Tensor, g_k: Tensor, q: Tensor, k: Tensor, cos: Tensor, sin: Tensor, w_q: Optional[Tensor],
                         w_k: Optional[Tensor], rstd_q: Tensor, rstd_k: Tensor, need_dw: bool
                         ) -> Tuple[Tensor, Tensor, Tensor]:
    """-> (dx_q [T, Hq, D], dx_k [T, Hkv, D], dw fp32 [2, D] = (dw_q, dw_k), empty unless ``need_dw``)"""
    lib = _capi.ensure_init()
    g_q, g_k, q, k = (_strided_rows(t) for t in (g_q, g_k, q, k))
    T, Hq, D = q.shape
    Hkv = k.shape[1]
    dx_q, dx_k = q.new_empty((T, Hq, D)), k.new_empty((T, Hkv, D))
    norm = w_q is not None
    need_dw = need_dw and norm
    dw = q.new_empty((2, D) if need_dw else (0,), dtype=torch.float32)
    if T == 0:
        return dx_q, dx_k, dw.zero_()
    ws = _scratch("qk_norm_rope_bwd", int(lib.xtb_qk_norm_rope_bwd_workspace_bytes(T, D)), q.device) if need_dw else None
    check(
        lib.xtb_qk_norm_rope_bwd(
            ptr(g_q), *_rows(g_q), ptr(g_k), *_rows(g_k), ptr(q), *_rows(q), ptr(k), *_rows(k), ptr(cos), ptr(sin), ptr(w_q),
            ptr(w_k), ptr(rstd_q) if norm else None, ptr(rstd_k) if norm else None, T, Hq, Hkv, D, ptr(dx_q), ptr(dx_k),
            ptr(dw) if need_dw else None, ptr(ws), current_stream(),
        ),
        "xtb_qk_norm_rope_bwd",
    )
    return dx_q, dx_k, dw


@_qk_norm_rope_bwd_op.register_fake
def _(g_q, g_k, q, k, cos, sin, w_q, w_k, rstd_q, rstd_k, need_dw):
    need = need_dw and w_q is not None
    return q.new_empty(q.shape), k.new_empty(k.shape), q.new_empty((2, q.shape[2]) if need else (0,), dtype=torch.float32)


class _QKNormRope(torch.autograd.Function):
    """q_norm / k_norm (``F.rms_norm``) followed by ``apply_rotary_pos_emb_cuda`` as one node.  Saves the projections
    (which the reference keeps alive too), the two rstd, cos and sin; no normalised copy."""

    @staticmethod
    def forward(ctx, q: Tensor, k: Tensor, cos: Tensor, sin: Tensor, w_q: Optional[Tensor], w_k: Optional[Tensor],
                eps: float):
        out_q, out_k, rstd_q, rstd_k = _qk_norm_rope_op(q, k, cos, sin, w_q, w_k, eps)
        ctx.save_for_backward(q, k, cos, sin, w_q, w_k, rstd_q, rstd_k)
        ctx.mark_non_differentiable(rstd_q, rstd_k)
        return out_q, out_k, rstd_q, rstd_k

    @staticmethod
    def backward(ctx, g_q, g_k, _g_rq, _g_rk):
        q, k, cos, sin, w_q, w_k, rstd_q, rstd_k = ctx.saved_tensors
        need_dw = w_q is not None and (ctx.needs_input_grad[4] or ctx.needs_input_grad[5])
        g_q = torch.zeros_like(q) if g_q is None else g_q
        g_k = torch.zeros_like(k) if g_k is None else g_k
        dx_q, dx_k, dw = _qk_norm_rope_bwd_op(g_q, g_k, q, k, cos, sin, w_q, w_k, rstd_q, rstd_k, need_dw)
        dw_q = dw[0] if need_dw and ctx.needs_input_grad[4] else None
        dw_k = dw[1] if need_dw and ctx.needs_input_grad[5] else None
        return dx_q, dx_k, None, None, dw_q, dw_k, None


def _strided_rows(t: Tensor) -> Tensor:
    """``t`` itself when the kernels can read it in place ([T, H, D] with the D axis contiguous and 16-byte aligned rows),
    otherwise a contiguous copy.  Called inside the custom ops, which always see real tensors."""
    if t.stride(2) == 1 and t.stride(0) % 8 == 0 and t.stride(1) % 8 == 0 and t.data_ptr() % 16 == 0:
        return t
    return t.contiguous()


def qk_norm_rope(q: Tensor, k: Tensor, cos: Tensor, sin: Tensor, q_norm_weight: Tensor | None = None,
                 k_norm_weight: Tensor | None = None, eps: float = 1e-6) -> Tuple[Tensor, Tensor]:
    """``apply_rotary_pos_emb_cuda(q_norm(q), k_norm(k), cos, sin)`` of ``MultiHeadAttention`` (mha.py:353-363) with the
    reference's roundings (``include/xtuner_b200.h``): ``q`` ``[T, Hq, D]`` and ``k`` ``[T, Hkv, D]`` bf16 (any token and
    head strides; the D axis contiguous), ``cos``/``sin`` ``[T, D]`` bf16, norm weights ``[D]`` (fp32 or bf16) or both
    None to skip the norm.  D is 64, 128 or 256.  Returns contiguous ``(q_embed [T, Hq, D], k_embed [T, Hkv, D])``; the
    weight gradients come back in the weights' dtype."""
    _require_cuda(q, k, cos, sin, q_norm_weight, k_norm_weight)
    for t, name in ((q, "q"), (k, "k"), (cos, "cos"), (sin, "sin")):
        _bf16(t, name)
    if (q_norm_weight is None) != (k_norm_weight is None):
        raise ValueError("qk_norm_rope: pass both norm weights or neither")
    if q.dim() != 3 or k.dim() != 3 or k.shape[0] != q.shape[0] or k.shape[2] != q.shape[2]:
        raise _capi.XtbError(f"qk_norm_rope: q must be [T, Hq, D] and k [T, Hkv, D] (got {tuple(q.shape)}, {tuple(k.shape)})")
    T, _, D = q.shape
    if D not in (64, 128, 256):
        raise _capi.XtbError(f"qk_norm_rope: head dim {D} is not 64, 128 or 256")
    cos, sin = cos.reshape(-1, cos.shape[-1]), sin.reshape(-1, sin.shape[-1])
    if tuple(cos.shape) != (T, D) or tuple(sin.shape) != (T, D):
        raise _capi.XtbError(f"qk_norm_rope: cos and sin must be [{T}, {D}] (got {tuple(cos.shape)}, {tuple(sin.shape)})")
    w_q = w_k = None
    if q_norm_weight is not None:
        if tuple(q_norm_weight.shape) != (D,) or tuple(k_norm_weight.shape) != (D,):
            raise _capi.XtbError(f"qk_norm_rope: norm weights must be [{D}]")
        w_q, w_k = q_norm_weight.float().contiguous(), k_norm_weight.float().contiguous()  # bf16 widens exactly
    out_q, out_k, _, _ = _QKNormRope.apply(q, k, cos.contiguous(), sin.contiguous(), w_q, w_k, float(eps))
    return out_q, out_k


# ======================================================================================================
# MoE auxiliary-loss statistics (AuxLossContext.accumulate, loss/aux_loss.py:84-151)
# ======================================================================================================

MOE_AUX_MAX_EXPERTS = 512  # the largest E xtb_moe_aux_stats takes


def _moe_aux_workspace(N: int, E: int, device) -> Tensor:
    """zero-filled once: the kernel's ticket must start at zero, and every call leaves it so"""
    need = int(_capi.ensure_init().xtb_moe_aux_stats_workspace_bytes(N, E))
    key = ("moe_aux", device, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(max(need, 1 << 16), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def _plain(t: Tensor) -> Tensor:
    """the tensor behind a pending functional collective's result (``AsyncCollectiveTensor.wait()``), else ``t``"""
    return t.wait() if type(t) is not Tensor and hasattr(t, "wait") else t


class _MoEAuxStats(torch.autograd.Function):
    """One node over ``xtb_moe_aux_stats`` / ``xtb_moe_aux_stats_bwd``.  Saves the logits and the row logsumexps only for
    the z-loss; an output that receives no gradient gives its input no gradient (no zero ``[N, E]`` tensor is made)."""

    @staticmethod
    def forward(ctx, rw: Tensor, logits: Optional[Tensor], ids: Tensor, n_experts: int, need_rw_sum: bool, need_z: bool):
        ctx.set_materialize_grads(False)
        N, K = ids.shape
        dev = ids.device
        tpe = torch.empty((n_experts,), dtype=torch.int64, device=dev)
        rw_sum = torch.empty((n_experts,), dtype=torch.float32, device=dev) if need_rw_sum else None
        z_sum = torch.empty((), dtype=torch.float32, device=dev) if need_z else None
        lse = torch.empty((N,), dtype=torch.float32, device=dev) if need_z else None
        lib = _capi.ensure_init()
        ws = _moe_aux_workspace(N, n_experts, dev)
        check(lib.xtb_moe_aux_stats(ptr(rw) if need_rw_sum else None, ptr(logits) if need_z else None, ptr(ids), N,
                                    n_experts, K, ptr(tpe), ptr(rw_sum), ptr(z_sum), ptr(lse), ptr(ws), current_stream()),
              "xtb_moe_aux_stats")
        ctx.mark_non_differentiable(tpe)
        if need_z:
            ctx.save_for_backward(logits, lse)
        ctx.shape = (N, n_experts)
        return tpe, rw_sum, z_sum

    @staticmethod
    def backward(ctx, _g_tpe, g_rw_sum, g_z):
        N, E = ctx.shape
        need_rw = g_rw_sum is not None and ctx.needs_input_grad[0]
        need_lg = g_z is not None and ctx.needs_input_grad[1]
        if not (need_rw or need_lg):
            return None, None, None, None, None, None
        logits, lse = ctx.saved_tensors if need_lg else (None, None)
        dev = (g_rw_sum if need_rw else g_z).device
        g_rw = torch.empty((N, E), dtype=torch.float32, device=dev) if need_rw else None
        g_logits = torch.empty((N, E), dtype=torch.float32, device=dev) if need_lg else None
        # held in locals until the launch is queued.  An expanded gradient becomes a contiguous copy; one that comes from a
        # functional all-reduce (the global-average balancing loss) is an AsyncCollectiveTensor, whose data pointer is only
        # valid after wait()
        g_rw_sum = _plain(g_rw_sum).float().contiguous() if need_rw else None
        g_z = _plain(g_z).float().contiguous() if need_lg else None
        check(_capi.ensure_init().xtb_moe_aux_stats_bwd(ptr(g_rw_sum), ptr(g_z), ptr(logits), ptr(lse), N, E, ptr(g_rw),
                                                        ptr(g_logits), current_stream()), "xtb_moe_aux_stats_bwd")
        return g_rw, g_logits, None, None, None, None


def moe_aux_stats(router_weights: Tensor, router_logits: Tensor | None, selected_experts: Tensor, n_experts: int, *,
                  need_rw_sum: bool = True, need_z: bool = False):
    """The statistics ``AuxLossContext.accumulate`` derives from one layer's router (loss/aux_loss.py:84-151), in one
    kernel: ``(tokens_per_expert, rw_sum, z_sum)`` with

    * ``tokens_per_expert`` int64 ``[E]`` = ``torch.histc(selected_experts.float(), bins=E, min=0, max=E).long()``,
      exactly (ids equal to E count in the last bin, ids below 0 or above E nowhere); not differentiable;
    * ``rw_sum`` fp32 ``[E]`` = ``router_weights.sum(dim=0)`` (None unless ``need_rw_sum``);
    * ``z_sum`` 0-d fp32 = ``torch.logsumexp(router_logits, -1).square().sum()`` (None unless ``need_z``).

    ``router_weights`` and ``router_logits`` are fp32 ``[N, E]``, ``selected_experts`` int64 ``[N, K]``, all CUDA;
    ``1 <= E <=`` :data:`MOE_AUX_MAX_EXPERTS`.  Sums are added in a fixed order: the same inputs give the same bits."""
    _require_cuda(router_weights, router_logits, selected_experts)
    E = int(n_experts)
    if not 1 <= E <= MOE_AUX_MAX_EXPERTS:
        raise _capi.XtbError(f"moe_aux_stats: n_experts={E} is outside [1, {MOE_AUX_MAX_EXPERTS}]")
    if selected_experts.dim() != 2 or selected_experts.dtype != torch.int64 or selected_experts.shape[1] < 1:
        raise _capi.XtbError(f"moe_aux_stats: selected_experts must be int64 [N, K] (got {tuple(selected_experts.shape)} "
                             f"{selected_experts.dtype})")
    N = selected_experts.shape[0]
    for t, name, need in ((router_weights, "router_weights", need_rw_sum), (router_logits, "router_logits", need_z)):
        if need and (t is None or t.dtype != torch.float32 or tuple(t.shape) != (N, E)):
            raise _capi.XtbError(f"moe_aux_stats: {name} must be float32 [{N}, {E}] (got "
                                 f"{None if t is None else (tuple(t.shape), t.dtype)})")
    rw = router_weights.contiguous() if need_rw_sum else router_weights
    logits = router_logits.contiguous() if need_z else router_logits
    return _MoEAuxStats.apply(rw, logits, selected_experts.contiguous(), E, bool(need_rw_sum), bool(need_z))


# ======================================================================================================
# fp8 tile-wise quantisation (row a15): what the reference's FSDP fp8 all-gather casts with
# ======================================================================================================


def _fp8_call(name: str, *args) -> None:
    check(getattr(_capi.ensure_init(), name)(*args), name)


def fp8_block_scales(w: Tensor, block_size: int = 128) -> Tensor:
    """``tensor_to_per_block_fp8_scales`` for ``dout >= 128`` (float8/fsdp_utils.py:75-116): ``w [nw, dout, din]`` fp32 or bf16
    -> fp32 scales ``[nw, dout/128, din/128]`` = ``clamp(amax of the 128x128 block, 1e-12) / 448``."""
    _require_cuda(w)
    if block_size != 128 or w.dim() != 3 or w.shape[1] % 128 or w.shape[2] % 128 or w.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"fp8_block_scales: needs [nw, dout, din] fp32/bf16 with dout, din multiples of 128 (got {tuple(w.shape)} {w.dtype})")
    w = w.contiguous()
    nw, dout, din = w.shape
    scales = torch.empty((nw, dout // 128, din // 128), dtype=torch.float32, device=w.device)
    _fp8_call("xtb_fp8_block_scales", ptr(w), int(w.dtype == torch.float32), nw, dout, din, ptr(scales), current_stream())
    return scales


def fp8_block_cast(w2d: Tensor, scales: Tensor, block_size: int = 128) -> Tensor:
    """``cast_to_per_block_fp8_with_scales`` for ``dout >= 128`` (float8/fsdp_utils.py:196-223): ``w2d [dout, din]`` divided by
    its block's scale, saturated to e4m3 -> ``torch.float8_e4m3fn [dout, din]``."""
    _require_cuda(w2d, scales)
    if block_size != 128 or w2d.dim() != 2 or w2d.shape[0] % 128 or w2d.shape[1] % 128 or w2d.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"fp8_block_cast: needs [dout, din] fp32/bf16 with dout, din multiples of 128 (got {tuple(w2d.shape)} {w2d.dtype})")
    dout, din = w2d.shape
    if scales.numel() != (dout // 128) * (din // 128) or scales.dtype != torch.float32:
        raise ValueError(f"fp8_block_cast: scales must be fp32 with {(dout // 128) * (din // 128)} elements (got {tuple(scales.shape)} {scales.dtype})")
    w2d, scales = w2d.contiguous(), scales.contiguous()
    q = torch.empty((dout, din), dtype=torch.uint8, device=w2d.device)
    _fp8_call("xtb_fp8_block_cast", ptr(w2d), int(w2d.dtype == torch.float32), 1, dout, din, ptr(scales), ptr(q), current_stream())
    return q.view(torch.float8_e4m3fn)
