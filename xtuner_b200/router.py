"""Routers with the reference's ``RouterProtocol`` surface (``xtuner/v1/module/router/protocol.py:7-18``):
``forward(logits, rollout_routed_experts=None) -> RouterResults`` with the five keys the reference returns
(including its spelling ``topkens_per_expert``); with ``rollout_routed_experts`` (RL routing replay) the weights are
gathered at the given ids instead of a top-k, as the reference's routers do.  One fused sm_90a kernel replaces the reference's
softmax -> topk -> renorm -> scale -> histc eager chain (``router/greedy.py:64-98``, K6 in SURVEY.md §2.3).
``logits`` / ``router_weights`` / ``topk_weights`` stay differentiable (they feed the aux losses and the
combine, SURVEY.md Appendix B)."""
from __future__ import annotations

from typing import Literal, Optional, TypedDict

import torch
from torch import Tensor, nn

from . import _capi
from ._capi import check, current_stream, ptr

SCORING = {"softmax": 0, "sigmoid": 1}


class RouterResults(TypedDict):
    logits: Tensor
    router_weights: Tensor
    topk_weights: Tensor
    topk_ids: Tensor
    topkens_per_expert: Tensor


@torch.library.custom_op("xtuner_b200::router_greedy", mutates_args=())
def _router_greedy_op(
    logits: Tensor, top_k: int, scoring: int, norm_topk_prob: bool, scaling: float
) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    lib = _capi.ensure_init()
    T, E = logits.shape
    dev = logits.device
    rw = torch.empty((T, E), dtype=torch.float32, device=dev)
    tw = torch.empty((T, top_k), dtype=torch.float32, device=dev)
    ids = torch.empty((T, top_k), dtype=torch.int64, device=dev)
    ids32 = torch.empty((T, top_k), dtype=torch.int32, device=dev)
    tpe = torch.empty((E,), dtype=torch.int64, device=dev)
    check(
        lib.xtb_router_greedy(
            ptr(logits), T, E, top_k, scoring, int(norm_topk_prob), float(scaling), ptr(rw), ptr(tw), ptr(ids),
            ptr(ids32), ptr(tpe), current_stream(),
        ),
        "xtb_router_greedy",
    )
    return rw, tw, ids, ids32, tpe


@_router_greedy_op.register_fake
def _(logits, top_k, scoring, norm_topk_prob, scaling):
    T, E = logits.shape
    return (
        logits.new_empty((T, E)),
        logits.new_empty((T, top_k)),
        logits.new_empty((T, top_k), dtype=torch.int64),
        logits.new_empty((T, top_k), dtype=torch.int32),
        logits.new_empty((E,), dtype=torch.int64),
    )


@torch.library.custom_op("xtuner_b200::router_greedy_bwd", mutates_args=())
def _router_greedy_bwd_op(
    rw: Tensor, tw: Tensor, ids: Tensor, g_tw: Optional[Tensor], g_rw: Optional[Tensor], scoring: int,
    norm_topk_prob: bool, scaling: float,
) -> Tensor:
    lib = _capi.ensure_init()
    T, E = rw.shape
    K = tw.shape[1]
    gl = torch.empty_like(rw)
    check(
        lib.xtb_router_greedy_bwd(
            ptr(rw), ptr(tw), ptr(ids), ptr(g_tw), ptr(g_rw), None, T, E, K, scoring, int(norm_topk_prob),
            float(scaling), ptr(gl), current_stream(),
        ),
        "xtb_router_greedy_bwd",
    )
    return gl


@_router_greedy_bwd_op.register_fake
def _(rw, tw, ids, g_tw, g_rw, scoring, norm_topk_prob, scaling):
    return torch.empty_like(rw)


def replay_ids_arg(replay: Tensor, T: int, K: int, device) -> tuple[Tensor, int]:
    """``(ids, row_stride)`` for the replay entries: the reference's ``rollout_routed_experts`` slice, an int64 ``[T, K]``
    tensor on the logits' device (other dtypes raise, as the reference's ``gather`` does).  A view whose last stride is 1
    (the ``[:, layer_idx, :]`` slice of the ``[S, L, K]`` tensor) is passed with its row stride and no copy; any other
    layout is made contiguous first."""
    if replay.dtype != torch.int64:
        raise TypeError(f"rollout_routed_experts must be int64 (got {replay.dtype})")
    if replay.dim() != 2 or tuple(replay.shape) != (T, K):
        raise ValueError(f"rollout_routed_experts must be [{T}, {K}] (got {list(replay.shape)})")
    if replay.device != device:
        raise ValueError(f"rollout_routed_experts is on {replay.device}, the logits on {device}")
    if T > 0 and not (replay.stride(1) == 1 and replay.stride(0) >= K):
        replay = replay.contiguous()
    return replay, (replay.stride(0) if T > 0 else K)


@torch.library.custom_op("xtuner_b200::router_greedy_replay", mutates_args=())
def _router_greedy_replay_op(
    logits: Tensor, replay: Tensor, top_k: int, scoring: int, norm_topk_prob: bool, scaling: float
) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    lib = _capi.ensure_init()
    T, E = logits.shape
    K = top_k
    dev = logits.device
    ids_in, stride = replay_ids_arg(replay, T, K, dev)
    rw = torch.empty((T, E), dtype=torch.float32, device=dev)
    tw = torch.empty((T, K), dtype=torch.float32, device=dev)
    ids = torch.empty((T, K), dtype=torch.int64, device=dev)
    ids32 = torch.empty((T, K), dtype=torch.int32, device=dev)
    tpe = torch.empty((E,), dtype=torch.int64, device=dev)
    check(
        lib.xtb_router_greedy_replay(
            ptr(logits), ptr(ids_in), stride, T, E, K, scoring, int(norm_topk_prob), float(scaling), ptr(rw), ptr(tw),
            ptr(ids), ptr(ids32), ptr(tpe), None, current_stream(),
        ),
        "xtb_router_greedy_replay",
    )
    return rw, tw, ids, ids32, tpe


@_router_greedy_replay_op.register_fake
def _(logits, replay, top_k, scoring, norm_topk_prob, scaling):
    T, E = logits.shape
    K = top_k
    return (
        logits.new_empty((T, E)),
        logits.new_empty((T, K)),
        logits.new_empty((T, K), dtype=torch.int64),
        logits.new_empty((T, K), dtype=torch.int32),
        logits.new_empty((E,), dtype=torch.int64),
    )


class _GreedyRoute(torch.autograd.Function):
    """Routing, or with ``replay`` (rollout-routed experts) the replay op; one backward for both: it reads the saved ids."""

    @staticmethod
    def forward(ctx, logits: Tensor, top_k: int, scoring: int, norm: bool, scaling: float, replay: Optional[Tensor] = None):
        if replay is None:
            rw, tw, ids, ids32, tpe = _router_greedy_op(logits, top_k, scoring, norm, scaling)
        else:
            rw, tw, ids, ids32, tpe = _router_greedy_replay_op(logits, replay, top_k, scoring, norm, scaling)
        ctx.save_for_backward(rw, tw, ids)
        ctx.cfg = (scoring, norm, scaling)
        ctx.mark_non_differentiable(ids, ids32, tpe)
        return rw, tw, ids, ids32, tpe

    @staticmethod
    def backward(ctx, g_rw, g_tw, _a, _b, _c):
        rw, tw, ids = ctx.saved_tensors
        scoring, norm, scaling = ctx.cfg
        g_rw = None if g_rw is None else g_rw.contiguous()
        g_tw = None if g_tw is None else g_tw.contiguous()
        return _router_greedy_bwd_op(rw, tw, ids, g_tw, g_rw, scoring, norm, scaling), None, None, None, None, None


def greedy_route(
    logits: Tensor, top_k: int, norm_topk_prob: bool = True, router_scaling_factor: float = 1.0,
    scoring_func: str = "softmax", rollout_routed_experts: Tensor | None = None,
):
    """Functional form; returns ``(RouterResults, topk_ids_int32)``.  With ``rollout_routed_experts`` (int64 ``[T, K]``)
    the weights are gathered at those ids instead of a top-k (routing replay, greedy.py:74-78)."""
    if not logits.is_cuda:
        raise _capi.XtbError("greedy_route needs CUDA tensors (no CPU fallback)")
    if logits.dtype != torch.float32:
        logits = logits.float()  # F.softmax(..., dtype=torch.float) in the reference (greedy.py:73)
    rw, tw, ids, ids32, tpe = _GreedyRoute.apply(
        logits.contiguous(), top_k, SCORING[scoring_func], norm_topk_prob, router_scaling_factor, rollout_routed_experts
    )
    res: RouterResults = {
        "logits": logits,
        "router_weights": rw,
        "topk_weights": tw,
        "topk_ids": ids,
        "topkens_per_expert": tpe,
    }
    return res, ids32


class GreedyRouter(nn.Module):
    """Drop-in for ``xtuner.v1.module.router.greedy.GreedyRouter`` (same constructor keywords)."""

    def __init__(
        self,
        *,
        n_routed_experts: int,
        num_experts_per_tok: int,
        norm_topk_prob: bool = True,
        scoring_func: Literal["sigmoid", "softmax"] = "softmax",
        router_scaling_factor: float = 1.0,
    ):
        super().__init__()
        self.n_routed_experts = n_routed_experts
        self.top_k = num_experts_per_tok
        self.norm_topk_prob = norm_topk_prob
        self.scoring_func = scoring_func
        self.router_scaling_factor = router_scaling_factor
        self.last_topk_ids_i32: Tensor | None = None  # int32 copy for the dispatcher (saves a cast kernel)

    def forward(self, logits: Tensor, rollout_routed_experts: Tensor | None = None) -> RouterResults:
        assert logits.shape[1] == self.n_routed_experts
        # the replay ids only when given: the routing call keeps greedy_route's five-argument form
        replay = {} if rollout_routed_experts is None else {"rollout_routed_experts": rollout_routed_experts}
        res, ids32 = greedy_route(
            logits, self.top_k, self.norm_topk_prob, self.router_scaling_factor, self.scoring_func, **replay
        )
        self.last_topk_ids_i32 = ids32
        return res


@torch.library.custom_op("xtuner_b200::router_noaux", mutates_args=())
def _router_noaux_op(
    logits: Tensor, bias: Tensor, top_k: int, n_group: int, topk_group: int, norm_topk_prob: bool, scaling: float
) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    lib = _capi.ensure_init()
    T, E = logits.shape
    dev = logits.device
    rw = torch.empty((T, E), dtype=torch.float32, device=dev)
    tw = torch.empty((T, top_k), dtype=torch.float32, device=dev)
    ids = torch.empty((T, top_k), dtype=torch.int64, device=dev)
    ids32 = torch.empty((T, top_k), dtype=torch.int32, device=dev)
    tpe = torch.empty((E,), dtype=torch.float32, device=dev)
    check(
        lib.xtb_router_noaux(
            ptr(logits), ptr(bias), T, E, top_k, n_group, topk_group, int(norm_topk_prob), float(scaling), ptr(rw),
            ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), current_stream(),
        ),
        "xtb_router_noaux",
    )
    return rw, tw, ids, ids32, tpe


@_router_noaux_op.register_fake
def _(logits, bias, top_k, n_group, topk_group, norm_topk_prob, scaling):
    T, E = logits.shape
    return (
        logits.new_empty((T, E)),
        logits.new_empty((T, top_k)),
        logits.new_empty((T, top_k), dtype=torch.int64),
        logits.new_empty((T, top_k), dtype=torch.int32),
        logits.new_empty((E,)),
    )


@torch.library.custom_op("xtuner_b200::router_noaux_replay", mutates_args=())
def _router_noaux_replay_op(
    logits: Tensor, bias: Tensor, replay: Tensor, top_k: int, n_group: int, topk_group: int, norm_topk_prob: bool,
    scaling: float,
) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    lib = _capi.ensure_init()
    T, E = logits.shape
    K = top_k
    dev = logits.device
    ids_in, stride = replay_ids_arg(replay, T, K, dev)
    rw = torch.empty((T, E), dtype=torch.float32, device=dev)
    tw = torch.empty((T, K), dtype=torch.float32, device=dev)
    ids = torch.empty((T, K), dtype=torch.int64, device=dev)
    ids32 = torch.empty((T, K), dtype=torch.int32, device=dev)
    tpe = torch.empty((E,), dtype=torch.float32, device=dev)
    check(
        lib.xtb_router_noaux_replay(
            ptr(logits), ptr(bias), ptr(ids_in), stride, T, E, K, n_group, topk_group, int(norm_topk_prob),
            float(scaling), ptr(rw), ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), current_stream(),
        ),
        "xtb_router_noaux_replay",
    )
    return rw, tw, ids, ids32, tpe


@_router_noaux_replay_op.register_fake
def _(logits, bias, replay, top_k, n_group, topk_group, norm_topk_prob, scaling):
    T, E = logits.shape
    K = top_k
    return (
        logits.new_empty((T, E)),
        logits.new_empty((T, K)),
        logits.new_empty((T, K), dtype=torch.int64),
        logits.new_empty((T, K), dtype=torch.int32),
        logits.new_empty((E,)),
    )


def noaux_group_spec(n_group: int, topk_group: int) -> int:
    """The ``group_spec`` argument of xtb_router_noaux_bwd (XTB_NOAUX_GROUP_SPEC in the header): 0 without a group
    mask, else n_group | topk_group << 8."""
    return 0 if n_group == topk_group else n_group | (topk_group << 8)


@torch.library.custom_op("xtuner_b200::router_noaux_bwd", mutates_args=())
def _router_noaux_bwd_op(
    logits: Tensor, bias: Tensor, rw: Tensor, tw: Tensor, ids: Tensor, g_tw: Optional[Tensor], g_rw: Optional[Tensor],
    group_spec: int, norm_topk_prob: bool, scaling: float,
) -> Tensor:
    lib = _capi.ensure_init()
    T, E = logits.shape
    gl = torch.empty_like(logits)
    check(
        lib.xtb_router_noaux_bwd(
            ptr(logits), ptr(bias), ptr(rw), ptr(tw), ptr(ids), ptr(g_tw), ptr(g_rw), T, E, tw.shape[1],
            group_spec, int(norm_topk_prob), float(scaling), ptr(gl), current_stream(),
        ),
        "xtb_router_noaux_bwd",
    )
    return gl


@_router_noaux_bwd_op.register_fake
def _(logits, bias, rw, tw, ids, g_tw, g_rw, group_spec, norm_topk_prob, scaling):
    return torch.empty_like(logits)


class _NoAuxRoute(torch.autograd.Function):
    """``logits`` -> (router_weights, topk_weights) stay differentiable (the reference's autograd through
    noaux_router.py:80-134); the bias is a buffer (updated outside autograd, model/moe/moe.py:334-398)."""

    @staticmethod
    def forward(ctx, logits, bias, top_k, n_group, topk_group, norm, scaling, replay=None):
        if replay is None:
            rw, tw, ids, ids32, tpe = _router_noaux_op(logits, bias, top_k, n_group, topk_group, norm, scaling)
        else:  # routing replay: one backward for both, it reads the saved ids
            rw, tw, ids, ids32, tpe = _router_noaux_replay_op(logits, bias, replay, top_k, n_group, topk_group, norm,
                                                              scaling)
        ctx.save_for_backward(logits, bias, rw, tw, ids)
        ctx.cfg = (noaux_group_spec(n_group, topk_group), norm, scaling)
        ctx.mark_non_differentiable(ids, ids32, tpe)
        return rw, tw, ids, ids32, tpe

    @staticmethod
    def backward(ctx, g_rw, g_tw, _a, _b, _c):
        logits, bias, rw, tw, ids = ctx.saved_tensors
        group_spec, norm, scaling = ctx.cfg
        g_rw = None if g_rw is None else g_rw.contiguous()
        g_tw = None if g_tw is None else g_tw.contiguous()
        gl = _router_noaux_bwd_op(logits, bias, rw, tw, ids, g_tw, g_rw, group_spec, norm, scaling)
        return gl, None, None, None, None, None, None, None


class NoAuxRouter(nn.Module):
    """Drop-in for ``xtuner.v1.module.router.noaux_router.NoAuxRouter`` (same constructor keywords; sigmoid scoring,
    the only one the reference implements, ``noaux_router.py:79-83``)."""

    def __init__(
        self,
        *,
        n_routed_experts: int,
        num_experts_per_tok: int,
        router_scaling_factor: float,
        scoring_func: Literal["sigmoid", "softmax"],
        n_group: int,
        topk_group: int,
        norm_topk_prob: bool = True,
        router_bias_update_speed: float = 0.001,
    ):
        super().__init__()
        if scoring_func != "sigmoid":
            raise NotImplementedError(f"insupportable scoring function for MoE gating: {scoring_func}")
        self.top_k = num_experts_per_tok
        self.n_routed_experts = n_routed_experts
        self.router_scaling_factor = router_scaling_factor
        self.scoring_func = scoring_func
        self.n_group = n_group
        self.topk_group = topk_group
        self.norm_topk_prob = norm_topk_prob
        self.register_buffer("e_score_correction_bias", torch.zeros((n_routed_experts,), dtype=torch.float32))
        self.last_topk_ids_i32: Tensor | None = None

    def forward(self, logits: Tensor, rollout_routed_experts: Tensor | None = None) -> RouterResults:
        if not logits.is_cuda:
            raise _capi.XtbError("NoAuxRouter needs CUDA tensors (no CPU fallback)")
        lg = logits.float().contiguous()
        # the reference adds the bias to fp32 scores (type promotion, noaux_router.py:85): a buffer that a blanket
        # `.to(bfloat16)` converted still contributes its value in fp32
        bias = self.e_score_correction_bias.detach().to(torch.float32).contiguous()
        rw, tw, ids, ids32, tpe = _NoAuxRoute.apply(  # with rollout_routed_experts: replay (noaux_router.py:114-121)
            lg, bias, self.top_k, self.n_group, self.topk_group, self.norm_topk_prob, self.router_scaling_factor,
            rollout_routed_experts,
        )
        self.last_topk_ids_i32 = ids32
        return {"logits": logits, "router_weights": rw, "topk_weights": tw, "topk_ids": ids, "topkens_per_expert": tpe}
