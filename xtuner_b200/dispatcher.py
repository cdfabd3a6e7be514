"""``FusedDispatcher``: the six-phase dispatcher protocol of the reference
(``xtuner/v1/module/dispatcher/base.py:86-176``) for ep=1, backed by the sm_90a dispatch/combine kernels.

Same keyword-only methods and TypedDict results as ``NaiveDispatcher`` (``base.py:222-539``); the real
work is in ``dispatch_postprocess`` (bucket + gather, which also yields ``tokens_per_expert`` from the
same pass instead of a second ``torch.histc``, base.py:398) and ``combine_preprocess`` (weighted combine).
``async_op=True`` (intra-layer micro-batch overlap) is a 'next' row (SURVEY.md §8f-1) and raises, exactly
like ``NaiveDispatcher`` does without ExpertTP (base.py:256-257)."""
from __future__ import annotations

from typing import Literal, Optional, TypedDict

import torch

from . import ops


class PreDispatchResult(TypedDict):
    hidden_states: torch.Tensor
    topk_ids: torch.Tensor


class DispatchResult(TypedDict):
    hidden_states: torch.Tensor
    topk_ids: torch.Tensor
    topk_weights: torch.Tensor


class PostDispatchResult(TypedDict):
    hidden_states: torch.Tensor
    tokens_per_expert: torch.Tensor
    row_ids_map: torch.Tensor


class PreCombineResult(TypedDict):
    hidden_states: torch.Tensor


class CombineResult(TypedDict):
    hidden_states: torch.Tensor


class PostCombineResult(TypedDict):
    hidden_states: torch.Tensor


class FusedDispatcher:
    def __init__(
        self,
        *,
        n_routed_experts: int,
        process_group: Optional["torch.distributed.ProcessGroup"] = None,
        tp_group: Optional["torch.distributed.ProcessGroup"] = None,
        training_dtype: Literal["fp8", "bf16"] = "bf16",
        generate_dtype: Literal["fp8", "bf16"] = "bf16",
    ):
        if process_group is not None and process_group.size() != 1:
            raise ValueError("FusedDispatcher is the ep=1 dispatcher (like NaiveDispatcher, base.py:247-248)")
        if tp_group is not None and tp_group.size() > 1:
            raise NotImplementedError("ExpertTP is out of scope (SURVEY.md §2.4 C10)")
        self._n_routed_experts = n_routed_experts
        self._process_group = process_group
        self._training_dtype = training_dtype
        self._generate_dtype = generate_dtype

    @staticmethod
    def _no_async(async_op: bool) -> None:
        if async_op:
            raise NotImplementedError("FusedDispatcher async_op=True (intra-layer micro-batching) is not built yet")

    def dispatch_preprocess(self, *, hidden_states, topk_ids, topk_weights, async_op: bool = False) -> PreDispatchResult:
        self._no_async(async_op)
        return PreDispatchResult(hidden_states=hidden_states, topk_ids=topk_ids)

    def dispatch(self, *, pre_dispatched, topk_weights, async_op: bool = False, decoding: bool = False) -> DispatchResult:
        self._no_async(async_op)
        return DispatchResult(
            hidden_states=pre_dispatched["hidden_states"], topk_ids=pre_dispatched["topk_ids"], topk_weights=topk_weights
        )

    def dispatch_postprocess(self, *, pre_dispatched, dispatched, async_op: bool = False, decoding: bool = False) -> PostDispatchResult:
        self._no_async(async_op)
        if decoding:
            raise NotImplementedError
        hidden_states, row_id_map, _sorted, tokens_per_expert = ops.permute(
            dispatched["hidden_states"], pre_dispatched["topk_ids"], n_experts=self._n_routed_experts, return_extra=True
        )
        return PostDispatchResult(hidden_states=hidden_states, row_ids_map=row_id_map, tokens_per_expert=tokens_per_expert)

    def combine_preprocess(self, *, hidden_states, pre_dispatched, dispatched, post_dispatched, async_op: bool = False, decoding: bool = False) -> PreCombineResult:
        self._no_async(async_op)
        if decoding:
            raise NotImplementedError("FusedDispatcher does not support decoding.")
        out = ops.unpermute(hidden_states, post_dispatched["row_ids_map"], probs=dispatched["topk_weights"])
        return PreCombineResult(hidden_states=out)

    def combine(self, *, pre_dispatched, dispatched, post_dispatched, pre_combined, async_op: bool = False, decoding: bool = False) -> CombineResult:
        self._no_async(async_op)
        if decoding:
            raise NotImplementedError
        return CombineResult(hidden_states=pre_combined["hidden_states"])

    def combine_postprocess(self, *, pre_dispatched, dispatched, post_dispatched, pre_combined, combined, async_op: bool = False) -> PostCombineResult:
        self._no_async(async_op)
        return PostCombineResult(hidden_states=combined["hidden_states"])
