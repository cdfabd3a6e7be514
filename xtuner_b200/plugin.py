"""Installs the H100 path into a reference XTuner V1 model without editing the reference tree (INTEGRATION.md §2).

``convert_model(model)`` walks the reference's modules and, for every ``MoEDecoderLayer``
(``xtuner/v1/module/decoder_layer/moe_decoder_layer.py:203``):

* replaces ``layer.dispatcher`` (``NaiveDispatcher`` for ep=1, built at ``moe_decoder_layer.py:300-309``) with
  :class:`xtuner_b200.dispatcher.FusedDispatcher`;
* replaces ``layer.gate.router`` (``GreedyRouter`` / ``NoAuxRouter``) with this package's router of the same
  configuration (state — e.g. ``e_score_correction_bias`` — is copied);
* rebinds the module-level ``group_gemm`` used by ``GroupedLinear`` (imported by value at
  ``module/grouped_linear/moe_group_linear.py:10``) and the MoE activation (``experts.moe_act``).

With ``fused=True`` the MoE half of every eligible layer (``post_attention_layernorm`` -> gate -> router -> dispatch ->
experts -> combine -> ``* hidden_factor + residual``, ``moe_decoder_layer.py:668-705,411-488``) additionally runs as ONE
autograd node (:func:`xtuner_b200.fused.fused_moe_block`), the form ``bench.py`` measures; the per-op classes above stay
installed for the paths the fused node does not cover (micro-batched forward, rollout-routed experts).

Everything else of the model (attention, norms, lm_head, FSDP wrapping, checkpoint keys) is untouched;
``install_lm_head_loss()`` separately moves the lm_head cross-entropy onto this package's kernels; parameters keep
their names, so state dicts and DCP checkpoints stay compatible.  ``restore_model`` undoes the conversion.
"""
from __future__ import annotations

import importlib
import types
from typing import Any

import torch
from torch import nn

from . import fused as _fused
from . import ops
from .dispatcher import FusedDispatcher
from .router import GreedyRouter, NoAuxRouter

_SAVED = "_xtuner_b200_saved"


def _router_convertible(router: nn.Module) -> bool:
    return type(router).__name__ in ("GreedyRouter", "NoAuxRouter")


def _gg_eligible(x, weights) -> bool:
    """what ``ops.group_gemm`` (xtb_group_gemm_nt/nn/tn) covers: plain bf16 CUDA operands, widths multiples of 128"""
    import torch

    return (type(x) is torch.Tensor and x.is_cuda and x.dtype == torch.bfloat16 and weights.dtype == torch.bfloat16
            and weights.dim() == 3 and weights.shape[1] % 128 == 0 and weights.shape[2] % 128 == 0)


def _group_gemm_dispatch(original):
    """Process-wide replacement for ``moe_group_linear.group_gemm``: inputs our kernels cover go to ``ops.group_gemm``;
    anything else — fp8 / fp32 experts, odd shapes, layers whose dispatcher was deliberately left alone but which share
    ``GroupedLinear`` — keeps the reference's own implementation."""

    def group_gemm(x, weights, split_sizes):
        if _gg_eligible(x, weights):
            return ops.group_gemm(x, weights, split_sizes)
        return original(x, weights, split_sizes)

    group_gemm.__wrapped__ = original
    return group_gemm


def _convert_router(router: nn.Module) -> nn.Module:
    name = type(router).__name__
    if name == "GreedyRouter":
        new = GreedyRouter(
            n_routed_experts=router.n_routed_experts, num_experts_per_tok=router.top_k, norm_topk_prob=router.norm_topk_prob,
            scoring_func=router.scoring_func, router_scaling_factor=router.router_scaling_factor,
        )
    elif name == "NoAuxRouter":
        new = NoAuxRouter(
            n_routed_experts=router.n_routed_experts, num_experts_per_tok=router.top_k,
            router_scaling_factor=router.router_scaling_factor, scoring_func=router.scoring_func, n_group=router.n_group,
            topk_group=router.topk_group, norm_topk_prob=router.norm_topk_prob,
        )
        new.e_score_correction_bias = router.e_score_correction_bias  # share the buffer (bias updates keep working)
    else:
        raise NotImplementedError(f"router {name} has no H100 counterpart (GreedyRouter, NoAuxRouter)")
    return new


def _local(t):
    return t.to_local() if hasattr(t, "to_local") else t


def _fused_eligible(layer: nn.Module) -> bool:
    """What ``fused_moe_block`` computes: RMSNorm("default") -> fp32 gate without bias -> GreedyRouter -> SwiGLU experts
    without bias, no shared experts."""
    norm = getattr(layer, "post_attention_layernorm", None)
    gate, experts = layer.gate, layer.experts
    return (
        type(layer.gate.router).__name__ == "GreedyRouter"
        and getattr(layer, "n_shared_experts", 0) == 0
        and norm is not None and getattr(norm, "_type", "default") == "default" and hasattr(norm, "variance_epsilon")
        and not getattr(gate, "gate_bias", False) and getattr(gate, "router_compute_dtype", "float32") == "float32"
        and hasattr(experts, "fused_w1w3") and hasattr(experts, "fused_w2")
        and not getattr(experts.fused_w1w3, "moe_bias", False) and not getattr(experts.fused_w2, "moe_bias", False)
    )


def _fused_layer_forward(self, hidden_states, seq_ctx, position_embeddings):
    """Replacement for ``MoEDecoderLayer._forward`` (``moe_decoder_layer.py:392-488``): the attention half is the
    reference's own modules (``_pre_moe_forward`` lines 634-666), the MoE half one fused autograd node."""
    if getattr(seq_ctx, "rollout_routed_experts", None) is not None:
        return type(self)._forward(self, hidden_states, seq_ctx, position_embeddings)  # RL replay routing: per-op path
    residual = hidden_states
    hidden_states = self.input_layernorm(hidden_states)
    attn_outputs = self.self_attn(hidden_states=hidden_states, position_embeddings=position_embeddings, seq_ctx=seq_ctx)
    hidden_states = residual + attn_outputs["projected_output"]
    router = self.gate.router
    out, rr = _fused.fused_moe_block(
        hidden_states, _local(self.post_attention_layernorm.weight), self.post_attention_layernorm.variance_epsilon,
        _local(self.gate.weight), _local(self.experts.fused_w1w3.weight), _local(self.experts.fused_w2.weight),
        top_k=router.top_k, norm_topk_prob=router.norm_topk_prob, router_scaling_factor=router.router_scaling_factor,
        hidden_factor=self.hidden_factor, scoring_func=router.scoring_func,
    )
    return out, rr["logits"], rr["router_weights"], rr["topk_ids"]


def convert_model(model: nn.Module, *, swiglu: bool = True, fused: bool = False, ep: "bool | str" = False) -> int:
    """Returns the number of MoE decoder layers converted.  ``ep`` also converts ``TorchAll2AllDispatcher`` layers (expert
    parallel): ``True`` / ``"nccl"`` -> :class:`All2AllDispatcher` (the reference's six phases, NCCL all-to-all, our
    permute/unpermute kernels); ``"peer"`` -> :class:`PeerAll2AllDispatcher` (device-side split sizes, peer-memory pull
    kernels, no host read; needs symmetric memory over the EP group).  Both are covered by ``tests/test_gpu_comm.py`` with
    ``XTB_TEST_EP=1`` on >= 2 GPUs."""
    if ep not in (False, True, "nccl", "peer"):
        raise ValueError(f"convert_model: ep must be False, True, 'nccl' or 'peer' (got {ep!r})")
    n = 0
    for layer in model.modules():
        # the layer itself, not a wrapper that forwards attribute reads to it (torch's CheckpointWrapper under the
        # reference's fully_shard does): `dispatcher` is a plain attribute, `gate` / `experts` are sub-modules
        if not ("dispatcher" in vars(layer) and "gate" in layer._modules and "experts" in layer._modules):
            continue
        disp = layer.dispatcher
        kind = type(disp).__name__
        if not _router_convertible(layer.gate.router):
            continue  # grouped routers etc.: the layer is left entirely on the reference path (nothing is half-converted)
        if kind == "TorchAll2AllDispatcher" and ep and getattr(disp, "_expert_tp", None) is None:
            # ep > 1 (reference key dispatcher="all2all", module/dispatcher/__init__.py:30-96): same six phases on our ops
            from .ep_dispatcher import All2AllDispatcher, PeerAll2AllDispatcher

            saved: dict[str, Any] = {"dispatcher": disp, "router": layer.gate.router}
            layer.dispatcher = (PeerAll2AllDispatcher if ep == "peer" else All2AllDispatcher)(
                n_routed_experts=disp._n_routed_experts, process_group=disp._process_group,
                training_dtype=disp._training_dtype, generate_dtype=disp._generate_dtype,
            )
        elif kind == "NaiveDispatcher":
            saved = {"dispatcher": disp, "router": layer.gate.router}
            layer.dispatcher = FusedDispatcher(
                n_routed_experts=disp._n_routed_experts, process_group=disp._process_group,
                training_dtype=disp._training_dtype, generate_dtype=disp._generate_dtype,
            )
        else:
            continue  # DeepEP / AGRS / ExpertTP dispatchers are left alone
        try:
            layer.gate.router = _convert_router(layer.gate.router)
        except Exception:
            layer.dispatcher = disp  # roll the layer back before the error leaves
            raise
        if swiglu and getattr(layer.experts, "moe_act", None) is not None and getattr(layer.experts.moe_act, "__name__", "") == "native_swiglu":
            saved["moe_act"] = layer.experts.moe_act
            layer.experts.moe_act = ops.swiglu
        if fused and kind == "NaiveDispatcher" and _fused_eligible(layer):
            saved["fused_forward"] = True
            layer._forward = types.MethodType(_fused_layer_forward, layer)  # instance attribute shadows the class method
        setattr(layer, _SAVED, saved)
        n += 1
    if n:
        mgl = importlib.import_module("xtuner.v1.module.grouped_linear.moe_group_linear")
        if not hasattr(mgl, _SAVED):
            setattr(mgl, _SAVED, mgl.group_gemm)
        mgl.group_gemm = _group_gemm_dispatch(getattr(mgl, _SAVED))
    return n


def restore_model(model: nn.Module) -> None:
    for layer in model.modules():
        saved = vars(layer).get(_SAVED)  # the layer's own attribute, not one a wrapper forwards
        if not saved:
            continue
        layer.dispatcher = saved["dispatcher"]
        layer.gate.router = saved["router"]
        if "moe_act" in saved:
            layer.experts.moe_act = saved["moe_act"]
        if saved.get("fused_forward"):
            del layer._forward
        delattr(layer, _SAVED)
    try:
        mgl = importlib.import_module("xtuner.v1.module.grouped_linear.moe_group_linear")
        if hasattr(mgl, _SAVED):
            mgl.group_gemm = getattr(mgl, _SAVED)
            delattr(mgl, _SAVED)
    except ImportError:
        pass


# ======================================================================================================
# exchange steps: FSDP comm objects and the Ulysses all-to-all
# ======================================================================================================


def install_fsdp_comm(model: nn.Module, *, all_gather: bool = True, reduce_scatter: bool = True) -> int:
    """Installs the peer-memory collectives on every FSDP2 module of ``model`` (the per-layer ``fully_shard`` wrappers
    the reference creates at ``xtuner/v1/model/moe/moe.py:1211-1217`` and the root, ``:1225-1313``) through torch's own
    extension point ``FSDPModule.set_custom_all_gather / set_custom_reduce_scatter``.  Returns the number of modules."""
    from torch.distributed.fsdp import FSDPModule

    from .comm import P2PAllGather, P2PReduceScatter

    n = 0
    for m in model.modules():
        if isinstance(m, FSDPModule):
            if all_gather:
                m.set_custom_all_gather(P2PAllGather())
            if reduce_scatter:
                m.set_custom_reduce_scatter(P2PReduceScatter())
            n += 1
    return n


def install_ulysses() -> None:
    """Rebinds ``ulysses_all_to_all`` where the reference imported it by value (``module/attention/mha.py:19``), so the
    SP block of ``MultiHeadAttention.forward`` (``mha.py:365-390,421-427``) uses the peer-memory exchange."""
    from .comm import ulysses_all_to_all

    mha = importlib.import_module("xtuner.v1.module.attention.mha")
    if not hasattr(mha, _SAVED):
        setattr(mha, _SAVED, mha.ulysses_all_to_all)
    mha.ulysses_all_to_all = ulysses_all_to_all


def uninstall_ulysses() -> None:
    mha = importlib.import_module("xtuner.v1.module.attention.mha")
    if hasattr(mha, _SAVED):
        mha.ulysses_all_to_all = getattr(mha, _SAVED)
        delattr(mha, _SAVED)


# ======================================================================================================
# lm_head + cross-entropy (f4)
# ======================================================================================================


def _lm_head_eligible(ctx, cls, hidden_states, head_weight, head_bias) -> bool:
    """what ``ops.lm_head_cross_entropy`` computes: the plain context (``MTPLossContext`` subclasses it with its own
    ``loss_fn``), no bias, bf16 CUDA hidden states and weight (``fp32_lm_head`` gives fp32), widths multiples of 128"""
    kw = ctx.loss_kwargs
    return (type(ctx) is cls and head_bias is None and kw is not None and kw.loss_weight is not None
            and all(type(t) in (torch.Tensor, nn.Parameter) and _on_device(t) and t.dtype == torch.bfloat16
                    for t in (hidden_states, head_weight))
            and head_weight.dim() == 2 and head_weight.shape[0] % 128 == 0 and head_weight.shape[1] % 128 == 0)


def _lm_head_loss(ctx, hidden_states, head_weight, loss_kwargs, chunk_size):
    loss = ops.lm_head_cross_entropy(hidden_states, head_weight, loss_kwargs.shifted_labels, loss_kwargs.loss_weight,
                                     ctx.loss_cfg.ignore_idx, chunk_size)
    return loss, (None, {})


def install_lm_head_loss() -> None:
    """Rebinds ``LMHeadLossContext.eager_mode`` and ``.chunk_mode`` (``xtuner/v1/loss/ce_loss.py``) so that modes
    ``"eager"`` and ``"chunk"`` run :func:`ops.lm_head_cross_entropy`: the logits GEMM with the cross-entropy epilogue, the
    loss and both gradients on this package's kernels, with the reference's roundings.  Calls it does not cover go to the
    original methods: subclasses such as ``MTPLossContext``, mode ``"liger"``, a head bias, fp32 or non-CUDA tensors,
    ``V`` or ``H`` not a multiple of 128, and chunk mode over a batch of more than one sequence (``ChunkLoss`` splits
    along the sequence dimension of each).

    Opt-in because it changes one output: like chunk mode, the served calls return ``(loss, (None, {}))``, so in eager
    mode the fp32 logits that the reference returns, and that end up in ``MoEModelOutputs.logits``, are not produced."""
    ce = importlib.import_module("xtuner.v1.loss.ce_loss")
    cls = ce.LMHeadLossContext
    if _SAVED in vars(cls):
        return
    orig_eager, orig_chunk = vars(cls)["eager_mode"], vars(cls)["chunk_mode"]

    def eager_mode(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if self.loss_cfg.mode == "eager" and _lm_head_eligible(self, cls, hidden_states, head_weight, head_bias):
            return _lm_head_loss(self, hidden_states, head_weight, loss_kwargs, None)
        return orig_eager(self, hidden_states, head_weight, head_bias, loss_kwargs)

    def chunk_mode(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if (self.loss_cfg.mode == "chunk" and self.loss_cfg.chunk_size is not None
                and (hidden_states.dim() == 2 or hidden_states.shape[0] == 1)
                and _lm_head_eligible(self, cls, hidden_states, head_weight, head_bias)):
            return _lm_head_loss(self, hidden_states, head_weight, loss_kwargs, self.loss_cfg.chunk_size)
        return orig_chunk(self, hidden_states, head_weight, head_bias, loss_kwargs)

    eager_mode.__wrapped__, chunk_mode.__wrapped__ = orig_eager, orig_chunk
    setattr(cls, _SAVED, (orig_eager, orig_chunk))
    cls.eager_mode, cls.chunk_mode = eager_mode, chunk_mode


def uninstall_lm_head_loss() -> None:
    ce = importlib.import_module("xtuner.v1.loss.ce_loss")
    cls = ce.LMHeadLossContext
    if _SAVED in vars(cls):
        cls.eager_mode, cls.chunk_mode = vars(cls)[_SAVED]
        delattr(cls, _SAVED)


# ======================================================================================================
# fp8 FSDP all-gather (row a15): the cast in front of the gather
# ======================================================================================================


def _on_device(t) -> bool:
    return t.is_cuda


def _fp8_eligible(t, block_size, float8_dtype) -> bool:
    """shapes / dtypes ``csrc/fp8.cu`` takes; everything else (shard rows % 128 == 64, < 128 rows, other fp8 formats) stays on
    the reference's own code"""
    return (isinstance(t, torch.Tensor) and _on_device(t) and block_size == 128 and float8_dtype == torch.float8_e4m3fn
            and t.dtype in (torch.float32, torch.bfloat16) and t.shape[-2] >= 128 and t.shape[-2] % 128 == 0 and t.shape[-1] % 128 == 0)


def install_fp8_cast() -> None:
    """Rebinds the two pure-arithmetic steps of the reference's tile-wise fp8 FSDP all-gather to ``csrc/fp8.cu``:
    ``cast_to_per_block_fp8_with_scales`` — called by ``WeightWithDynamicTilewiseFloat8CastTensor.fsdp_pre_all_gather``
    (``float8/fsdp_utils.py:379-409``) on the local fp32 shard in front of every all-gather — and
    ``tensor_to_per_block_fp8_scales`` (``:75-116``, the per-step scale precompute) when no cross-rank amax reduction is
    involved.  The module functions are looked up by name at call time, so the rebind takes effect for existing tensors.
    Kernels: bit-exact against reference-made vectors on an H100 (``tests/test_gpu_fp8.py``); this glue: CPU-tested against
    the reference's functions (``tests/test_plugin_reference_cpu.py``); the two together have not run inside an fp8 training
    step (the reference's fp8 grouped GEMM wheel is absent here)."""
    fu = importlib.import_module("xtuner.v1.float8.fsdp_utils")
    if hasattr(fu, _SAVED):
        return
    orig_cast, orig_scales = fu.cast_to_per_block_fp8_with_scales, fu.tensor_to_per_block_fp8_scales

    def cast_to_per_block_fp8_with_scales(tensor, scales, block_size=128, float8_dtype=torch.float8_e4m3fn):
        if tensor.dim() == 2 and _fp8_eligible(tensor, block_size, float8_dtype):
            return ops.fp8_block_cast(tensor, scales.float(), block_size)
        return orig_cast(tensor, scales, block_size, float8_dtype)

    def tensor_to_per_block_fp8_scales(tensor, reduce_mesh=None, float8_dtype=torch.float8_e4m3fn, block_size=128):
        local = tensor.to_local() if hasattr(tensor, "to_local") else tensor
        if reduce_mesh is None and local.dim() == 3 and _fp8_eligible(local, block_size, float8_dtype):
            return ops.fp8_block_scales(local, block_size)
        return orig_scales(tensor, reduce_mesh, float8_dtype, block_size)

    setattr(fu, _SAVED, (orig_cast, orig_scales))
    fu.cast_to_per_block_fp8_with_scales = cast_to_per_block_fp8_with_scales
    fu.tensor_to_per_block_fp8_scales = tensor_to_per_block_fp8_scales


def uninstall_fp8_cast() -> None:
    fu = importlib.import_module("xtuner.v1.float8.fsdp_utils")
    if hasattr(fu, _SAVED):
        fu.cast_to_per_block_fp8_with_scales, fu.tensor_to_per_block_fp8_scales = getattr(fu, _SAVED)
        delattr(fu, _SAVED)
