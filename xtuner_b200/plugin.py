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
autograd node (:func:`xtuner_b200.fused.fused_moe_block`), the form ``bench.py`` measures, rollout-routed experts (RL
routing replay) included; the per-op classes above stay installed for the path the fused node does not cover
(micro-batched forward).  ``recompute="act"`` or ``"experts"`` (with ``fused=True`` only) has every fused node rebuild
some of its expert intermediates in the backward instead of keeping them (:data:`xtuner_b200.fused.RECOMPUTE`): less
activation memory for the same results, without checkpointing the whole decoder layer.

Everything else of the model (attention, norms, lm_head, FSDP wrapping, checkpoint keys) is untouched;
``install_lm_head_loss()`` separately moves the lm_head cross-entropy onto this package's kernels,
``install_rl_lm_head()`` the RL trainer's lm_head log-probabilities and GRPO loss, and
``install_qk_norm_rope(model)`` the q/k norm and rotary embedding in front of the attention, and
``install_moe_aux_loss()`` the statistics behind the MoE balancing and z losses; parameters keep their
names, so state dicts and DCP checkpoints stay compatible.  ``restore_model`` undoes the conversion.
"""
from __future__ import annotations

import functools
import importlib
import types

import torch
from torch import nn

from . import fused as _fused
from . import ops
from .dispatcher import FusedDispatcher
from .router import GreedyRouter, NoAuxRouter

_SAVED = "_xtuner_b200_saved"
_ABSENT = object()  # saved for a name the owner did not carry itself (a class attribute showed through)


def _rebind(owner, **replacements) -> bool:
    """Sets each name on ``owner`` (a class, a module or an object) and keeps what the owner itself held under it in
    ``vars(owner)[_SAVED]``, for :func:`_restore`: a class's raw entry (descriptors such as ``staticmethod`` survive,
    subclasses keep inheriting), an ``nn.Module``'s registered submodule, or :data:`_ABSENT`.  An owner that already
    carries a rebind is left as it is and False returned: installing twice changes nothing."""
    if _SAVED in vars(owner):
        return False
    subs = owner._modules if isinstance(owner, nn.Module) else {}
    saved = {name: subs[name] if name in subs else vars(owner).get(name, _ABSENT) for name in replacements}
    setattr(owner, _SAVED, saved)
    for name, value in replacements.items():
        setattr(owner, name, value)
    return True


def _restore(owner) -> None:
    """Puts back what :func:`_rebind` saved on ``owner``: ``setattr`` (so a submodule is registered again), or deletes
    the name the owner did not carry before.  Nothing to do when the owner carries no rebind."""
    saved = vars(owner).get(_SAVED)
    if saved is None:
        return
    for name, original in saved.items():
        if original is _ABSENT:
            delattr(owner, name)
        else:
            setattr(owner, name, original)
    delattr(owner, _SAVED)


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


def _fused_layer_forward(self, hidden_states, seq_ctx, position_embeddings, *, recompute=None):
    """Replacement for ``MoEDecoderLayer._forward`` (``moe_decoder_layer.py:392-488``): the attention half is the
    reference's own modules (``_pre_moe_forward`` lines 634-666), the MoE half one fused autograd node.  ``recompute`` is
    bound by :func:`convert_model`."""
    residual = hidden_states
    hidden_states = self.input_layernorm(hidden_states)
    attn_outputs = self.self_attn(hidden_states=hidden_states, position_embeddings=position_embeddings, seq_ctx=seq_ctx)
    hidden_states = residual + attn_outputs["projected_output"]
    router = self.gate.router
    # RL routing replay: this layer's slice of the [S, L, K] ids, moved to the device if offloaded, exactly as the
    # reference does (moe_decoder_layer.py:669-677)
    opts = {}  # keywords only when set: the call keeps fused_moe_block's own defaults
    ids = getattr(seq_ctx, "rollout_routed_experts", None)
    if ids is not None and self.layer_idx < ids.shape[1]:
        ids = ids[:, self.layer_idx, :]
        if seq_ctx.offload_rollout_routed_experts and ids.device != hidden_states.device:
            ids = ids.contiguous().to(hidden_states.device)
        opts["rollout_routed_experts"] = ids
    if recompute is not None:
        opts["recompute"] = recompute
    out, rr = _fused.fused_moe_block(
        hidden_states, _local(self.post_attention_layernorm.weight), self.post_attention_layernorm.variance_epsilon,
        _local(self.gate.weight), _local(self.experts.fused_w1w3.weight), _local(self.experts.fused_w2.weight),
        top_k=router.top_k, norm_topk_prob=router.norm_topk_prob, router_scaling_factor=router.router_scaling_factor,
        hidden_factor=self.hidden_factor, scoring_func=router.scoring_func, **opts,
    )
    return out, rr["logits"], rr["router_weights"], rr["topk_ids"]


def _is_moe_layer(layer: nn.Module) -> bool:
    # the layer itself, not a wrapper that forwards attribute reads to it (torch's CheckpointWrapper under the
    # reference's fully_shard does): `dispatcher` is a plain attribute, `gate` / `experts` are sub-modules
    return "dispatcher" in vars(layer) and "gate" in layer._modules and "experts" in layer._modules


def convert_model(model: nn.Module, *, swiglu: bool = True, fused: bool = False, ep: "bool | str" = False,
                  recompute: "str | None" = None) -> int:
    """Returns the number of MoE decoder layers converted.  ``ep`` also converts ``TorchAll2AllDispatcher`` layers (expert
    parallel): ``True`` / ``"nccl"`` -> :class:`All2AllDispatcher` (the reference's six phases, NCCL all-to-all, our
    permute/unpermute kernels); ``"peer"`` -> :class:`PeerAll2AllDispatcher` (device-side split sizes, peer-memory pull
    kernels, no host read; needs symmetric memory over the EP group).  Both are covered by ``tests/test_gpu_comm.py`` with
    ``XTB_TEST_EP=1`` on >= 2 GPUs.  ``recompute`` (``"act"`` or ``"experts"``, needs ``fused=True``): what the fused nodes
    rebuild in the backward, as in :func:`xtuner_b200.fused.fused_moe_block`."""
    if ep not in (False, True, "nccl", "peer"):
        raise ValueError(f"convert_model: ep must be False, True, 'nccl' or 'peer' (got {ep!r})")
    _fused._check_recompute("convert_model", recompute)
    if recompute is not None and not fused:
        raise ValueError(f"convert_model: recompute={recompute!r} applies to the fused nodes: it needs fused=True")
    n = 0
    for layer in model.modules():
        if not _is_moe_layer(layer):
            continue
        disp = layer.dispatcher
        kind = type(disp).__name__
        if not _router_convertible(layer.gate.router):
            continue  # grouped routers etc.: the layer is left entirely on the reference path (nothing is half-converted)
        if kind == "TorchAll2AllDispatcher" and ep and getattr(disp, "_expert_tp", None) is None:
            # ep > 1 (reference key dispatcher="all2all", module/dispatcher/__init__.py:30-96): same six phases on our ops
            from .ep_dispatcher import All2AllDispatcher, PeerAll2AllDispatcher

            dispatcher_cls = PeerAll2AllDispatcher if ep == "peer" else All2AllDispatcher
        elif kind == "NaiveDispatcher":
            dispatcher_cls = FusedDispatcher
        else:
            continue  # DeepEP / AGRS / ExpertTP dispatchers are left alone
        # every replacement is built before the first is set: a router that fails to convert leaves the layer whole
        layer_names = {"dispatcher": dispatcher_cls(
            n_routed_experts=disp._n_routed_experts, process_group=disp._process_group,
            training_dtype=disp._training_dtype, generate_dtype=disp._generate_dtype,
        )}
        router = _convert_router(layer.gate.router)
        if fused and kind == "NaiveDispatcher" and _fused_eligible(layer):  # an instance attribute shadows the class method
            layer_names["_forward"] = types.MethodType(functools.partial(_fused_layer_forward, recompute=recompute), layer)
        _rebind(layer, **layer_names)
        _rebind(layer.gate, router=router)
        if swiglu and getattr(layer.experts, "moe_act", None) is not None and getattr(layer.experts.moe_act, "__name__", "") == "native_swiglu":
            _rebind(layer.experts, moe_act=ops.swiglu)
        n += 1
    if n:
        mgl = importlib.import_module("xtuner.v1.module.grouped_linear.moe_group_linear")
        _rebind(mgl, group_gemm=_group_gemm_dispatch(mgl.group_gemm))
    return n


def restore_model(model: nn.Module) -> None:
    for layer in model.modules():
        if _is_moe_layer(layer):
            for owner in (layer, layer.gate, layer.experts):
                _restore(owner)
    try:
        _restore(importlib.import_module("xtuner.v1.module.grouped_linear.moe_group_linear"))
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

    _rebind(importlib.import_module("xtuner.v1.module.attention.mha"), ulysses_all_to_all=ulysses_all_to_all)


def uninstall_ulysses() -> None:
    _restore(importlib.import_module("xtuner.v1.module.attention.mha"))


# ======================================================================================================
# lm_head + cross-entropy (f4)
# ======================================================================================================


def _lm_head_eligible(ctx, cls, hidden_states, head_weight, head_bias) -> bool:
    """what the lm_head kernels (``ops.lm_head_cross_entropy``, ``ops.lm_head_logprobs``) compute: the plain context
    (subclasses such as ``MTPLossContext`` bring their own ``loss_fn``), no bias, bf16 CUDA hidden states and weight
    (``fp32_lm_head`` gives fp32), widths multiples of 128"""
    return (type(ctx) is cls and head_bias is None
            and all(type(t) in (torch.Tensor, nn.Parameter) and _on_device(t) and t.dtype == torch.bfloat16
                    for t in (hidden_states, head_weight))
            and head_weight.dim() == 2 and head_weight.shape[0] % 128 == 0 and head_weight.shape[1] % 128 == 0)


def _ce_eligible(ctx, cls, hidden_states, head_weight, head_bias) -> bool:
    """:func:`_lm_head_eligible` for the cross-entropy, which also needs the loss weight ``build_batches`` sets"""
    kw = ctx.loss_kwargs
    return (kw is not None and kw.loss_weight is not None
            and _lm_head_eligible(ctx, cls, hidden_states, head_weight, head_bias))


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
    cls = importlib.import_module("xtuner.v1.loss.ce_loss").LMHeadLossContext
    orig_eager, orig_chunk = vars(cls)["eager_mode"], vars(cls)["chunk_mode"]

    def eager_mode(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if self.loss_cfg.mode == "eager" and _ce_eligible(self, cls, hidden_states, head_weight, head_bias):
            return _lm_head_loss(self, hidden_states, head_weight, loss_kwargs, None)
        return orig_eager(self, hidden_states, head_weight, head_bias, loss_kwargs)

    def chunk_mode(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if (self.loss_cfg.mode == "chunk" and self.loss_cfg.chunk_size is not None
                and (hidden_states.dim() == 2 or hidden_states.shape[0] == 1)
                and _ce_eligible(self, cls, hidden_states, head_weight, head_bias)):
            return _lm_head_loss(self, hidden_states, head_weight, loss_kwargs, self.loss_cfg.chunk_size)
        return orig_chunk(self, hidden_states, head_weight, head_bias, loss_kwargs)

    eager_mode.__wrapped__, chunk_mode.__wrapped__ = orig_eager, orig_chunk
    _rebind(cls, eager_mode=eager_mode, chunk_mode=chunk_mode)


def uninstall_lm_head_loss() -> None:
    _restore(importlib.import_module("xtuner.v1.loss.ce_loss").LMHeadLossContext)


# ======================================================================================================
# lm_head label log-probabilities (f5): LogProbContext and GRPOLossContext
# ======================================================================================================


def _policy_extra_info(logprobs, old_logprobs, valid, cliprange_low, cliprange_high) -> dict:
    """The statistics ``GRPOLossContext.loss_fn`` returns beside its loss, from detached log-probabilities.  With
    d = logp - old and r = exp(clamp(d, -20, 20)), over the valid positions: the largest and smallest r, the sums of
    |r - 1|, of k1 = -d and of k3 = r - 1 - clamp(d, -20, 20), their number, and, when both clip bounds are set, how many
    r lie below 1 - low and above 1 + high.  Invalid positions enter the sums as exact zeros, so each sum runs over the
    same tensor shape as the reference's and keeps its bits."""
    d = logprobs.detach() - old_logprobs.detach()
    d_clamped = d.clamp(-20.0, 20.0)
    r = d_clamped.exp()
    on = valid.float()
    r_max = torch.where(valid, r, 0.0).max()
    info = {
        "max_ratio": r_max,
        "reduced_train_policy_ratio_abs_dev_sum": ((r - 1.0).abs() * on).sum(),
        "reduced_train_policy_kl1_sum": (d.neg() * on).sum(),
        "reduced_train_policy_kl3_sum": ((r - 1.0 - d_clamped) * on).sum(),
        "reduced_train_policy_valid_count": on.sum(),
        "reduced_train_policy_ratio_max": r_max,
        "reduced_train_policy_ratio_min": torch.where(valid, r, float("inf")).min(),
    }
    if cliprange_low is not None and cliprange_high is not None:
        info["reduced_train_policy_clip_low_count"] = (valid & (r < 1 - cliprange_low)).float().sum()
        info["reduced_train_policy_clip_high_count"] = (valid & (r > 1 + cliprange_high)).float().sum()
    return info


def install_rl_lm_head() -> None:
    """Moves the lm_head of the RL trainer's three calls per micro-batch onto :func:`ops.lm_head_logprobs`:

    * ``LogProbContext.loss_fn`` and ``.chunk_mode`` (``xtuner/v1/loss/rl_loss.py``; the actor's and the reference
      model's log-probabilities) return ``(ops.lm_head_logprobs(...), (None, {}))``;
    * ``GRPOLossContext.loss_fn`` (``xtuner/v1/rl/loss/grpo_loss.py``) takes the log-probabilities from the op and runs
      the context's own ``policy_loss_fn`` and, with ``use_kl_loss``, ``kl_penalty`` on them in torch, so every registered
      loss type and KL type is served; it returns ``(loss, (None, extra_info))`` with the reference's statistics.  Modes
      "eager" and "chunk" both reach it (chunk mode through ``ChunkLoss``).

    Calls it does not cover go to the original methods: subclasses with their own ``loss_fn`` (``OrealLossContext``),
    mode ``"liger"``, a head bias, fp32 or non-CUDA tensors, a weight that is not a plain tensor, ``V`` or ``H`` not a
    multiple of 128.  Opt-in because the served calls return no logits.  Composes with :func:`install_lm_head_loss` in
    either order.  The RL modules (which import ``ray``) are loaded here only."""
    lp_cls = importlib.import_module("xtuner.v1.loss.rl_loss").LogProbContext
    grpo_mod = importlib.import_module("xtuner.v1.rl.loss.grpo_loss")
    grpo_cls = grpo_mod.GRPOLossContext
    lp_loss_fn, lp_chunk_mode = vars(lp_cls)["loss_fn"], vars(lp_cls)["chunk_mode"]
    grpo_loss_fn = vars(grpo_cls)["loss_fn"]

    def logprob_loss_fn(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if _lm_head_eligible(self, lp_cls, hidden_states, head_weight, head_bias):
            return ops.lm_head_logprobs(hidden_states, head_weight, loss_kwargs.shifted_labels), (None, {})
        return lp_loss_fn(self, hidden_states, head_weight, head_bias, loss_kwargs)

    def logprob_chunk_mode(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if (self.loss_cfg.chunk_size is not None
                and _lm_head_eligible(self, lp_cls, hidden_states, head_weight, head_bias)):
            logprobs = ops.lm_head_logprobs(hidden_states, head_weight, loss_kwargs.shifted_labels,
                                            self.loss_cfg.chunk_size)
            return logprobs, (None, {})
        return lp_chunk_mode(self, hidden_states, head_weight, head_bias, loss_kwargs)

    def grpo_loss(self, hidden_states, head_weight, head_bias, loss_kwargs):
        if not (self.loss_cfg.mode in ("eager", "chunk")
                and _lm_head_eligible(self, grpo_cls, hidden_states, head_weight, head_bias)):
            return grpo_loss_fn(self, hidden_states, head_weight, head_bias, loss_kwargs)
        cfg = self.loss_cfg
        labels = loss_kwargs.shifted_labels
        logprobs = ops.lm_head_logprobs(hidden_states, head_weight, labels)
        loss = self.policy_loss_fn(logprobs, loss_kwargs.old_logprobs, loss_kwargs.advantages,
                                   loss_kwargs.policy_loss_weight, cfg.policy_loss_cfg)
        extra_info = _policy_extra_info(logprobs, loss_kwargs.old_logprobs, labels != cfg.ignore_idx,
                                        cfg.policy_loss_cfg.get("cliprange_low"), cfg.policy_loss_cfg.get("cliprange_high"))
        if cfg.use_kl_loss:
            loss = loss + grpo_mod.kl_penalty(logprobs, loss_kwargs.ref_logprobs, loss_kwargs.kl_loss_weight,
                                              cfg.kl_loss_type)
        return loss, (None, extra_info)

    logprob_loss_fn.__wrapped__, logprob_chunk_mode.__wrapped__, grpo_loss.__wrapped__ = (lp_loss_fn, lp_chunk_mode,
                                                                                          grpo_loss_fn)
    if _SAVED not in vars(grpo_cls) and _rebind(lp_cls, loss_fn=logprob_loss_fn, chunk_mode=logprob_chunk_mode):
        _rebind(grpo_cls, loss_fn=grpo_loss)  # both classes or neither


def uninstall_rl_lm_head() -> None:
    _restore(importlib.import_module("xtuner.v1.loss.rl_loss").LogProbContext)
    _restore(importlib.import_module("xtuner.v1.rl.loss.grpo_loss").GRPOLossContext)


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

    _rebind(fu, cast_to_per_block_fp8_with_scales=cast_to_per_block_fp8_with_scales,
            tensor_to_per_block_fp8_scales=tensor_to_per_block_fp8_scales)


def uninstall_fp8_cast() -> None:
    _restore(importlib.import_module("xtuner.v1.float8.fsdp_utils"))


# ======================================================================================================
# q/k RMSNorm + rotary embedding in front of the attention (SURVEY.md §8f-3)
# ======================================================================================================


def _qk_layer_eligible(attn: nn.Module, apply_rotary_pos_emb_cuda) -> bool:
    """what ``ops.qk_norm_rope`` computes: the full-width rotary embedding (not partial rotary or FoPE sep-head), the
    "default" RMSNorm (or none), one eps for both norms, head dim 64, 128 or 256"""
    if vars(attn).get("apply_rotary_emb") is not apply_rotary_pos_emb_cuda or attn.head_dim not in (64, 128, 256):
        return False
    if not attn.qk_norm:
        return True
    qn, kn = attn.q_norm, attn.k_norm
    return (getattr(qn, "_type", None) == "default" and getattr(kn, "_type", None) == "default"
            and qn.variance_epsilon == kn.variance_epsilon and "forward" not in vars(qn) and "forward" not in vars(kn))


def _qk_call_eligible(q, k, cos, sin, position_ids, unsqueeze_dim) -> bool:
    """[1, H, S, D] bf16 CUDA q / k with the D axis contiguous, [1, S, D] cos / sin"""
    return (unsqueeze_dim == 1 and position_ids is None
            and all(type(t) in (torch.Tensor, nn.Parameter) and _on_device(t) and t.dtype == torch.bfloat16
                    for t in (q, k, cos, sin))
            and q.dim() == 4 and k.dim() == 4 and q.shape[0] == 1 and k.shape[0] == 1 and q.stride(-1) == 1
            and k.stride(-1) == 1 and cos.dim() == 3 and cos.shape[0] == 1 and sin.shape == cos.shape
            and cos.shape[1] == q.shape[2] and cos.shape[2] == q.shape[3])


def _qk_rope_closure(attn: nn.Module, orig_rope, norms):
    """the ``ApplyRotaryEmbProtocol`` callable set on ``attn``: with the norms made pass-throughs, it receives the raw
    projections and runs norm + rope as one op; calls it does not cover run the saved norm forwards and the original rope"""

    def apply_rotary_emb(q, k, cos, sin, position_ids=None, unsqueeze_dim=1):
        if not _qk_call_eligible(q, k, cos, sin, position_ids, unsqueeze_dim):
            if norms is not None:  # RMSNorm over the last dim: the same values on the transposed view
                q, k = norms[0](q), norms[1](k)
            return orig_rope(q, k, cos, sin, position_ids, unsqueeze_dim)
        w_q = w_k = None
        eps = 1e-6
        if norms is not None:
            w_q, w_k = _local(attn.q_norm.weight), _local(attn.k_norm.weight)
            eps = attn.q_norm.variance_epsilon
        S, D = q.shape[2], q.shape[3]
        out_q, out_k = ops.qk_norm_rope(q[0].transpose(0, 1), k[0].transpose(0, 1), cos[0], sin[0], w_q, w_k, eps)
        return out_q.view(1, S, -1, D).transpose(1, 2), out_k.view(1, S, -1, D).transpose(1, 2)

    apply_rotary_emb.__wrapped__ = orig_rope
    return apply_rotary_emb


def _identity(hidden_states):
    return hidden_states


def install_qk_norm_rope(model: nn.Module) -> int:
    """Runs q_norm / k_norm and the rotary embedding of every eligible ``MultiHeadAttention``
    (``xtuner/v1/module/attention/mha.py``) as one fused op (:func:`ops.qk_norm_rope`) in ``forward``, ``prefilling`` and
    ``decoding``.  The seam is the reference's own per-instance ``apply_rotary_emb`` (set at ``mha.py:202``); with
    ``qk_norm`` the two norms' ``forward`` become per-instance pass-throughs and the rope reads their weights at call time,
    so module objects, parameters and state-dict keys stay as they are.  Layers with partial rotary, FoPE sep-head or the
    zero-centred norm are left alone; calls outside [1, H, S, D] bf16 CUDA tensors run the original norms and rope.
    Opt-in and separate from :func:`convert_model`.  Returns the number of attention modules changed."""
    mha = importlib.import_module("xtuner.v1.module.attention.mha")
    rope = importlib.import_module("xtuner.v1.ops.rotary_emb").apply_rotary_pos_emb_cuda
    n = 0
    for attn in model.modules():
        if not isinstance(attn, mha.MultiHeadAttention) or _SAVED in vars(attn) or not _qk_layer_eligible(attn, rope):
            continue
        norms = (attn.q_norm.forward, attn.k_norm.forward) if attn.qk_norm else None
        _rebind(attn, apply_rotary_emb=_qk_rope_closure(attn, attn.apply_rotary_emb, norms))
        if attn.qk_norm:
            _rebind(attn.q_norm, forward=_identity)
            _rebind(attn.k_norm, forward=_identity)
        n += 1
    return n


def uninstall_qk_norm_rope(model: nn.Module) -> None:
    mha = importlib.import_module("xtuner.v1.module.attention.mha")
    for attn in model.modules():
        if isinstance(attn, mha.MultiHeadAttention):
            for owner in (attn, attn.q_norm, attn.k_norm) if attn.qk_norm else (attn,):
                _restore(owner)


# ======================================================================================================
# MoE auxiliary losses: the statistics AuxLossContext.accumulate takes from every MoE layer's router
# ======================================================================================================


def _aux_eligible(aux, classes, bal, zs, rw, logits, ids) -> bool:
    """what ``ops.moe_aux_stats`` computes: the reference's own context classes (a subclass may change what they do),
    fp32 ``[N, E]`` weights and logits and int64 ``[N, K]`` ids on the device, ``E`` within the kernel's range"""
    aux_cls, bal_cls, z_cls = classes
    E = aux.n_routed_experts
    return (type(aux) is aux_cls and all(type(c) is bal_cls for c in bal) and all(type(c) is z_cls for c in zs)
            and 1 <= E <= ops.MOE_AUX_MAX_EXPERTS
            and all(type(t) is torch.Tensor and _on_device(t) for t in (rw, logits, ids))
            and ids.dtype == torch.int64 and ids.dim() == 2 and ids.shape[1] >= 1
            and all(t.dtype == torch.float32 and tuple(t.shape) == (ids.shape[0], E) for t in (rw, logits)))


def install_moe_aux_loss() -> None:
    """Rebinds ``AuxLossContext.accumulate`` (``xtuner/v1/loss/aux_loss.py``) so that each MoE layer's expert counts, the
    balancing contexts' router-weight sums and the z-loss sum of squared logsumexps come from one
    :func:`ops.moe_aux_stats` call, forward and backward, instead of the reference's eager chain of ``histc``, ``sum``
    and ``logsumexp``.  Everything around them is the reference's: the counts go to ``_local_load_logits_list``, the sum
    to each balancing context's ``routing_weights_sum_list``, and each z context applies its own scaling (the alpha 0
    branch, ``/ denom_local``, the global-average factor with the device tensor ``num_tokens_global``, ``* alpha /
    batch_size``), updates its running log value and is attached to the hidden states through ``AuxLossScaler``.
    ``finalize`` is untouched.  Calls it does not cover run the original method: context subclasses, non-CUDA tensors,
    weights or logits that are not fp32 ``[N, E]``, ids that are not int64 ``[N, K]``, and ``E`` above
    :data:`ops.MOE_AUX_MAX_EXPERTS`.  Opt-in; installing twice is harmless, and it composes with :func:`convert_model`
    and the other installs."""
    aux_mod = importlib.import_module("xtuner.v1.loss.aux_loss")
    moe_loss = importlib.import_module("xtuner.v1.loss.moe_loss")
    cls = aux_mod.AuxLossContext
    orig = vars(cls)["accumulate"]
    classes = (cls, moe_loss.BalancingLossContext, moe_loss.ZLossContext)

    def accumulate(self, *, selected_router_weights, selected_router_logits, selected_experts, hidden_states,
                   balancing_ctx=None, z_ctx=None, num_tokens_local=0, num_tokens_global=None, world_size=1):
        bal, zs = aux_mod._as_list(balancing_ctx), aux_mod._as_list(z_ctx)
        if not _aux_eligible(self, classes, bal, zs, selected_router_weights, selected_router_logits, selected_experts):
            return orig(self, selected_router_weights=selected_router_weights,
                        selected_router_logits=selected_router_logits, selected_experts=selected_experts,
                        hidden_states=hidden_states, balancing_ctx=balancing_ctx, z_ctx=z_ctx,
                        num_tokens_local=num_tokens_local, num_tokens_global=num_tokens_global, world_size=world_size)
        tokens_per_expert, rw_sum, z_sum = ops.moe_aux_stats(
            selected_router_weights, selected_router_logits, selected_experts, self.n_routed_experts,
            need_rw_sum=bool(bal), need_z=any(ctx.loss_cfg.z_loss_alpha != 0 for ctx in zs))
        self._local_load_logits_list.append(tokens_per_expert)
        for ctx in bal:
            ctx.routing_weights_sum_list.append(rw_sum)
        for ctx in zs:
            if ctx.loss_cfg.z_loss_alpha == 0:
                loss = torch.tensor(0.0, device=selected_router_logits.device, dtype=torch.float32)
                ctx._update_running(loss)
            else:  # ZLossContext.accumulate's scaling lines, applied to the kernel's sum of lse^2
                loss = z_sum / max(num_tokens_local, 1)
                if ctx.loss_cfg.z_loss_global_average and num_tokens_global is not None:
                    denom_global = torch.clamp(num_tokens_global, min=1)
                    loss = loss * num_tokens_local * world_size / denom_global
                loss = loss * ctx.loss_cfg.z_loss_alpha / ctx._batch_size
                ctx._update_running(loss.detach())
            hidden_states = aux_mod.AuxLossScaler.apply(hidden_states, loss)
        return hidden_states

    accumulate.__wrapped__ = orig
    _rebind(cls, accumulate=accumulate)


def uninstall_moe_aux_loss() -> None:
    _restore(importlib.import_module("xtuner.v1.loss.aux_loss").AuxLossContext)
