"""ctypes binding of the C-ABI library declared in ``include/xtuner_b200.h``.

The library is the product: if it is missing or does not load, importing the compute ops raises —
there is no PyTorch/CPU fallback (the CPU oracle under ``oracle/`` is test infrastructure only).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_void_p

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libxtuner_b200.so")

_lib = None


class XtbError(RuntimeError):
    pass


# name -> (restype, argtypes); must list every symbol of include/xtuner_b200.h (tests check this)
SIGNATURES = {
    "xtb_version": (c_int, []),
    "xtb_last_error": (c_char_p, []),
    "xtb_init": (c_int, []),
    "xtb_launch_count": (c_int64, []),
    "xtb_reset_launch_count": (None, []),
    "xtb_gate_logits": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "xtb_gate_logits_bwd_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "xtb_gate_logits_bwd": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    ),
    "xtb_router_greedy": (
        c_int,
        [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_router_greedy_dispatch": (
        c_int,
        [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_gate_route_dispatch": (
        c_int,
        [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
         c_void_p, c_void_p, c_void_p],
    ),
    "xtb_router_greedy_replay": (
        c_int,
        [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
         c_void_p, c_void_p, c_void_p],
    ),
    "xtb_gate_route_replay_dispatch": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_router_noaux_replay": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
         c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_router_greedy_bwd": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p],
    ),
    "xtb_router_gate_bwd": (
        c_int,
        [c_void_p] * 10 + [c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p],
    ),
    "xtb_router_noaux": (
        c_int,
        [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_router_noaux_bwd": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p],
    ),
    "xtb_moe_permute_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "xtb_moe_permute": (
        c_int,
        [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_moe_permute_prepared": (
        c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "xtb_moe_unpermute": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "xtb_moe_combine": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_void_p, c_void_p],
    ),
    "xtb_moe_unpermute_bwd": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_group_gemm_nt": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "xtb_group_gemm_nt_swiglu": (
        c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "xtb_group_gemm_nn": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "xtb_group_gemm_tn": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "xtb_group_gemm_tn_pair": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                       c_void_p, c_int64, c_int, c_void_p]),
    "xtb_rmsnorm_gate": (
        c_int, [c_void_p, c_void_p, c_void_p, c_float, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes": (c_size_t, [c_int, c_int]),
    "xtb_moe_dispatch_bwd_rmsnorm": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
         c_void_p, c_void_p],
    ),
    "xtb_qk_norm_rope": (
        c_int,
        [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int,
         c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    ),
    "xtb_qk_norm_rope_bwd_workspace_bytes": (c_size_t, [c_int, c_int]),
    "xtb_qk_norm_rope_bwd": (
        c_int,
        [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64,
         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
         c_void_p, c_void_p],
    ),
    "xtb_moe_aux_stats_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "xtb_moe_aux_stats": (
        c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "xtb_moe_aux_stats_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "xtb_fp8_per_tile_quant":(c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p]),
    "xtb_fp8_block_scales": (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "xtb_fp8_block_cast": (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "xtb_peer_barrier": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p]),
    "xtb_a2a_pull": (
        c_int,
        [c_void_p, c_void_p, c_int, c_int, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64, c_int64,
         c_int64, c_int64, c_int64, c_void_p],
    ),
    "xtb_allgather_push": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_int, c_void_p]),
    "xtb_reduce_scatter_pull": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_float, c_int, c_void_p]),
    "xtb_allreduce_pull_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_float, c_void_p]),
    "xtb_peer_memcpy_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "xtb_ep_write_header": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "xtb_ep_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p]),
    "xtb_ep_pull_to_experts": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int64,
                                       c_int64, c_int64, c_void_p]),
    "xtb_ep_pull_to_sources": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64,
                                       c_void_p]),
    "xtb_lm_head_ce_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "xtb_lm_head_ce": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
         c_void_p, c_void_p, c_void_p],
    ),
    "xtb_lm_head_logprob_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "xtb_lm_head_logprob": (
        c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "xtb_lm_head_logprob_bwd": (
        c_int,
        [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
         c_void_p],
    ),
    "xtb_swiglu": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "xtb_swiglu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "xtb_swiglu_bwd_act": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
}


def load(path: str | None = None) -> ctypes.CDLL:
    """Load the shared library (once) and bind every declared symbol."""
    global _lib
    if _lib is not None:
        return _lib
    path = path or os.environ.get("XTUNER_B200_LIB", LIB_PATH)
    if not os.path.exists(path):
        raise XtbError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(xtuner_b200 has no CPU/PyTorch fallback)"
        )
    lib = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().xtb_last_error()
        raise XtbError(f"{what or 'xtuner_b200'} failed (status {rc}): {msg.decode() if msg else '?'}")


def ptr(t) -> int | None:
    """Raw device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def current_stream() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream


_initialised = False


def ensure_init() -> ctypes.CDLL:
    """Load + xtb_init() (checks for an sm_90 device).  Raises if there is no usable GPU."""
    global _initialised
    lib = load()
    if not _initialised:
        check(lib.xtb_init(), "xtb_init")
        _initialised = True
    return lib
