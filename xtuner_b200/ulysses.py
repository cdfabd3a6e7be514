"""Ulysses sequence-parallel attention (SURVEY.md §8a row a11): the SP block of
``MultiHeadAttention.forward`` (``xtuner/v1/module/attention/mha.py:365-390, 404-427``) with the three input
all-to-alls and the output all-to-all done by the peer-memory kernel of ``csrc/comm.cu`` and **pipelined against
the attention kernel by head group**:

    comm stream :  a2a(K) a2a(V) a2a(Q_0)  a2a(Q_1) ............ a2a(O_0)  a2a(O_1) ...
    main stream :                          attn(Q_0,K,V)  attn(Q_1,K,V) ...

Only K/V, the first Q group and the last O group are exposed; the rest of the 160 MiB per layer (config C4) moves
while the tensor cores work.  Autograd replays each op on the stream it ran on in forward, so the backward pass
overlaps the same way without extra code.

The attention kernel itself is the FlashAttention library in this image (``flash_attn`` 2.8, varlen causal GQA) —
the same call the reference makes (``ops/attn_imp.py:236-267``); an attention kernel of our own is not built yet
(DESIGN.md §8).  What is ours here: the exchange (one NVLink hop straight into the ``[S, heads, D]`` layout the
attention kernel wants — no contiguous/movedim/split/cat copies) and the overlap.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from . import _capi
from .comm import ulysses_all_to_all

_comm_streams: dict = {}


def _comm_stream(device) -> torch.cuda.Stream:
    s = _comm_streams.get(device)
    if s is None:
        # high priority: the small exchange kernels get the first SMs that free up while attention CTAs are running
        s = _comm_streams[device] = torch.cuda.Stream(device=device, priority=-1)
    return s


def repeat_kv(x: torch.Tensor, n_rep: int) -> torch.Tensor:
    """[1, Hkv, S, D] -> [1, Hkv*n_rep, S, D] (mha.py:368-371 / HF repeat_kv): each kv head n_rep times, adjacent."""
    if n_rep == 1:
        return x
    b, h, s, d = x.shape
    return x[:, :, None].expand(b, h, n_rep, s, d).reshape(b, h * n_rep, s, d)


def _flash(q, k, v, cu_q, cu_k, max_q, max_k, scale, causal):
    try:
        from flash_attn import flash_attn_varlen_func
    except Exception as e:  # pragma: no cover
        raise _capi.XtbError(f"flash_attn is required for ulysses_attention: {e}")
    return flash_attn_varlen_func(q, k, v, cu_q, cu_k, max_q, max_k, softmax_scale=scale, causal=causal)


def ulysses_attention(
    query_states: torch.Tensor,  # [1, Hq, S_loc, D]   (after RoPE, as at mha.py:363)
    key_states: torch.Tensor,  # [1, Hkv, S_loc, D]
    value_states: torch.Tensor,  # [1, Hkv, S_loc, D]
    cu_seqlens: torch.Tensor,  # int32, GLOBAL cumulative lengths (seq_ctx.cu_seq_lens_q)
    max_seqlen: int,
    group: dist.ProcessGroup,
    softmax_scale: Optional[float] = None,
    causal: bool = True,
    head_groups: Optional[int] = None,
    overlap: bool = True,
) -> torch.Tensor:
    """Returns ``raw_output`` [1, S_loc, Hq, D] — what ``mha.py:421-429`` has after the output all-to-all."""
    if not query_states.is_cuda:
        raise _capi.XtbError("ulysses_attention needs CUDA tensors (no CPU fallback)")
    sp = dist.get_world_size(group)
    _, Hq, S_loc, D = query_states.shape
    Hkv = key_states.shape[1]
    if sp > Hkv:  # mha.py:368-371
        assert sp % Hkv == 0
        key_states = repeat_kv(key_states, sp // Hkv)
        value_states = repeat_kv(value_states, sp // Hkv)
        Hkv = sp
    assert Hq % sp == 0 and Hkv % sp == 0
    hq_loc, hkv_loc = Hq // sp, Hkv // sp
    rep = hq_loc // hkv_loc  # q heads per kv head on this rank
    # head groups for pipelining: split along q heads that share a kv head (or along kv heads when there are several)
    if head_groups is None:
        head_groups = 2  # two groups already hide half of the Q/O traffic; more groups only add per-call overhead
    head_groups = max(1, min(head_groups, hq_loc if hkv_loc == 1 else hkv_loc))
    while hq_loc % head_groups or (hkv_loc > 1 and hkv_loc % head_groups):
        head_groups -= 1
    main = torch.cuda.current_stream()
    comm = _comm_stream(query_states.device) if (overlap and sp > 1) else main

    def on_comm(fn, *tensors):
        """run fn on the comm stream after everything already enqueued on main; returns (result, event)"""
        if comm is main:
            return fn(), None
        comm.wait_stream(main)
        with torch.cuda.stream(comm):
            out = fn()
            ev = torch.cuda.Event()
            ev.record(comm)
        for t in tensors:
            t.record_stream(comm)
        return out, ev

    # [1, H, S_loc, D] -> (a2a: scatter heads, gather sequence) -> [1, H/sp, S, D] -> [S, H/sp, D] view for FA
    k_full, ev_k = on_comm(lambda: ulysses_all_to_all(key_states, 1, 2, group), key_states)
    v_full, ev_v = on_comm(lambda: ulysses_all_to_all(value_states, 1, 2, group), value_states)
    q_heads_per_rank = hq_loc
    gq = hq_loc // head_groups  # q heads per group (per rank)
    # q viewed as [1, sp, hq_loc, S_loc, D]: group g takes heads [g*gq, (g+1)*gq) of every rank's slice
    q5 = query_states.view(1, sp, q_heads_per_rank, S_loc, D)
    outs = []
    q_parts = []
    for g in range(head_groups):
        # strided 5-D view [1, sp, gq, S_loc, D]: scatter the rank-slice dim, gather the sequence dim; the copy into
        # the symmetric staging buffer does the gather of the non-contiguous slice (no extra reshape copy)
        qg = q5[:, :, g * gq : (g + 1) * gq]
        q_parts.append(on_comm(lambda qg=qg: ulysses_all_to_all(qg, 1, 3, group).view(1, gq, S_loc * sp, D), query_states))
    pending_o = []
    for g in range(head_groups):
        q_full, ev_q = q_parts[g]
        for ev in (ev_k, ev_v, ev_q):
            if ev is not None:
                main.wait_event(ev)
        if comm is not main:
            for t in (k_full, v_full, q_full):
                t.record_stream(main)
        if hkv_loc == 1:
            kg, vg = k_full, v_full
        else:
            per = hkv_loc // head_groups
            kg, vg = k_full[:, g * per : (g + 1) * per], v_full[:, g * per : (g + 1) * per]
        o = _flash(
            q_full[0].transpose(0, 1), kg[0].transpose(0, 1), vg[0].transpose(0, 1), cu_seqlens, cu_seqlens, max_seqlen,
            max_seqlen, softmax_scale, causal,
        )  # [S, gq, D]
        # output a2a for this group: [1, S, gq, D] -> scatter S, gather heads -> [1, S_loc, sp*gq, D]
        o4 = o.unsqueeze(0)
        pending_o.append(on_comm(lambda o4=o4: ulysses_all_to_all(o4, 1, 2, group), o4))
    for o_loc, ev in pending_o:
        if ev is not None:
            main.wait_event(ev)
            o_loc.record_stream(main)
        outs.append(o_loc.view(1, S_loc, sp, gq, D))
    # reassemble heads in the reference order: head index = rank_slice * hq_loc + g * gq + j
    raw = torch.stack(outs, dim=3).reshape(1, S_loc, Hq, D) if head_groups > 1 else outs[0].reshape(1, S_loc, Hq, D)
    return raw
