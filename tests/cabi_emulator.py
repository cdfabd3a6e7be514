"""HOST-memory emulation of the C-ABI of include/xtuner_b200.h (test infrastructure only — nothing under xtuner_b200/
imports it).  Each method takes exactly the arguments of the header's declaration (raw addresses, sizes, a stream
handle that is ignored) and computes the documented result with plain torch-CPU / oracle arithmetic on the memory the
addresses point at.  It lets the CPU suite drive the shipped host orchestration above the boundary — the single-node
fused layer of ``xtuner_b200/fused.py``: buffer shapes, argument order, the backward chain — which otherwise only
runs on an H100.  It is NOT bit-compatible with the kernels in every rounding (tests use bf16-level tolerances) and
implements only the entry points that orchestration uses."""
from __future__ import annotations

import ctypes

import torch

from oracle import moe_oracle as O

_SIZES = {torch.bfloat16: 2, torch.float32: 4, torch.int32: 4, torch.int64: 8, torch.uint8: 1}


def _view(addr, dtype, *shape):
    """Tensor aliasing host memory at ``addr`` (None -> None)."""
    if addr is None:
        return None
    n = 1
    for s in shape:
        n *= int(s)
    if n == 0:
        return torch.empty(shape, dtype=dtype)
    buf = (ctypes.c_char * (n * _SIZES[dtype])).from_address(int(addr))
    return torch.frombuffer(buf, dtype=dtype).view(*shape)


class EmulatedLib:
    """Drop-in for the ctypes library object returned by ``_capi.ensure_init()``."""

    def __init__(self, real_lib):
        self._real = real_lib  # host-only helpers (workspace sizes) come from the real library
        self.calls: list[str] = []

    # ---- host-only entry points ---------------------------------------------------------------------------
    def xtb_moe_permute_workspace_bytes(self, T, K, E):
        return self._real.xtb_moe_permute_workspace_bytes(T, K, E)

    def xtb_gate_logits_bwd_workspace_bytes(self, T, H, E):
        return self._real.xtb_gate_logits_bwd_workspace_bytes(T, H, E)

    def xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(self, T, H):
        return self._real.xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(T, H)

    def xtb_last_error(self):
        return b"emulated"

    # ---- a1 --------------------------------------------------------------------------------------------------
    def xtb_gate_logits(self, x, w, bias, logits, T, H, E, stream):
        self.calls.append("xtb_gate_logits")
        out = O.gate_logits(_view(x, torch.bfloat16, T, H), _view(w, torch.float32, E, H))
        if bias is not None:
            out = out + _view(bias, torch.float32, E)
        _view(logits, torch.float32, T, E).copy_(out)
        return 0

    def xtb_gate_logits_bwd(self, gl, x, w, gw, gx, gbias, T, H, E, ws, stream):
        self.calls.append("xtb_gate_logits_bwd")
        assert ws is not None
        g = _view(gl, torch.float32, T, E)
        _view(gw, torch.float32, E, H).copy_(g.t() @ _view(x, torch.bfloat16, T, H).float())
        _view(gx, torch.bfloat16, T, H).copy_((g @ _view(w, torch.float32, E, H)).to(torch.bfloat16))
        if gbias is not None:
            _view(gbias, torch.float32, E).copy_(g.sum(0))
        return 0

    # ---- a2 (+ index half of a4) --------------------------------------------------------------------------
    def xtb_router_greedy_dispatch(self, logits, T, E, K, scoring, norm, scaling, rw, tw, ids, ids32, tpe, ws, stream):
        self.calls.append("xtb_router_greedy_dispatch")
        assert ws is not None and ids32 is not None
        r = O.greedy_router(_view(logits, torch.float32, T, E), K, bool(norm), scaling, "softmax" if scoring == 0 else "sigmoid")
        _view(rw, torch.float32, T, E).copy_(r["router_weights"])
        _view(tw, torch.float32, T, K).copy_(r["topk_weights"])
        _view(ids, torch.int64, T, K).copy_(r["topk_ids"])
        _view(ids32, torch.int32, T, K).copy_(r["topk_ids"].to(torch.int32))
        _view(tpe, torch.int64, E).copy_(r["topkens_per_expert"])
        return 0

    def xtb_router_greedy(self, logits, T, E, K, scoring, norm, scaling, rw, tw, ids, ids32, tpe, stream):
        self.calls.append("xtb_router_greedy")
        r = O.greedy_router(_view(logits, torch.float32, T, E), K, bool(norm), scaling, "softmax" if scoring == 0 else "sigmoid")
        _view(rw, torch.float32, T, E).copy_(r["router_weights"])
        _view(tw, torch.float32, T, K).copy_(r["topk_weights"])
        _view(ids, torch.int64, T, K).copy_(r["topk_ids"])
        if ids32 is not None:
            _view(ids32, torch.int32, T, K).copy_(r["topk_ids"].to(torch.int32))
        _view(tpe, torch.int64, E).copy_(r["topkens_per_expert"])
        return 0

    def xtb_router_noaux(self, logits, bias, T, E, K, n_group, topk_group, norm, scaling, rw, tw, ids, ids32, tpe, stream):
        self.calls.append("xtb_router_noaux")
        r = O.noaux_router(_view(logits, torch.float32, T, E), _view(bias, torch.float32, E), K, n_group, topk_group, scaling, bool(norm))
        _view(rw, torch.float32, T, E).copy_(r["router_weights"])
        _view(tw, torch.float32, T, K).copy_(r["topk_weights"])
        _view(ids, torch.int64, T, K).copy_(r["topk_ids"])
        if ids32 is not None:
            _view(ids32, torch.int32, T, K).copy_(r["topk_ids"].to(torch.int32))
        _view(tpe, torch.float32, E).copy_(r["topkens_per_expert"])
        return 0

    def xtb_router_noaux_bwd(self, logits, bias, rw, tw, ids, g_tw, g_rw, T, E, K, group_spec, norm, scaling, gl, stream):
        self.calls.append("xtb_router_noaux_bwd")
        out = O.noaux_router_bwd(
            _view(logits, torch.float32, T, E), _view(bias, torch.float32, E), _view(rw, torch.float32, T, E),
            _view(tw, torch.float32, T, K), _view(ids, torch.int64, T, K), _view(g_tw, torch.float32, T, K),
            _view(g_rw, torch.float32, T, E), group_spec != 0, scaling, bool(norm), n_group=group_spec & 0xFF,
            topk_group=group_spec >> 8)
        _view(gl, torch.float32, T, E).copy_(out)
        return 0

    def xtb_gate_route_dispatch(self, x, w, T, H, E, K, scoring, norm, scaling, logits, rw, tw, ids, ids32, tpe, ws, stream):
        self.calls.append("xtb_gate_route_dispatch")
        if E > 8 or K > 8 or H % 128 or H > 4096:
            return 1
        self.xtb_gate_logits(x, w, None, logits, T, H, E, stream)
        rc = self.xtb_router_greedy_dispatch(logits, T, E, K, scoring, norm, scaling, rw, tw, ids, ids32, tpe, ws, stream)
        self.calls = self.calls[:-2]
        return rc

    def xtb_router_gate_bwd(self, rw, tw, ids, g_tw, g_rw, g_direct, x, w, gw, gx, T, H, E, K, scoring, norm, scaling, ws, stream):
        self.calls.append("xtb_router_gate_bwd")
        if E > 8 or H % 8:
            return 1
        gl = torch.empty(T, E, dtype=torch.float32)
        self.xtb_router_greedy_bwd(rw, tw, ids, g_tw, g_rw, g_direct, T, E, K, scoring, norm, scaling, gl.data_ptr(), stream)
        rc = self.xtb_gate_logits_bwd(gl.data_ptr(), x, w, gw, gx, None, T, H, E, ws, stream)
        self.calls = self.calls[:-2]
        return rc

    def xtb_router_greedy_bwd(self, rw, tw, ids, g_tw, g_rw, g_direct, T, E, K, scoring, norm, scaling, gl, stream):
        self.calls.append("xtb_router_greedy_bwd")
        p = _view(rw, torch.float32, T, E)
        idx = _view(ids, torch.int64, T, K)
        gp = torch.zeros(T, E) if g_rw is None else _view(g_rw, torch.float32, T, E).clone()
        if g_tw is not None:
            g = _view(g_tw, torch.float32, T, K)
            v = p.gather(1, idx)
            if norm:
                s = v.sum(1, keepdim=True)
                dot = (g * v / s).sum(1, keepdim=True)
                gv = scaling * (g - dot) / s
            else:
                gv = scaling * g
            gp = gp.scatter_add(1, idx, gv)
        if scoring == 0:
            out = p * (gp - (gp * p).sum(1, keepdim=True))
        else:
            out = gp * p * (1 - p)
        if g_direct is not None:
            out = out + _view(g_direct, torch.float32, T, E)
        _view(gl, torch.float32, T, E).copy_(out)
        return 0

    # ---- a4 -------------------------------------------------------------------------------------------------
    def xtb_moe_permute_prepared(self, x, ids32, T, K, E, row_bytes, permuted, row_id_map, sorted_indices, ws, stream):
        self.calls.append("xtb_moe_permute_prepared")
        assert ws is not None and row_bytes % 16 == 0
        H = row_bytes // 2
        perm, sorted_idx = O.permute(_view(x, torch.bfloat16, T, H), _view(ids32, torch.int32, T, K))
        _view(permuted, torch.bfloat16, T * K, H).copy_(perm)
        rmap = torch.empty(T * K, dtype=torch.int64)
        rmap[sorted_idx] = torch.arange(T * K)
        _view(row_id_map, torch.int32, T * K).copy_(rmap.to(torch.int32))
        if sorted_indices is not None:
            _view(sorted_indices, torch.int64, T * K).copy_(sorted_idx)
        return 0

    def xtb_moe_permute(self, x, ids32, T, K, E, row_bytes, permuted, row_id_map, sorted_indices, tpe, ws, stream):
        self.calls.append("xtb_moe_permute")
        rc = self.xtb_moe_permute_prepared(x, ids32, T, K, E, row_bytes, permuted, row_id_map, sorted_indices, ws, stream)
        if tpe is not None:
            _view(tpe, torch.int64, E).copy_(O.tokens_per_expert_hist(_view(ids32, torch.int32, T, K), E))
        return rc

    # ---- a5 -------------------------------------------------------------------------------------------------
    def xtb_moe_unpermute(self, y, row_id_map, probs, T, K, H, out, stream):
        self.calls.append("xtb_moe_unpermute")
        return self.xtb_moe_combine(y, row_id_map, probs, None, 1.0, T, K, H, out, stream)

    def xtb_moe_combine(self, y, row_id_map, probs, residual, hidden_factor, T, K, H, out, stream):
        self.calls.append("xtb_moe_combine")
        rows = _view(row_id_map, torch.int32, T * K).long()
        g = _view(y, torch.bfloat16, T * K, H)[rows].view(T, K, H).float()
        if probs is not None:
            g = g * _view(probs, torch.float32, T, K).unsqueeze(-1)
        o = g.sum(1).to(torch.bfloat16)
        if hidden_factor != 1.0:
            o = (o.float() * hidden_factor).to(torch.bfloat16)
        if residual is not None:
            o = (o.float() + _view(residual, torch.bfloat16, T, H).float()).to(torch.bfloat16)
        _view(out, torch.bfloat16, T, H).copy_(o)
        return 0

    def xtb_moe_unpermute_bwd(self, g_out, y_fwd, row_id_map, probs, T, K, H, act_grad, prob_grad, stream):
        self.calls.append("xtb_moe_unpermute_bwd")
        rows = _view(row_id_map, torch.int32, T * K).long()
        g = _view(g_out, torch.bfloat16, T, H).float()
        p = torch.ones(T, K) if probs is None else _view(probs, torch.float32, T, K)
        ag = _view(act_grad, torch.bfloat16, T * K, H)
        ag[rows] = (g.unsqueeze(1) * p.unsqueeze(-1)).to(torch.bfloat16).view(T * K, H)
        if prob_grad is not None:
            yf = _view(y_fwd, torch.bfloat16, T * K, H)[rows].view(T, K, H).float()
            _view(prob_grad, torch.float32, T, K).copy_((g.unsqueeze(1) * yf).sum(-1))
        return 0

    # ---- a6/a7/a8 -------------------------------------------------------------------------------------------
    @staticmethod
    def _groups(tpe, E):
        return _view(tpe, torch.int64, E).tolist()

    def xtb_group_gemm_nt(self, x, w, tpe, M, N, Kd, E, out, stream):
        self.calls.append("xtb_group_gemm_nt")
        res = O.group_gemm(_view(x, torch.bfloat16, M, Kd), _view(w, torch.bfloat16, E, N, Kd), _view(tpe, torch.int64, E))
        _view(out, torch.bfloat16, M, N).copy_(res)
        return 0

    def xtb_group_gemm_nt_swiglu(self, x, w13, tpe, M, I, Kd, E, h_out, a_out, stream):
        self.calls.append("xtb_group_gemm_nt_swiglu")
        h = O.group_gemm(_view(x, torch.bfloat16, M, Kd), _view(w13, torch.bfloat16, E, 2 * I, Kd), _view(tpe, torch.int64, E))
        _view(h_out, torch.bfloat16, M, 2 * I).copy_(h)
        _view(a_out, torch.bfloat16, M, I).copy_(O.swiglu(h))
        return 0

    def xtb_group_gemm_nn(self, dy, w, tpe, M, N, Kd, E, out, stream):
        self.calls.append("xtb_group_gemm_nn")
        d, W, o = _view(dy, torch.bfloat16, M, N), _view(w, torch.bfloat16, E, N, Kd), _view(out, torch.bfloat16, M, Kd)
        s = 0
        for e, n in enumerate(self._groups(tpe, E)):
            o[s : s + n] = d[s : s + n] @ W[e]
            s += n
        return 0

    def xtb_group_gemm_tn(self, dy, x, tpe, M, N, Kd, E, dw, stream):
        self.calls.append("xtb_group_gemm_tn")
        d, X, o = _view(dy, torch.bfloat16, M, N), _view(x, torch.bfloat16, M, Kd), _view(dw, torch.bfloat16, E, N, Kd)
        s = 0
        for e, n in enumerate(self._groups(tpe, E)):
            o[e] = d[s : s + n].t() @ X[s : s + n]
            s += n
        return 0

    def xtb_group_gemm_tn_pair(self, dy_a, x_a, N_a, Kd_a, dw_a, dy_b, x_b, N_b, Kd_b, dw_b, tpe, M, E, stream):
        self.xtb_group_gemm_tn(dy_a, x_a, tpe, M, N_a, Kd_a, E, dw_a, stream)
        self.xtb_group_gemm_tn(dy_b, x_b, tpe, M, N_b, Kd_b, E, dw_b, stream)
        self.calls.append("xtb_group_gemm_tn_pair")
        return 0

    # ---- a15: fp8 block scales / cast of a weight (the oracle restates float8/fsdp_utils.py:75-116,196-223) -----------
    def xtb_fp8_block_scales(self, w, w_is_f32, nw, dout, din, scales, stream):
        self.calls.append("xtb_fp8_block_scales")
        W = _view(w, torch.float32 if w_is_f32 else torch.bfloat16, nw, dout, din)
        _view(scales, torch.float32, nw, dout // 128, din // 128).copy_(O.per_block_fp8_scales(W).view(nw, dout // 128, din // 128))
        return 0

    def xtb_fp8_block_cast(self, w, w_is_f32, nw, dout, din, scales, q, stream):
        self.calls.append("xtb_fp8_block_cast")
        W = _view(w, torch.float32 if w_is_f32 else torch.bfloat16, nw, dout, din)
        S = _view(scales, torch.float32, nw, dout // 128, din // 128)
        out = _view(q, torch.uint8, nw, dout, din)
        for i in range(nw):
            out[i].copy_(O.cast_to_per_block_fp8(W[i], S[i]).view(torch.uint8))
        return 0

    @staticmethod
    def _swiglu_bwd(g, h):
        """autograd of ``silu(x1) * x2`` on bf16 tensors spelled with the aten kernels autograd itself dispatches to
        (usable where autograd recording is off, e.g. inside a custom-op body)."""
        I = h.shape[1] // 2
        x1, x2 = h[:, :I], h[:, I:]
        s = torch.nn.functional.silu(x1)
        return torch.cat([torch.ops.aten.silu_backward(g * x2, x1), g * s], dim=1)

    def xtb_swiglu(self, h, out, M, I, stream):
        self.calls.append("xtb_swiglu")
        _view(out, torch.bfloat16, M, I).copy_(O.swiglu(_view(h, torch.bfloat16, M, 2 * I)))
        return 0

    def xtb_swiglu_bwd(self, grad_out, h, grad_h, M, I, stream):
        self.calls.append("xtb_swiglu_bwd")
        _view(grad_h, torch.bfloat16, M, 2 * I).copy_(self._swiglu_bwd(_view(grad_out, torch.bfloat16, M, I), _view(h, torch.bfloat16, M, 2 * I)))
        return 0

    def xtb_rmsnorm_gate(self, h, norm_w, gate_w, eps, T, H, E, x_out, rstd_out, logits, stream):
        self.calls.append("xtb_rmsnorm_gate")
        hf = _view(h, torch.bfloat16, T, H).float()
        rstd = torch.rsqrt(hf.pow(2).mean(-1) + eps)
        x = (hf * rstd.unsqueeze(-1) * _view(norm_w, torch.float32, H)).to(torch.bfloat16)
        _view(x_out, torch.bfloat16, T, H).copy_(x)
        _view(rstd_out, torch.float32, T).copy_(rstd)
        if gate_w is not None:
            _view(logits, torch.float32, T, E).copy_(x.float() @ _view(gate_w, torch.float32, E, H).t())
        return 0

    def xtb_moe_dispatch_bwd_rmsnorm(self, g_xperm, row_id_map, g_x_gate, h, rstd, norm_w, g_res, T, K, H, g_h, g_norm_w, ws, stream):
        self.calls.append("xtb_moe_dispatch_bwd_rmsnorm")
        rows = _view(row_id_map, torch.int32, T * K).long()
        gx = _view(g_xperm, torch.bfloat16, T * K, H)[rows].view(T, K, H).float().sum(1).to(torch.bfloat16)
        if g_x_gate is not None:
            gx = (gx.float() + _view(g_x_gate, torch.bfloat16, T, H).float()).to(torch.bfloat16)
        g = gx.float()
        hf = _view(h, torch.bfloat16, T, H).float()
        r = _view(rstd, torch.float32, T).unsqueeze(-1)
        w = _view(norm_w, torch.float32, H)
        gw = g * w
        gh = r * gw - hf * r.pow(3) * (gw * hf).mean(-1, keepdim=True)
        if g_res is not None:
            gh = gh.to(torch.bfloat16).float() + _view(g_res, torch.bfloat16, T, H).float()
        _view(g_h, torch.bfloat16, T, H).copy_(gh.to(torch.bfloat16))
        if g_norm_w is not None:
            assert ws is not None
            _view(g_norm_w, torch.float32, H).copy_((g * hf * r).sum(0))
        return 0
