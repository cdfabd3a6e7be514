"""The float64 restatement of the fused MoE nodes (tests/fused_node_reference.py) on CPU, no GPU needed.

* The unrounded chain (``forward64`` and ``backward_reference(fw=...)``) equals float64 autograd through the oracle's
  permute, grouped GEMMs, SwiGLU and unpermute: the output and every gradient, through out, logits and router_weights.
* An fp32 / bf16 emulation of either node, rounding where the kernels round, passes every forward and backward check,
  with the worst ratio far below 1.
* The same emulation with one wiring mistake planted is rejected (among them the residual gradient taken from
  g_out * hidden_factor instead of g_out), with a message naming the quantity; a one-ulp systematic shift of g_a is
  rejected too, so the bounds are not vacuous."""
import pytest
import torch
import torch.nn.functional as F

from oracle import moe_oracle as O
from tests import fused_node_reference as FN
from tests import gemm_reference as G
from tests import norm_combine_reference as NC
from tests import router_reference as R

CONFIGS = {
    "softmax": dict(norm=True, scaling=1.0, hf=1.0, scoring="softmax", res=True),
    "sigmoid": dict(norm=False, scaling=2.5, hf=0.5, scoring="sigmoid", res=False),
}
T, H, I, E, K = 48, 64, 32, 8, 2


def inputs(kind, cfg, seed=0):
    g = torch.Generator().manual_seed(seed)
    bf = torch.bfloat16
    inp = {
        "gate_w": torch.randn(E, H, generator=g) * 0.3,
        "w13": (torch.randn(E, 2 * I, H, generator=g) * H ** -0.5).to(bf),
        "w2": (torch.randn(E, H, I, generator=g) * I ** -0.5).to(bf),
    }
    if kind == "block":
        inp["h_in"] = (torch.randn(T, H, generator=g) * 2).to(bf)
        inp["norm_w"] = NC.norm_weight(H, seed + 1)
    else:
        inp["x"] = torch.randn(T, H, generator=g).to(bf)
        inp["residual"] = torch.randn(T, H, generator=g).to(bf) if cfg["res"] else None
    grads = {
        "g_out": torch.randn(T, H, generator=g).to(bf),
        "g_logits": torch.randn(T, E, generator=g) * 1e-2,
        "g_rw": torch.randn(T, E, generator=g) * 1e-1,
    }
    return inp, grads


def _bf(t):
    return t.to(torch.bfloat16)


def _next_away(t):
    """Every bf16 element moved one step away from zero."""
    i = t.contiguous().view(torch.int16)
    return torch.where(i & 0x7FFF != 0, i + 1, i).view(torch.bfloat16)


def emulate(kind, inp, cfg, g_out, g_logits, g_rw, mutate=None, replay=None):
    """``(Node, grads)`` of an fp32 emulation of the node with the kernels' bf16 storage points; ``mutate`` plants one
    mistake."""
    Kk, hf, norm, scaling, scoring = K, cfg["hf"], cfg["norm"], cfg["scaling"], cfg["scoring"]
    eps = 1e-6
    t = {}
    if kind == "block":
        h_in, nw = inp["h_in"], inp["norm_w"]
        rstd = torch.rsqrt(h_in.float().square().mean(-1) + eps)
        x = NC.rmsnorm_x(h_in, rstd, nw)
        t.update(h_in=h_in, norm_w=nw, rstd=rstd)
        residual = h_in
    else:
        x, residual = inp["x"], inp["residual"]
    gw, w13, w2 = inp["gate_w"], inp["w13"], inp["w2"]
    logits = x.float() @ gw.T
    rw = torch.softmax(logits, -1) if scoring == "softmax" else torch.sigmoid(logits)
    ids = R.topk_rounds(rw, Kk) if replay is None else replay
    tw = R.topk_weights_restated(rw, ids, norm, scaling)
    tpe = torch.bincount(ids.reshape(-1), minlength=E)
    order, rmap = FN.permutation(ids)
    x_perm = x[order // Kk]
    c = [int(v) for v in tpe.tolist()]
    o = G.offsets(c)
    shifted = max(range(E), key=lambda e: c[e])
    h = torch.empty(T * Kk, 2 * I, dtype=torch.bfloat16)
    for e in range(E):
        rows = x_perm[o[e] : o[e + 1]]
        if mutate == "expert_shift" and e == shifted:
            rows = x_perm[o[e] + 1 : o[e + 1] + 1]
            rows = torch.cat([rows, x_perm[: o[e + 1] - o[e] - rows.shape[0]]])
        h[o[e] : o[e + 1]] = _bf(rows.float() @ w13[e].float().T)
    a = G.swiglu_act(h)
    y = torch.cat([_bf(a[o[e] : o[e + 1]].float() @ w2[e].float().T) for e in range(E)])
    tw_c = tw.clone()
    if mutate == "tw_swap":
        tw_c[3, 0], tw_c[3, 1] = tw[3, 1], tw[3, 0]
    out = NC.combine(y, rmap, tw_c, residual, hf * hf if mutate == "hf_twice" else hf, Kk)
    t.update(x=x, gate_w=gw, w13=w13, w2=w2, rw=rw, tw=tw, ids=ids, rmap=rmap, tpe=tpe, x_perm=x_perm, h=h, a=a, y=y,
             out=out, logits=logits, residual=None if kind == "block" else residual)
    node = FN.Node(kind, t, Kk, norm, scaling, hf, scoring, eps)

    # backward
    M = T * Kk
    g_comb = g_out if hf == 1.0 else _bf(g_out.float() * hf)
    g_y = NC.act_grad(g_comb, rmap, tw, Kk, M)[0]
    g_tw = (g_comb.float()[:, None, :] * y[rmap.long()].float().view(T, Kk, H)).sum(-1)
    g_a = torch.cat([_bf(g_y[o[e] : o[e + 1]].float() @ w2[e].float()) for e in range(E)])
    if mutate == "g_a_shift":
        g_a = _next_away(g_a)
    gf, uf = h[:, :I].float(), h[:, I:].float()
    sig = torch.sigmoid(gf)
    s = _bf(gf * sig)
    gu = _bf(g_a.float() * s.float())
    ds = _bf(g_a.float() * uf)
    gg = _bf(ds.float() * sig * (1 + gf * (1 - sig)))
    g_h = torch.cat([gg, gu], 1)
    g_xp = torch.cat([_bf(g_h[o[e] : o[e + 1]].float() @ w13[e].float()) for e in range(E)])
    g_w13 = torch.stack([_bf(g_h[o[e] : o[e + 1]].float().T @ x_perm[o[e] : o[e + 1]].float()) for e in range(E)])
    if mutate == "w13_halves":
        g_w13 = torch.cat([g_w13[:, I:], g_w13[:, :I]], 1)
    g_w2 = torch.stack([_bf(g_y[o[e] : o[e + 1]].float().T @ a[o[e] : o[e + 1]].float()) for e in range(E)])
    lg = logits.clone().requires_grad_(True)
    with torch.enable_grad():
        p = torch.softmax(lg, -1) if scoring == "softmax" else torch.sigmoid(lg)
        w = p.gather(1, ids)
        if norm:
            w = w / w.sum(-1, keepdim=True)
        loss = (w * scaling * g_tw).sum()
        if mutate != "g_rw_ignored":
            loss = loss + (p * g_rw).sum()
        (gl,) = torch.autograd.grad(loss, lg)
    gl = gl + g_logits
    g_gate_w = gl.T @ x.float()
    g_x_gate = _bf(gl @ gw)
    g_x = NC.dispatch_gx(g_xp, rmap, None if mutate == "g_x_gate_dropped" else g_x_gate, Kk)
    grads = {"g_w13": g_w13, "g_w2": g_w2, "g_gate_w": g_gate_w}
    if kind == "moe":
        grads["g_x"] = g_x
        if residual is not None:
            wrong = {"residual_missing": torch.zeros_like(g_out), "residual_gets_g_comb": g_comb}
            grads["g_res"] = wrong.get(mutate, g_out)
    else:
        wg = g_x.float() * t["norm_w"]
        hf32 = t["h_in"].float()
        r = t["rstd"][:, None]
        cc = (wg * hf32).sum(-1, keepdim=True) * r * r / H
        gh = _bf((wg - hf32 * cc) * r)
        g_res = g_comb if mutate == "residual_gets_g_comb" else g_out
        grads["g_h"] = gh if mutate == "residual_missing" else _bf(gh.float() + g_res.float())
        grads["g_norm_w"] = (g_x.float() * hf32 * r).sum(0)
    return node, grads


def oracle_fp64(kind, inp, cfg, g_out, g_logits, g_rw):
    """float64 autograd through the oracle's permute / experts / unpermute; the router restated in float64 as
    greedy.py computes it (the oracle's softmax promotes to fp32)."""
    d = {k: (v.double().clone().requires_grad_(True) if v is not None else None) for k, v in inp.items()}
    if kind == "block":
        hh = d["h_in"]
        x = hh * torch.rsqrt(hh.square().mean(-1, keepdim=True) + 1e-6) * d["norm_w"]
        residual = hh
    else:
        x, residual = d["x"], d["residual"]
    logits = F.linear(x, d["gate_w"])
    p = torch.softmax(logits, -1) if cfg["scoring"] == "softmax" else torch.sigmoid(logits)
    tw, ids = torch.topk(p, K, dim=-1)
    if cfg["norm"]:
        tw = tw / tw.sum(-1, keepdim=True)
    tw = tw * cfg["scaling"]
    x_perm, row_id_map = O.permute(x, ids.to(torch.int32))
    tpe = O.tokens_per_expert_hist(ids, E)
    y = O.experts_forward(x_perm, d["w13"].view(E * 2 * I, H), d["w2"].view(E * H, I), tpe, E)
    out = O.unpermute(y, row_id_map, probs=tw) * cfg["hf"]
    if residual is not None:
        out = out + residual
    loss = (out * g_out.double()).sum() + (logits * g_logits.double()).sum() + (p * g_rw.double()).sum()
    wrt = {k: v for k, v in d.items() if v is not None}
    gr = torch.autograd.grad(loss, list(wrt.values()))
    return out.detach(), ids, dict(zip(wrt.keys(), gr))


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("kind", ["moe", "block"])
def test_unrounded_chain_is_float64_autograd_through_the_oracle(kind, cfg):
    c = CONFIGS[cfg]
    inp, gr = inputs(kind, c)
    node, _ = emulate(kind, inp, c, **gr)
    out64, ids64, want = oracle_fp64(kind, inp, c, **gr)
    assert torch.equal(node.t["ids"], ids64)
    fw = FN.forward64(inp, node.t["ids"], K, c["norm"], c["scaling"], c["hf"], c["scoring"])
    torch.testing.assert_close(fw["out"], out64, rtol=1e-12, atol=1e-12)
    got = FN.backward_reference(node, gr["g_out"], gr["g_logits"], gr["g_rw"], fw=fw)
    pairs = [("g_gate_w", "gate_w"), ("g_w13", "w13"), ("g_w2", "w2")]
    pairs += [("g_h", "h_in"), ("g_norm_w", "norm_w")] if kind == "block" else [("g_x", "x")]
    if kind == "moe" and c["res"]:
        pairs.append(("g_res", "residual"))
    for mine, theirs in pairs:
        torch.testing.assert_close(got[mine][0], want[theirs], rtol=1e-10, atol=1e-12, msg=lambda m: f"{mine}: {m}")


def _check(node, grads, gr, replay=None):
    r = FN.check_forward(node, replay)
    r.update(FN.check_backward(node, grads, gr["g_out"], gr["g_logits"], gr["g_rw"]))
    fw = FN.forward64({k: node.t[k] for k in ("gate_w", "w13", "w2")} | (
        {"h_in": node.t["h_in"], "norm_w": node.t["norm_w"]} if node.kind == "block" else
        {"x": node.t["x"], "residual": node.t["residual"]}), node.t["ids"], K, node.norm, node.scaling, node.hf,
        node.scoring, rounded=True)
    FN.check_loss(node.t["out"], fw["out"])
    return r


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("kind", ["moe", "block"])
def test_emulated_node_passes_far_inside_the_bounds(kind, cfg):
    c = CONFIGS[cfg]
    inp, gr = inputs(kind, c, seed=1)
    node, grads = emulate(kind, inp, c, **gr)
    r = _check(node, grads, gr)
    for q in ("g_w13", "g_w2", "g_gate_w", "g_h" if kind == "block" else "g_x"):
        assert r[q] < 0.5, (q, r[q])
    # replayed ids with a duplicate in a row and an empty expert
    rp = node.t["ids"].clone()
    rp[rp == 0] = 1
    rp[5] = torch.tensor([3, 3])
    node, grads = emulate(kind, inp, c, **gr, replay=rp)
    _check(node, grads, gr, replay=rp)


MUTANTS = {
    "hf_twice": "out",
    "tw_swap": "out",
    "expert_shift": "h",
    "g_rw_ignored": "g_x|g_h|g_gate_w",
    "g_x_gate_dropped": "g_x|g_h",
    "residual_missing": "g_residual|g_h",
    "residual_gets_g_comb": "g_residual|g_h",
    "w13_halves": "g_w13",
    "g_a_shift": "g_w13|g_x|g_h",
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
@pytest.mark.parametrize("kind", ["moe", "block"])
def test_each_planted_mistake_is_rejected(kind, mutant):
    c = dict(CONFIGS["softmax"], hf=0.5) if mutant in ("hf_twice", "residual_gets_g_comb") else CONFIGS["softmax"]
    inp, gr = inputs(kind, c, seed=2)
    node, grads = emulate(kind, inp, c, **gr, mutate=mutant)
    with pytest.raises(AssertionError, match=rf"^({MUTANTS[mutant]})\b.*first") as ei:
        _check(node, grads, gr)
    print(f"{kind} {mutant}: {str(ei.value)[:200]}")
