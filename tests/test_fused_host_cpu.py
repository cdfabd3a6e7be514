"""CPU coverage of the shipped host orchestration of the fused MoE layer (``xtuner_b200/fused.py``): the two autograd
nodes run forward+backward against ``tests/cabi_emulator.EmulatedLib`` (host-memory emulation of the C-ABI, written from
the header's contract) and must agree with the oracle under torch autograd.  What this pins: buffer shapes/dtypes,
argument order at every call, the backward chain (which saved tensor feeds which product, where gradients are
summed), optional paths (no residual, norm-weight grad not needed, one-launch vs separate gate/router entry points by
shape).  The kernels themselves are covered by the `-m gpu` parity tests."""
import pytest
import torch
from torch.nn import functional as F

from oracle import moe_oracle as O
from tests.cabi_emulator import EmulatedLib


@pytest.fixture
def emu(monkeypatch):
    from xtuner_b200 import _capi, fused, ops

    lib = EmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    monkeypatch.setattr(fused, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "permute_workspace", lambda T, K, E, dev: torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8))
    monkeypatch.setattr(ops, "_scratch", lambda tag, n, dev: torch.empty(max(int(n), 16), dtype=torch.uint8))
    return lib


def _weights(T, H, I, E, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16)
    gate_w = torch.randn(E, H, generator=g) * 0.3
    w13 = (torch.randn(E * 2 * I, H, generator=g) * H**-0.5).to(torch.bfloat16)
    w2 = (torch.randn(E * H, I, generator=g) * I**-0.5).to(torch.bfloat16)
    g_out = torch.randn(T, H, generator=g).to(torch.bfloat16)
    g_rw = torch.randn(T, E, generator=g) * 0.01
    g_lg = torch.randn(T, E, generator=g) * 0.01
    return x, gate_w, w13, w2, g_out, g_rw, g_lg


def _close(a, b, what, frac=0.01, tol=3e-2):
    a, b = a.float(), b.float()
    bad = (a - b).abs() > tol * (1 + b.abs())
    assert bad.float().mean() <= frac, f"{what}: {bad.float().mean():.4f} of elements off (max {(a - b).abs().max():.3e})"


@pytest.mark.parametrize("has_res,hidden_factor", [(True, 1.0), (False, 0.5)])
def test_fused_moe_function_matches_oracle_autograd(emu, monkeypatch, has_res, hidden_factor):
    from xtuner_b200 import fused

    T, H, I, E, K = 96, 128, 256, 8, 2
    x, gate_w, w13, w2, g_out, g_rw, g_lg = _weights(T, H, I, E, 1)
    res = torch.randn(T, H).to(torch.bfloat16) if has_res else None
    leaves = [t.clone().requires_grad_(True) for t in (x, gate_w, w13, w2)] + ([res.clone().requires_grad_(True)] if has_res else [])
    xr, gr, w13r, w2r = leaves[:4]
    ref = O.moe_layer_forward(xr, gr, w13r, w2r, K, True, 1.0, hidden_factor, residual=leaves[4] if has_res else None)
    ref_grads = torch.autograd.grad(
        [ref["hidden_states"], ref["router.router_weights"], ref["router.logits"]], leaves, [g_out, g_rw, g_lg])

    ours = [t.clone().requires_grad_(True) for t in (x, gate_w, w13, w2)] + ([res.clone().requires_grad_(True)] if has_res else [])
    out, logits, rw, ids, tpe = fused.FusedMoEFunction.apply(
        ours[0], ours[4] if has_res else None, ours[1], ours[2], ours[3], K, True, 1.0, hidden_factor, 0)
    assert torch.equal(ids, ref["router.topk_ids"]) and torch.equal(tpe, ref["tokens_per_expert"])
    _close(out, ref["hidden_states"], "hidden_states")
    torch.testing.assert_close(logits, ref["router.logits"], rtol=1e-5, atol=1e-5)
    grads = torch.autograd.grad([out, rw, logits], ours, [g_out, g_rw, g_lg])
    for name, a, b in zip(["x", "gate_w", "w13", "w2", "residual"], grads, ref_grads):
        _close(a, b, f"grad {name}")
    assert "xtb_swiglu_bwd" in emu.calls
    assert emu.calls.count("xtb_group_gemm_tn") == 2 and emu.calls.count("xtb_group_gemm_nn") == 2


@pytest.mark.parametrize("need_norm_grad", [True, False])
def test_fused_moe_block_function_matches_oracle_autograd(emu, monkeypatch, need_norm_grad):
    from xtuner_b200 import fused

    T, H, I, E, K = 80, 128, 256, 4, 2
    eps = 1e-6
    h, gate_w, w13, w2, g_out, g_rw, g_lg = _weights(T, H, I, E, 2)
    norm_w = 1.0 + 0.1 * torch.randn(H)

    hr, nr, gr, w13r, w2r = (t.clone().requires_grad_(True) for t in (h, norm_w, gate_w, w13, w2))
    x = F.rms_norm(hr.float(), (H,), nr, eps).to(torch.bfloat16)
    ref = O.moe_layer_forward(x, gr, w13r, w2r, K, True, 1.0, 1.0, residual=hr)
    ref_grads = torch.autograd.grad([ref["hidden_states"], ref["router.router_weights"], ref["router.logits"]],
                                    [hr, nr, gr, w13r, w2r], [g_out, g_rw, g_lg])

    ho, no, go, w13o, w2o = (t.clone().requires_grad_(True) for t in (h, norm_w, gate_w, w13, w2))
    if not need_norm_grad:
        no = norm_w.clone()
    out, logits, rw, ids, tpe = fused.FusedMoEBlockFunction.apply(ho, no, eps, go, w13o, w2o, K, True, 1.0, 1.0, 0)
    assert torch.equal(ids, ref["router.topk_ids"])
    _close(out, ref["hidden_states"], "hidden_states")
    leaves = [ho, no, go, w13o, w2o] if need_norm_grad else [ho, go, w13o, w2o]
    grads = torch.autograd.grad([out, rw, logits], leaves, [g_out, g_rw, g_lg])
    refs = list(ref_grads) if need_norm_grad else [ref_grads[0]] + list(ref_grads[2:])
    names = ["h", "norm_w", "gate_w", "w13", "w2"] if need_norm_grad else ["h", "gate_w", "w13", "w2"]
    for name, a, b in zip(names, grads, refs):
        _close(a, b, f"grad {name}", tol=5e-2)
    assert "xtb_moe_dispatch_bwd_rmsnorm" in emu.calls and "xtb_rmsnorm_gate" in emu.calls


@pytest.mark.parametrize("tag", ["grouped", "ungrouped", "nonorm"])
def test_noaux_router_autograd_wiring(emu, monkeypatch, tag):
    """``router._NoAuxRoute`` (what is saved, which grads reach the backward entry, has_group_mask) against the
    reference-made gradient fixture, with the C-ABI emulated."""
    from tests.conftest import load_golden
    from xtuner_b200 import router

    monkeypatch.setattr(router, "current_stream", lambda: None)
    g = load_golden("noaux_router_bwd")[tag]
    lg = g["logits"].clone().requires_grad_(True)
    rw, tw, ids, ids32, tpe = router._NoAuxRoute.apply(
        lg, g["e_score_correction_bias"], g["top_k"], g["n_group"], g["topk_group"], g["norm_topk_prob"], g["router_scaling_factor"])
    assert torch.equal(ids, g["topk_ids"]) and ids32.dtype == torch.int32 and tpe.dtype == torch.float32
    tol = dict(rtol=2e-5, atol=2e-6)
    (a,) = torch.autograd.grad(tw, lg, g["grad_topk_weights"], retain_graph=True)
    torch.testing.assert_close(a, g["grad_logits_from_topk"], **tol)
    (b,) = torch.autograd.grad(rw, lg, g["grad_router_weights"], retain_graph=True)
    torch.testing.assert_close(b, g["grad_logits_from_router_weights"], **tol)
    (c,) = torch.autograd.grad([tw, rw], lg, [g["grad_topk_weights"], g["grad_router_weights"]])
    torch.testing.assert_close(c, g["grad_logits"], **tol)


def test_module_path_moe_layer_matches_golden_layer(emu, monkeypatch):
    """The per-op module path (``moe.MoELayer``: MoEGate -> GreedyRouter -> FusedDispatcher -> MoEBlock -> combine) with
    the C-ABI emulated, against the reference-made layer fixture (outputs and all gradients)."""
    import functools

    from tests.conftest import load_golden
    from xtuner_b200 import moe, ops, router

    for mod in (ops, router):
        monkeypatch.setattr(mod, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)

    def route_nocheck(logits, top_k, norm_topk_prob=True, router_scaling_factor=1.0, scoring_func="softmax"):
        rw, tw, ids, ids32, tpe = router._GreedyRoute.apply(logits.float().contiguous(), top_k, router.SCORING[scoring_func],
                                                            norm_topk_prob, router_scaling_factor)
        return {"logits": logits, "router_weights": rw, "topk_weights": tw, "topk_ids": ids, "topkens_per_expert": tpe}, ids32

    monkeypatch.setattr(router, "greedy_route", route_nocheck)
    g = load_golden("moe_layer_ragged")
    _, T, H = g["x"].shape
    E = g["n_experts"]
    I = g["w2"].shape[1]
    layer = moe.MoELayer(hidden_size=H, moe_intermediate_size=I, n_routed_experts=E, num_experts_per_tok=g["top_k"])
    layer.experts.to(torch.bfloat16)
    with torch.no_grad():
        layer.gate.weight.copy_(g["gate_weight"])
        layer.experts.fused_w1w3.weight.copy_(g["w13"])
        layer.experts.fused_w2.weight.copy_(g["w2"])
    x = g["x"].clone().requires_grad_(True)
    res = g["residual"].clone().requires_grad_(True)
    out, rr = layer(x, res)
    assert torch.equal(rr["topk_ids"], g["topk_ids"]) and torch.equal(rr["topkens_per_expert"], g["tokens_per_expert"])
    assert torch.equal(out, g["out"])  # the emulator is oracle arithmetic, and the oracle is pinned bit-exact to this fixture
    params = [layer.gate.weight, layer.experts.fused_w1w3.weight, layer.experts.fused_w2.weight]
    gx, gg, g13, g2 = torch.autograd.grad(out, [x] + params, g["grad_out"])
    assert torch.equal(gx, g["grad_x"])
    torch.testing.assert_close(gg, g["grad_gate_weight"], rtol=1e-5, atol=1e-6)
    assert torch.equal(g13, g["grad_w13"]) and torch.equal(g2, g["grad_w2"])
    assert {"xtb_gate_logits", "xtb_router_greedy", "xtb_moe_permute", "xtb_moe_unpermute", "xtb_gate_logits_bwd"} <= set(emu.calls)


@pytest.mark.parametrize("tag", ["layer_k4_hf", "layer_sigmoid"])
def test_fused_moe_function_on_reference_variants(emu, tag):
    """hidden_factor != 1, top-4, un-normalised scaled router, sigmoid scoring: the fused node's host orchestration
    against reference-made outputs and gradients (fixture `variants`)."""
    from tests.conftest import load_golden
    from xtuner_b200 import fused
    from xtuner_b200.router import SCORING

    g = load_golden("variants")[tag]
    T = g["x"].shape[1]
    leaves = [g["x"].view(T, -1).clone().requires_grad_(True), g["residual"].view(T, -1).clone().requires_grad_(True),
              g["gate_weight"].clone().requires_grad_(True), g["w13"].clone().requires_grad_(True), g["w2"].clone().requires_grad_(True)]
    out, logits, rw, ids, tpe = fused.FusedMoEFunction.apply(
        leaves[0], leaves[1], leaves[2], leaves[3], leaves[4], g["top_k"], g["norm_topk_prob"], g["router_scaling_factor"],
        g["hidden_factor"], SCORING[g["scoring_func"]])
    assert torch.equal(ids, g["topk_ids"]) and torch.equal(tpe, g["tokens_per_expert"])
    assert torch.equal(logits, g["logits"])
    assert torch.equal(out, g["out"].view(T, -1))  # forward: emulator == oracle arithmetic == reference bits
    gx, gres, ggw, g13, g2 = torch.autograd.grad(out, leaves, g["grad_out"].view(T, -1))
    assert torch.equal(gres, g["grad_out"].view(T, -1))
    _close(gx, g["grad_x"].view(T, -1), "grad x")
    _close(ggw, g["grad_gate_weight"], "grad gate", tol=5e-2)
    _close(g13, g["grad_w13"], "grad w13")
    _close(g2, g["grad_w2"], "grad w2")


@pytest.mark.parametrize("tag", ["c2", "k8", "empty_expert"])
def test_op_protocol_permute_unpermute_on_reference_fixtures(emu, monkeypatch, tag):
    """``ops.permute`` / ``ops.unpermute`` (protocol callables + their autograd Functions) over the emulated C-ABI against
    the reference-made dispatch fixtures: outputs and gradients bit-exact."""
    from tests.conftest import load_golden
    from xtuner_b200 import ops

    monkeypatch.setattr(ops, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    g = load_golden(f"dispatch_{tag}")
    x = g["x"].clone().requires_grad_(True)
    perm, rmap = ops.permute(x, g["topk_ids"], n_experts=g["n_experts"])
    assert torch.equal(perm, g["permuted"]) and rmap.dtype == torch.int32 and rmap.numel() == g["topk_ids"].numel()
    (gx,) = torch.autograd.grad(perm, x, g["grad_permuted"])
    assert torch.equal(gx, g["grad_x"])
    y = g["y"].clone().requires_grad_(True)
    p = g["probs"].clone().requires_grad_(True)
    out = ops.unpermute(y, rmap, p)
    assert torch.equal(out, g["out"])
    gy, gp = torch.autograd.grad(out, (y, p), g["grad_out"])
    assert torch.equal(gy, g["grad_y"])
    torch.testing.assert_close(gp, g["grad_probs"], rtol=1e-6, atol=1e-6)
    # zero-token inputs stay in the graph (permute_unpermute.py:101-102, group_gemm.py:34-36)
    e = torch.zeros(0, x.shape[1], dtype=torch.bfloat16, requires_grad=True)
    pe, me = ops.permute(e, torch.zeros(0, 2, dtype=torch.int32), n_experts=4)
    assert pe is e and me is None
    w = torch.randn(4, 128, x.shape[1]).to(torch.bfloat16).requires_grad_(True)
    ge = ops.group_gemm(e, w, torch.zeros(4, dtype=torch.int64))
    assert ge.shape == (0, 128) and ge.requires_grad


@pytest.mark.parametrize("E", [8, 16])
@pytest.mark.parametrize("block", [False, True])
def test_route_entry_points_follow_the_shape(emu, block, E):
    """Both fused nodes at H = 128: E = 8 runs the gate + router forward as xtb_gate_route_dispatch and the router + gate
    backward as xtb_router_gate_bwd, E = 16 the separate calls each of them replaces.  Outputs and gradients against
    the oracle either way."""
    from xtuner_b200 import fused

    T, H, I, K, eps = 64, 128, 256, 2, 1e-6
    h, gate_w, w13, w2, g_out, g_rw, g_lg = _weights(T, H, I, E, 5)
    norm_w = 1.0 + 0.1 * torch.randn(H, generator=torch.Generator().manual_seed(E))

    hr, gr = (t.clone().requires_grad_(True) for t in (h, gate_w))
    x = F.rms_norm(hr.float(), (H,), norm_w, eps).to(torch.bfloat16) if block else hr
    ref = O.moe_layer_forward(x, gr, w13, w2, K, True, 1.0, 1.0, residual=hr if block else None)
    ref_grads = torch.autograd.grad([ref["hidden_states"], ref["router.router_weights"], ref["router.logits"]], [hr, gr],
                                    [g_out, g_rw, g_lg])

    emu.calls.clear()
    ho, go = (t.clone().requires_grad_(True) for t in (h, gate_w))
    if block:
        out, logits, rw, ids, tpe = fused.FusedMoEBlockFunction.apply(ho, norm_w, eps, go, w13, w2, K, True, 1.0, 1.0, 0)
    else:
        out, logits, rw, ids, tpe = fused.FusedMoEFunction.apply(ho, None, go, w13, w2, K, True, 1.0, 1.0, 0)
    fwd = list(emu.calls)
    grads = torch.autograd.grad([out, rw, logits], [ho, go], [g_out, g_rw, g_lg])
    bwd = emu.calls[len(fwd):]

    one_launch = {"xtb_gate_route_dispatch", "xtb_router_gate_bwd"}
    split = {"xtb_gate_logits", "xtb_router_greedy_dispatch", "xtb_router_greedy_bwd", "xtb_gate_logits_bwd"}
    called = set(emu.calls)
    want, unwanted = (one_launch, split) if E <= 8 else (split, one_launch)
    assert want <= called and not (unwanted & called), sorted(called)
    # the launch order: the block node is the plain node with the norm ahead of it and the norm backward as its last
    # launch in place of the dispatch backward (the emulator logs xtb_group_gemm_tn_pair after its two inner tn calls)
    route = ["xtb_gate_route_dispatch"] if E <= 8 else ["xtb_gate_logits", "xtb_router_greedy_dispatch"]
    route_bwd = ["xtb_router_gate_bwd"] if E <= 8 else ["xtb_router_greedy_bwd", "xtb_gate_logits_bwd"]
    moe_fwd = route + ["xtb_moe_permute_prepared", "xtb_group_gemm_nt_swiglu", "xtb_group_gemm_nt", "xtb_moe_combine"]
    moe_bwd = ["xtb_moe_unpermute_bwd", "xtb_group_gemm_nn", "xtb_swiglu_bwd", "xtb_group_gemm_nn", "xtb_group_gemm_tn",
               "xtb_group_gemm_tn", "xtb_group_gemm_tn_pair"] + route_bwd
    assert fwd == (["xtb_rmsnorm_gate"] + moe_fwd if block else moe_fwd), fwd
    assert bwd == moe_bwd + (["xtb_moe_dispatch_bwd_rmsnorm"] if block else ["xtb_moe_combine"]), bwd
    assert torch.equal(ids, ref["router.topk_ids"]) and torch.equal(tpe, ref["tokens_per_expert"])
    _close(out, ref["hidden_states"], "hidden_states")
    torch.testing.assert_close(logits, ref["router.logits"], rtol=1e-5, atol=1e-5)
    for name, a, b in zip(["h" if block else "x", "gate_w"], grads, ref_grads):
        _close(a, b, f"grad {name}", tol=5e-2)
