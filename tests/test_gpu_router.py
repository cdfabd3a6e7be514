"""GPU parity of the router kernels against golden vectors (made by the reference's own code) and
the CPU oracle.  Bit-exact integer outputs; fp32 outputs to 1e-6 (exp implementation differs by ulps)."""
import pytest
import torch

from oracle import moe_oracle as O
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu

F32_TOL = dict(rtol=2e-6, atol=1e-7)


@pytest.mark.parametrize("tag", ["c2", "q3", "skew"])
def test_greedy_router_golden(tag):
    from xtuner_b200.router import greedy_route

    g = load_golden(f"greedy_router_{tag}")
    lg = g["logits"].cuda().requires_grad_(True)
    res, ids32 = greedy_route(lg, g["top_k"], g["norm_topk_prob"], g["router_scaling_factor"])
    assert res["topk_ids"].dtype == torch.int64
    assert torch.equal(res["topk_ids"].cpu(), g["topk_ids"])
    assert torch.equal(ids32.cpu().long(), g["topk_ids"])
    assert res["topkens_per_expert"].dtype == torch.int64
    assert torch.equal(res["topkens_per_expert"].cpu(), g["tokens_per_expert"])
    torch.testing.assert_close(res["router_weights"].cpu(), g["router_weights"], **F32_TOL)
    torch.testing.assert_close(res["topk_weights"].cpu(), g["topk_weights"], **F32_TOL)
    loss = (res["topk_weights"] * g["grad_topk_weights"].cuda()).sum() + (
        res["router_weights"] * g["grad_router_weights"].cuda()
    ).sum()
    loss.backward()
    torch.testing.assert_close(lg.grad.cpu(), g["grad_logits"], rtol=1e-4, atol=2e-6)


@pytest.mark.parametrize("T,E,K", [(8192, 8, 2), (4096, 128, 8), (1000, 64, 6), (33, 32, 4), (5000, 256, 8)])
def test_greedy_router_vs_oracle_large(T, E, K):
    from xtuner_b200.router import greedy_route

    g = torch.Generator().manual_seed(T + E)
    logits = torch.randn(T, E, generator=g) * 3
    ref = O.greedy_router(logits, K)
    # tie-free rows only (torch.topk tie order is implementation-defined; SURVEY.md §7)
    # (only the top K+1 values decide the selection)
    srt = ref["router_weights"].topk(K + 1, dim=1).values
    assert (srt[:, 1:] != srt[:, :-1]).all(), "test input has ties among the top-(K+1); change the seed"
    res, _ = greedy_route(logits.cuda(), K)
    got = res["topk_ids"].cpu()
    if not torch.equal(got, ref["topk_ids"]):
        # rows may legitimately differ only where two *distinct* logits round to softmax values whose
        # order flips between exp implementations; require none on these seeds
        bad = (got != ref["topk_ids"]).any(dim=1).nonzero().flatten()
        raise AssertionError(f"{bad.numel()} rows differ, first {bad[:5].tolist()}")
    assert torch.equal(res["topkens_per_expert"].cpu(), ref["topkens_per_expert"])
    assert int(res["topkens_per_expert"].sum()) == T * K
    torch.testing.assert_close(res["topk_weights"].cpu(), ref["topk_weights"], **F32_TOL)


def test_noaux_router_golden():
    from xtuner_b200.router import NoAuxRouter

    g = load_golden("noaux_router_dsv3")
    E = g["logits"].shape[1]
    r = NoAuxRouter(
        n_routed_experts=E, num_experts_per_tok=g["top_k"], router_scaling_factor=g["router_scaling_factor"],
        scoring_func="sigmoid", n_group=g["n_group"], topk_group=g["topk_group"],
    ).cuda()
    r.e_score_correction_bias.copy_(g["e_score_correction_bias"])
    res = r(g["logits"].cuda())
    assert torch.equal(res["topk_ids"].cpu(), g["topk_ids"])
    assert res["topkens_per_expert"].dtype == torch.float32
    assert torch.equal(res["topkens_per_expert"].cpu(), g["tokens_per_expert"])
    torch.testing.assert_close(res["topk_weights"].cpu(), g["topk_weights"], **F32_TOL)
    torch.testing.assert_close(res["router_weights"].cpu(), g["router_weights"], rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("T,H,E", [(8192, 2048, 8), (777, 512, 8), (300, 256, 16), (257, 320, 40), (0, 256, 8),
                                   (250_000, 64, 8), (120_000, 64, 16)])
def test_gate_logits_and_bwd(T, H, E):
    """the two large T: more tokens than one block per SM can hold in 48 KB of dynamic shared memory (the block count grows
    instead); T=0: an empty micro-batch gives zero weight gradients, as autograd's sums over no rows do"""
    from xtuner_b200 import ops

    g = torch.Generator().manual_seed(T)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16)
    w = torch.randn(E, H, generator=g) * 0.05
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ref = O.gate_logits(xr, wr)
    gl = torch.randn(T, E, generator=g)
    gx_ref, gw_ref = torch.autograd.grad(ref, (xr, wr), gl)
    xd, wd = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    out = ops.gate_logits(xd, wd)
    torch.testing.assert_close(out.cpu(), ref.detach(), rtol=1e-4, atol=1e-4)
    gx, gw = torch.autograd.grad(out, (xd, wd), gl.cuda())  # E > 16 takes the strided-SGEMM backward
    torch.testing.assert_close(gw.cpu(), gw_ref, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(gx.float().cpu(), gx_ref.float(), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("T,E,K", [(8192, 8, 2), (1000, 128, 8), (4100, 64, 6), (31, 16, 2), (2500, 256, 8)])
def test_router_dispatch_fused_workspace(T, E, K):
    """xtb_router_greedy_dispatch (+ xtb_moe_permute_prepared) == xtb_router_greedy + xtb_moe_permute."""
    from xtuner_b200 import _capi, ops
    from xtuner_b200._capi import check, current_stream, ptr

    lib = _capi.ensure_init()
    g = torch.Generator().manual_seed(T + E)
    logits = (torch.randn(T, E, generator=g) * 3).cuda()
    H = 64
    x = torch.randn(T, H, generator=g).to(torch.bfloat16).cuda()
    dev = x.device

    def bufs():
        return (torch.empty(T, E, device=dev), torch.empty(T, K, device=dev), torch.empty(T, K, dtype=torch.int64, device=dev),
                torch.empty(T, K, dtype=torch.int32, device=dev), torch.empty(E, dtype=torch.int64, device=dev))

    rw1, tw1, ids1, i32_1, tpe1 = bufs()
    check(lib.xtb_router_greedy(ptr(logits), T, E, K, 0, 1, 1.0, ptr(rw1), ptr(tw1), ptr(ids1), ptr(i32_1), ptr(tpe1), current_stream()))
    perm1, rmap1, sorted1, tpe_p = ops.permute(x, i32_1, n_experts=E, return_extra=True)

    rw2, tw2, ids2, i32_2, tpe2 = bufs()
    ws = torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8, device=dev)
    check(lib.xtb_router_greedy_dispatch(ptr(logits), T, E, K, 0, 1, 1.0, ptr(rw2), ptr(tw2), ptr(ids2), ptr(i32_2), ptr(tpe2), ptr(ws), current_stream()))
    perm2 = torch.empty_like(perm1)
    rmap2 = torch.empty_like(rmap1)
    sorted2 = torch.empty_like(sorted1)
    check(lib.xtb_moe_permute_prepared(ptr(x), ptr(i32_2), T, K, E, H * 2, ptr(perm2), ptr(rmap2), ptr(sorted2), ptr(ws), current_stream()))
    assert torch.equal(ids1, ids2) and torch.equal(tw1, tw2) and torch.equal(rw1, rw2)
    assert torch.equal(tpe1, tpe2) and torch.equal(tpe1, tpe_p) and int(tpe2.sum()) == T * K
    assert torch.equal(rmap1, rmap2) and torch.equal(sorted1, sorted2) and torch.equal(perm1, perm2)


@pytest.mark.parametrize("tag", ["grouped", "ungrouped", "nonorm"])
def test_noaux_router_backward_golden(tag):
    """Gradients through topk_weights and router_weights vs the reference's own autograd (fixture noaux_router_bwd)."""
    from xtuner_b200.router import NoAuxRouter

    g = load_golden("noaux_router_bwd")[tag]
    E = g["logits"].shape[1]
    r = NoAuxRouter(
        n_routed_experts=E, num_experts_per_tok=g["top_k"], router_scaling_factor=g["router_scaling_factor"],
        scoring_func="sigmoid", n_group=g["n_group"], topk_group=g["topk_group"], norm_topk_prob=g["norm_topk_prob"],
    ).cuda()
    r.e_score_correction_bias.copy_(g["e_score_correction_bias"])
    lg = g["logits"].cuda().requires_grad_(True)
    res = r(lg)
    assert torch.equal(res["topk_ids"].cpu(), g["topk_ids"])
    g_tw, g_rw = g["grad_topk_weights"].cuda(), g["grad_router_weights"].cuda()
    tol = dict(rtol=1e-4, atol=1e-6)  # fp32; expf vs torch's sigmoid differ by a few ulps
    (a,) = torch.autograd.grad(res["topk_weights"], lg, g_tw, retain_graph=True)
    torch.testing.assert_close(a.cpu(), g["grad_logits_from_topk"], **tol)
    (b,) = torch.autograd.grad(res["router_weights"], lg, g_rw, retain_graph=True)
    torch.testing.assert_close(b.cpu(), g["grad_logits_from_router_weights"], **tol)
    (c,) = torch.autograd.grad([res["topk_weights"], res["router_weights"]], lg, [g_tw, g_rw])
    torch.testing.assert_close(c.cpu(), g["grad_logits"], **tol)


@pytest.mark.parametrize("tag", ["router_sigmoid_norm", "router_sigmoid_raw", "router_softmax_k1"])
def test_greedy_router_variants_golden(tag):
    """Validated kernels, parameter corners not covered by the default suite yet (fixture `variants`): sigmoid scoring,
    un-normalised scaled weights, top-1.  Promote to test_gpu_router.py once green."""
    from xtuner_b200.router import GreedyRouter

    g = load_golden("variants")[tag]
    E = g["logits"].shape[1]
    r = GreedyRouter(n_routed_experts=E, num_experts_per_tok=g["top_k"], norm_topk_prob=g["norm_topk_prob"],
                     scoring_func=g["scoring_func"], router_scaling_factor=g["router_scaling_factor"])
    lg = g["logits"].cuda().requires_grad_(True)
    res = r(lg)
    assert torch.equal(res["topk_ids"].cpu(), g["topk_ids"])
    assert torch.equal(res["topkens_per_expert"].cpu(), g["tokens_per_expert"])
    torch.testing.assert_close(res["topk_weights"].cpu(), g["topk_weights"], rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(res["router_weights"].cpu(), g["router_weights"], rtol=1e-5, atol=1e-7)
    (gl,) = torch.autograd.grad([res["topk_weights"], res["router_weights"]], lg,
                                [g["grad_topk_weights"].cuda(), g["grad_router_weights"].cuda()])
    torch.testing.assert_close(gl.cpu(), g["grad_logits"], rtol=1e-4, atol=1e-6)
