"""Routing replay (RL rollout-routed experts) on an H100: xtb_router_greedy_replay, xtb_gate_route_replay_dispatch,
xtb_router_noaux_replay and the host layers above them (router.py custom ops, the fused MoE node).

* Replaying the ids a routing entry chose reproduces every output of that entry bit for bit, the dispatch workspace
  included: every XTB_ROUTER_DISPATCH instantiation (E = 8 to 512), the tensor-core gate + route kernel, and the
  no-aux router with and without the group mask.
* Random ids with duplicates and ids the router would not pick: forward and the existing backward entries against
  float64 replay references written here (tests/router_reference.py's greedy_bwd_ref picks its own top-k).
* The strided [:, l, :] slice of an [S, L, K] tensor equals its contiguous copy; T = 0, 1 and T not a multiple of 32.
* Ids outside [0, E): id 0, NaN weights for that token only, counted under expert 0, and a permute + combine over those
  outputs stays in bounds (NaN rows for that token, the others untouched).
* The fixture made by the reference's own routers (tests/golden/router_replay.pt) through the routers, all four id
  patterns, to the standard of the routing fixtures.
* The fused node: its own routing replayed equals the routing node bit for bit, forward and every gradient; random ids
  match the per-op path; forward + backward replays in a CUDA graph; opcheck on both new custom ops."""
import pytest
import torch

from tests.router_reference import check_bound
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ws(T, K, E):
    return torch.zeros(int(ensure_init().xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8, device=DEV)


def _outs(T, E, K):
    """NaN / -7 filled outputs; at T = 0 still real (non-null) addresses, as the entries require"""
    n, i64 = max(T, 1), torch.int64
    return dict(rw=torch.full((n, E), float("nan"), device=DEV)[:T], tw=torch.full((n, K), float("nan"), device=DEV)[:T],
                ids=torch.full((n, K), -7, dtype=i64, device=DEV)[:T],
                ids32=torch.full((n, K), -7, dtype=torch.int32, device=DEV)[:T], tpe=torch.full((E,), -7, dtype=i64, device=DEV))


def greedy_route(logits, K, scoring, norm, scaling, ws=None):
    T, E = logits.shape
    o = _outs(T, E, K)
    if ws is None:
        rc = ensure_init().xtb_router_greedy(ptr(logits), T, E, K, scoring, int(norm), float(scaling), ptr(o["rw"]),
                                             ptr(o["tw"]), ptr(o["ids"]), ptr(o["ids32"]), ptr(o["tpe"]),
                                             current_stream())
    else:
        rc = ensure_init().xtb_router_greedy_dispatch(ptr(logits), T, E, K, scoring, int(norm), float(scaling),
                                                      ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]), ptr(o["ids32"]),
                                                      ptr(o["tpe"]), ptr(ws), current_stream())
    check(rc, "route")
    return o


def greedy_replay(logits, replay, scoring, norm, scaling, ws=None):
    T, E = logits.shape
    K = replay.shape[1]
    o = _outs(T, E, K)
    stride = replay.stride(0) if T else K
    check(ensure_init().xtb_router_greedy_replay(ptr(logits), ptr(replay), stride, T, E, K, scoring, int(norm),
                                                 float(scaling), ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]),
                                                 ptr(o["ids32"]), ptr(o["tpe"]), ptr(ws), current_stream()), "replay")
    return o


def _same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]) or (a[k].dtype.is_floating_point and torch.equal(a[k].view(torch.int32),
                                                                                        b[k].view(torch.int32))), f"{what}: {k}"


# ---- float64 replay references ---------------------------------------------------------------------------------------


def greedy_replay_ref(logits, ids, scoring, norm, scaling):
    """(router_weights, topk_weights) in float64 as greedy.py:70-86 computes them with replayed ids"""
    lg = logits.double()
    p = torch.softmax(lg, 1) if scoring == 0 else torch.sigmoid(lg)
    w = p.gather(1, ids)
    if norm:
        w = w / w.sum(1, keepdim=True)
    return p, w * scaling


def noaux_replay_ref(logits, bias, ids, K, n_group, topk_group, norm, scaling):
    lg = logits.double()
    s = torch.sigmoid(lg)
    ch = s + bias.double()
    if n_group != topk_group:
        T, E = lg.shape
        gs = ch.view(T, n_group, -1).topk(2, dim=-1)[0].sum(-1)
        gi = gs.topk(topk_group, dim=-1, sorted=False)[1]
        m = torch.zeros_like(gs).scatter_(1, gi, 1).unsqueeze(-1).expand(T, n_group, E // n_group).reshape(T, E)
        ch = ch.masked_fill(~m.bool(), 0.0)
    w = s.gather(1, ids)
    if K > 1 and norm:
        w = w / (w.sum(1, keepdim=True) + 1e-20)
    return ch / ch.sum(1, keepdim=True), w * scaling


def _rand_ids(T, E, K, g):
    ids = torch.randint(0, E, (T, K), generator=g)
    ids[::3, 0] = ids[::3, -1]  # duplicates in every third row
    return ids.to(DEV)


# ---- greedy router ---------------------------------------------------------------------------------------------------

E_ALL = [8, 16, 32, 64, 128, 256, 512]


@pytest.mark.parametrize("E", E_ALL)
@pytest.mark.parametrize("scoring,norm,scaling", [(0, True, 1.0), (1, False, 2.5), (0, False, 1.0), (1, True, 2.5)])
def test_greedy_replay_of_own_ids_is_the_routing_bit_for_bit(E, scoring, norm, scaling):
    g = torch.Generator().manual_seed(E)
    for K in sorted({1, 2, min(8, E)}):
        for T in (1, 31, 1000):
            logits = (torch.randn(T, E, generator=g) * 2).to(DEV)
            for with_ws in (False, True):
                ws_a = _ws(T, K, E) if with_ws else None
                ws_b = _ws(T, K, E) if with_ws else None
                a = greedy_route(logits, K, scoring, norm, scaling, ws_a)
                perm = a["ids"].clone()
                b = greedy_replay(logits, perm, scoring, norm, scaling, ws_b)
                _same(a, b, f"E={E} K={K} T={T} ws={with_ws}")
                if with_ws:
                    assert torch.equal(ws_a, ws_b)


@pytest.mark.parametrize("E,K", [(8, 2), (128, 8), (512, 8), (16, 1)])
@pytest.mark.parametrize("scoring,norm", [(0, True), (1, False), (1, True)])
def test_greedy_replay_random_ids_against_float64(E, K, scoring, norm):
    g = torch.Generator().manual_seed(7 * E + K)
    T, scaling = 333, 1.7
    logits = (torch.randn(T, E, generator=g) * 3).to(DEV)
    # random ids with duplicates; the last rows take the router's lowest-scored experts (never chosen)
    ids = _rand_ids(T, E, K, g)
    ids[-5:] = logits[-5:].argsort(1)[:, :K]
    o = greedy_replay(logits, ids, scoring, norm, scaling)
    assert torch.equal(o["ids"], ids) and torch.equal(o["ids32"], ids.int())
    assert torch.equal(o["tpe"].cpu(), torch.bincount(ids.flatten().cpu(), minlength=E))
    p64, w64 = greedy_replay_ref(logits.cpu(), ids.cpu(), scoring, norm, scaling)
    u = 2.0 ** -24
    # softmax: the row sum over E lanes is the widest error term
    check_bound(o["rw"].cpu(), p64, (16 + E) * u * p64.abs() + 1e-30, "router_weights")
    check_bound(o["tw"].cpu(), w64, (16 + E + 4 * K) * u * w64.abs() + 1e-30, "topk_weights")
    # backward through the existing entry: gather's backward with the replayed (duplicated) ids
    g_tw = torch.randn(T, K, generator=g).to(DEV)
    g_rw = torch.randn(T, E, generator=g).to(DEV)
    gl = torch.empty(T, E, device=DEV)
    check(ensure_init().xtb_router_greedy_bwd(ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]), ptr(g_tw), ptr(g_rw), None, T,
                                              E, K, scoring, int(norm), float(scaling), ptr(gl), current_stream()),
          "bwd")
    lg = logits.cpu().double().requires_grad_(True)
    p = torch.softmax(lg, 1) if scoring == 0 else torch.sigmoid(lg)
    w = p.gather(1, ids.cpu())
    if norm:
        w = w / w.sum(1, keepdim=True)
    ((w * scaling) * g_tw.cpu().double()).sum().add((p * g_rw.cpu().double()).sum()).backward()
    ref = lg.grad
    scale = ref.abs().amax(1, keepdim=True) + g_tw.abs().amax().item() * scaling + 1
    check_bound(gl.cpu(), ref, (64 + 2 * E) * u * scale, "grad_logits")


def test_greedy_replay_strided_slice_and_small_T():
    g = torch.Generator().manual_seed(3)
    E, K, L = 64, 4, 5
    for T in (0, 1, 33, 1000):
        logits = torch.randn(T, E, generator=g).to(DEV)
        full = torch.randint(0, E, (T, L, K), generator=g).to(DEV)
        sl = full[:, 2, :]
        a = greedy_replay(logits, sl, 0, True, 1.0, _ws(T, K, E))
        b = greedy_replay(logits, sl.contiguous(), 0, True, 1.0, _ws(T, K, E))
        _same(a, b, f"T={T}")
        if T == 0:
            assert int(a["tpe"].abs().sum()) == 0


def test_out_of_range_ids_give_nan_weights_for_that_token_only_and_stay_in_bounds():
    g = torch.Generator().manual_seed(11)
    T, E, K, H = 70, 8, 2, 128
    logits = torch.randn(T, E, generator=g).to(DEV)
    ids = _rand_ids(T, E, K, g)
    bad_rows = {5: -1, 17: E, 40: 2 ** 40}
    bad = ids.clone()
    for r, v in bad_rows.items():
        bad[r, 1] = v
    ws = _ws(T, K, E)
    o = greedy_replay(logits, bad, 0, True, 1.0, ws)
    ref = greedy_replay(logits, ids, 0, True, 1.0)
    rows = list(bad_rows)
    keep = torch.ones(T, dtype=torch.bool)
    keep[rows] = False
    assert torch.equal(o["tw"][keep.to(DEV)], ref["tw"][keep.to(DEV)]) and torch.equal(o["rw"], ref["rw"])
    assert torch.isnan(o["tw"][rows]).all()
    assert (o["ids"][rows, 1] == 0).all() and (o["ids32"][rows, 1] == 0).all()
    fixed = ids.clone()
    fixed[rows, 1] = 0
    assert torch.equal(o["ids"], fixed)
    assert torch.equal(o["tpe"].cpu(), torch.bincount(fixed.flatten().cpu(), minlength=E))
    # permute + combine over those outputs: in bounds, NaN rows only for the bad tokens
    lib = ensure_init()
    x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(DEV)
    xp = torch.empty(T * K, H, dtype=torch.bfloat16, device=DEV)
    rmap = torch.empty(T * K, dtype=torch.int32, device=DEV)
    check(lib.xtb_moe_permute_prepared(ptr(x), ptr(o["ids32"]), T, K, E, H * 2, ptr(xp), ptr(rmap), None, ptr(ws),
                                       current_stream()), "permute")
    out = torch.empty(T, H, dtype=torch.bfloat16, device=DEV)
    check(lib.xtb_moe_combine(ptr(xp), ptr(rmap), ptr(o["tw"]), None, 1.0, T, K, H, ptr(out), current_stream()),
          "combine")
    torch.cuda.synchronize()
    assert torch.isnan(out[rows].float()).all()
    assert torch.isfinite(out[keep.to(DEV)].float()).all()
    assert sorted(rmap.cpu().tolist()) == list(range(T * K))
    # the gate + route kernel and the no-aux router follow the same rule
    wg = torch.randn(E, H, generator=g).to(DEV) * 0.05
    go = _gate_route(x, wg, bad, 0, True, 1.0, _ws(T, K, E), replay=True)
    assert torch.isnan(go["tw"][rows]).all() and torch.equal(go["ids"], fixed)
    E2 = 64
    lg2 = torch.randn(T, E2, generator=g).to(DEV)
    bias = torch.zeros(E2, device=DEV)
    ids2 = _rand_ids(T, E2, K, g)
    ids2[5, 0] = -1
    n = noaux_replay(lg2, bias, ids2, 8, 4, True, 2.5)
    assert torch.isnan(n["tw"][5]).all() and int(n["ids"][5, 0]) == 0 and torch.isfinite(n["tw"][6:]).all()


# ---- gate + route (tensor cores) --------------------------------------------------------------------------------------


def _gate_route(x, w, K_or_ids, scoring, norm, scaling, ws, replay=False):
    T, H = x.shape
    E = w.shape[0]
    K = K_or_ids.shape[1] if replay else K_or_ids
    o = _outs(T, E, K)
    o["logits"] = torch.full((T, E), float("nan"), device=DEV)
    if replay:
        rc = ensure_init().xtb_gate_route_replay_dispatch(ptr(x), ptr(w), ptr(K_or_ids), K_or_ids.stride(0) if T else K,
                                                          T, H, E, K, scoring, int(norm), float(scaling),
                                                          ptr(o["logits"]), ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]),
                                                          ptr(o["ids32"]), ptr(o["tpe"]), ptr(ws), current_stream())
    else:
        rc = ensure_init().xtb_gate_route_dispatch(ptr(x), ptr(w), T, H, E, K, scoring, int(norm), float(scaling),
                                                   ptr(o["logits"]), ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]),
                                                   ptr(o["ids32"]), ptr(o["tpe"]), ptr(ws), current_stream())
    check(rc, "gate_route")
    return o


@pytest.mark.parametrize("E,K,H", [(8, 2, 2048), (4, 4, 256), (8, 8, 4096), (1, 1, 128)])
def test_gate_route_replay_of_own_ids_is_the_routing_bit_for_bit(E, K, H):
    g = torch.Generator().manual_seed(E * 100 + H)
    for T in (1, 45, 4096):
        x = torch.randn(T, H, generator=g).to(torch.bfloat16).to(DEV)
        w = (torch.randn(E, H, generator=g) * 0.05).to(DEV)
        ws_a, ws_b = _ws(T, K, E), _ws(T, K, E)
        a = _gate_route(x, w, K, 0, True, 1.0, ws_a)
        full = torch.stack([a["ids"], a["ids"]], 1)  # [T, 2, K]: replay a strided slice
        b = _gate_route(x, w, full[:, 1, :], 0, True, 1.0, ws_b, replay=True)
        _same(a, b, f"T={T}")
        assert torch.equal(ws_a, ws_b)
        # random ids: the replay router on the same logits
        ids = _rand_ids(T, E, K, g)
        c = _gate_route(x, w, ids, 1, False, 2.5, _ws(T, K, E), replay=True)
        d = greedy_replay(c["logits"], ids, 1, False, 2.5)
        _same({k: c[k] for k in d}, d, f"random T={T}")


# ---- no-aux router -----------------------------------------------------------------------------------------------------


def noaux_route(logits, bias, K, n_group, topk_group, norm, scaling):
    T, E = logits.shape
    o = _outs(T, E, K)
    o["tpe"] = torch.full((E,), -7.0, device=DEV)
    check(ensure_init().xtb_router_noaux(ptr(logits), ptr(bias), T, E, K, n_group, topk_group, int(norm),
                                         float(scaling), ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]), ptr(o["ids32"]),
                                         ptr(o["tpe"]), current_stream()), "noaux")
    return o


def noaux_replay(logits, bias, replay, n_group, topk_group, norm, scaling):
    T, E = logits.shape
    K = replay.shape[1]
    o = _outs(T, E, K)
    o["tpe"] = torch.full((E,), -7.0, device=DEV)
    check(ensure_init().xtb_router_noaux_replay(ptr(logits), ptr(bias), ptr(replay), replay.stride(0) if T else K, T, E,
                                                K, n_group, topk_group, int(norm), float(scaling), ptr(o["rw"]),
                                                ptr(o["tw"]), ptr(o["ids"]), ptr(o["ids32"]), ptr(o["tpe"]),
                                                current_stream()), "noaux_replay")
    return o


@pytest.mark.parametrize("E,K,n_group,topk_group", [(256, 8, 8, 4), (256, 8, 8, 8), (64, 6, 4, 2), (512, 8, 16, 16)])
def test_noaux_replay_own_ids_bit_for_bit_and_random_ids_against_float64(E, K, n_group, topk_group):
    from xtuner_b200.router import noaux_group_spec

    g = torch.Generator().manual_seed(E + K + n_group)
    for T in (1, 37, 777):
        logits = torch.randn(T, E, generator=g).to(DEV)
        bias = (torch.randn(E, generator=g) * 0.1).to(DEV)
        a = noaux_route(logits, bias, K, n_group, topk_group, True, 2.5)
        _same(a, noaux_replay(logits, bias, a["ids"].clone(), n_group, topk_group, True, 2.5), f"T={T}")
        ids = _rand_ids(T, E, K, g)
        o = noaux_replay(logits, bias, ids, n_group, topk_group, True, 2.5)
        assert torch.equal(o["ids"], ids) and torch.equal(o["rw"], a["rw"])
        assert torch.equal(o["tpe"].cpu(), torch.bincount(ids.flatten().cpu(), minlength=E).float())
        r64, w64 = noaux_replay_ref(logits.cpu(), bias.cpu(), ids.cpu(), K, n_group, topk_group, True, 2.5)
        u = 2.0 ** -24
        check_bound(o["tw"].cpu(), w64, (4 * K + 8) * u * w64.abs() + 1e-30, "topk_weights")
        # backward through the existing entry
        g_tw = torch.randn(T, K, generator=g).to(DEV)
        g_rw = torch.randn(T, E, generator=g).to(DEV)
        gl = torch.empty(T, E, device=DEV)
        check(ensure_init().xtb_router_noaux_bwd(ptr(logits), ptr(bias), ptr(o["rw"]), ptr(o["tw"]), ptr(o["ids"]),
                                                 ptr(g_tw), ptr(g_rw), T, E, K, noaux_group_spec(n_group, topk_group),
                                                 1, 2.5, ptr(gl), current_stream()), "noaux_bwd")
        lg = logits.cpu().double().requires_grad_(True)
        r, w = noaux_replay_ref(lg, bias.cpu(), ids.cpu(), K, n_group, topk_group, True, 2.5)
        (w * g_tw.cpu().double()).sum().add((r * g_rw.cpu().double()).sum()).backward()
        scale = lg.grad.abs().amax(1, keepdim=True) + 2.5 * g_tw.abs().amax().item() + g_rw.abs().amax().item() + 1
        check_bound(gl.cpu(), lg.grad, (256 + 2 * E) * u * scale, "grad_logits")


# ---- host layers -------------------------------------------------------------------------------------------------------


def test_router_modules_replay_and_opcheck():
    from xtuner_b200 import router

    g = torch.Generator().manual_seed(5)
    T, E, K = 96, 128, 8
    logits = torch.randn(T, E, generator=g).to(DEV)
    full = torch.randint(0, E, (T, 3, K), generator=g).to(DEV)
    r = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=1.5)
    res = r(logits, full[:, 1, :])
    assert torch.equal(res["topk_ids"], full[:, 1, :]) and torch.equal(r.last_topk_ids_i32, full[:, 1, :].int())
    with pytest.raises(TypeError):
        r(logits, full[:, 1, :].int())
    n = router.NoAuxRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=2.5, scoring_func="sigmoid",
                           n_group=8, topk_group=4).to(DEV)
    res = n(logits, full[:, 2, :])
    assert torch.equal(res["topk_ids"], full[:, 2, :])
    ids = full[:, 0, :].contiguous()
    torch.library.opcheck(router._router_greedy_replay_op, (logits, ids, K, 0, True, 1.5))
    torch.library.opcheck(router._router_noaux_replay_op, (logits, torch.zeros(E, device=DEV), ids, K, 8, 4, True, 2.5))
    torch.library.opcheck(router._router_greedy_replay_op, (logits, full[:, 1, :], K, 1, False, 1.0))  # strided ids


def _block_inputs(T, H, I, E, seed):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(T, H, generator=g).to(torch.bfloat16).to(DEV)
    nw = (1 + 0.1 * torch.randn(H, generator=g)).to(DEV)
    gw = (torch.randn(E, H, generator=g) * 0.05).to(DEV)
    w13 = (torch.randn(E, 2 * I, H, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    w2 = (torch.randn(E, H, I, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    return h, nw, gw, w13, w2


def _grad_out(inputs, seed=9):
    return torch.randn(inputs[0].shape, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16).to(DEV)


def _run_block(inputs, K, replay=None, go=None):
    from xtuner_b200 import fused

    ps = [t.clone().requires_grad_(True) for t in inputs]
    out, rr = fused.fused_moe_block(ps[0], ps[1], 1e-6, ps[2], ps[3], ps[4], top_k=K, rollout_routed_experts=replay)
    go = _grad_out(inputs) if go is None else go
    (out.float() * go.float()).sum().add(rr["router_weights"].square().sum() * 0.1).backward()
    return out.detach(), rr, [p.grad for p in ps]


@pytest.mark.parametrize("T,H,I,E,K", [(512, 2048, 256, 8, 2), (300, 1024, 256, 16, 4)])
def test_fused_block_replay(T, H, I, E, K):
    inputs = _block_inputs(T, H, I, E, T + E)
    out, rr, grads = _run_block(inputs, K)
    full = torch.stack([rr["topk_ids"], rr["topk_ids"]], 1)
    out2, rr2, grads2 = _run_block(inputs, K, full[:, 0, :])
    assert torch.equal(out, out2) and torch.equal(rr["topk_ids"], rr2["topk_ids"])
    assert torch.equal(rr["router_weights"], rr2["router_weights"]) and torch.equal(rr["logits"], rr2["logits"])
    for a, b in zip(grads, grads2):
        assert torch.equal(a, b)
    # random ids: the fused node against the per-op composition (rms_norm -> gate -> router -> experts -> combine)
    ids = _rand_ids(T, E, K, torch.Generator().manual_seed(1))
    out3, rr3, _ = _run_block(inputs, K, ids)
    assert torch.equal(rr3["topk_ids"], ids)
    from xtuner_b200 import router

    h, nw, gw, w13, w2 = inputs
    x = torch.nn.functional.rms_norm(h.float(), (H,), nw, 1e-6).to(torch.bfloat16)
    logits = x.float() @ gw.t()
    res = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K)(logits, ids)
    ref = torch.zeros(T, H, device=DEV)
    for e in range(E):
        tok, slot = (res["topk_ids"] == e).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        hh = x[tok].float() @ w13[e].float().t()
        a = (torch.nn.functional.silu(hh[:, :I]) * hh[:, I:]).to(torch.bfloat16).float()
        y = (a @ w2[e].float().t()).to(torch.bfloat16).float()
        ref.index_add_(0, tok, y * res["topk_weights"][tok, slot].unsqueeze(1))
    ref = ref + h.float()
    # the composition rounds the norm and the gate its own way: near-tie bf16 roundings differ on a few elements
    err = (out3.float() - ref).abs()
    assert float(err.max()) < 0.25
    assert float((err > 3e-2 * (ref.abs() + ref.abs().mean())).float().mean()) < 5e-3


def test_fused_block_replay_in_a_cuda_graph():
    T, H, I, E, K = 256, 1024, 256, 8, 2
    inputs = _block_inputs(T, H, I, E, 4)
    ids = _rand_ids(T, E, K, torch.Generator().manual_seed(2))
    go = _grad_out(inputs)
    want_out, _, want_g = _run_block(inputs, K, ids, go)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run_block(inputs, K, ids, go)  # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, _, grads = _run_block(inputs, K, ids, go)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want_out)
    for a, b in zip(grads, want_g):
        assert torch.equal(a, b)


# ---- the fixture made by the reference's own routers -------------------------------------------------------------------

from tests.test_router_replay_cpu import PATTERNS, fixture_case_names, fixture_config, fixture_ids  # noqa: E402

W_TOL = dict(rtol=1e-5, atol=1e-6)  # fp32 weights: expf vs torch's softmax / sigmoid differ by a few ulps
G_TOL = dict(rtol=1e-4, atol=2e-6)  # the logits gradient, as the routing fixtures hold it


@pytest.fixture(scope="module")
def gold():
    from tests.conftest import load_golden

    return load_golden("router_replay")


@pytest.mark.parametrize("case", fixture_case_names())
def test_fixture_cases_match_the_reference(gold, case):
    from xtuner_b200 import router

    kind, E, K, a, b, scaling = fixture_config(case)
    if kind == "greedy":
        r = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K, norm_topk_prob=b, scoring_func=a,
                                router_scaling_factor=scaling)
    else:
        r = router.NoAuxRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=scaling,
                               scoring_func="sigmoid", n_group=a, topk_group=b).to(DEV)
        r.e_score_correction_bias = gold[f"{case}.bias"].to(DEV)
    for pat in PATTERNS:
        ids = gold[f"{case}.slice.full"].to(DEV)[:, 1, :] if pat == "slice" else fixture_ids(gold, case, pat).to(DEV)
        lg = gold[f"{case}.logits"].to(DEV).requires_grad_(True)
        res = r(lg, ids)
        assert torch.equal(res["topk_ids"], ids) and torch.equal(r.last_topk_ids_i32, ids.int()), pat
        assert torch.equal(res["topkens_per_expert"].cpu().double(), gold[f"{case}.{pat}.tokens_per_expert"].double()), pat
        torch.testing.assert_close(res["router_weights"].cpu(), gold[f"{case}.router_weights"], **W_TOL)
        torch.testing.assert_close(res["topk_weights"].cpu(), gold[f"{case}.{pat}.topk_weights"], **W_TOL)
        ((res["topk_weights"] * gold[f"{case}.{pat}.g_tw"].to(DEV)).sum()
         + (res["router_weights"] * gold[f"{case}.g_rw"].to(DEV)).sum()).backward()
        torch.testing.assert_close(lg.grad.cpu(), gold[f"{case}.{pat}.grad_logits"], **G_TOL)
