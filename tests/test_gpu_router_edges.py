"""The gate and router kernels (csrc/route.cu, csrc/gate_mma.cu) against the float64 references and exact restatements
of tests/router_reference.py, at the edges the parity tests of tests/test_gpu_router.py do not reach.

* Gate forward: xtb_gate_logits at every kernel it selects (small <8,4> at E = 1, 3, 8, <16,2> at E = 9, 16; strided
  at E = 17, 40, 64 and at H not a multiple of 256; the 200 KiB shared-memory boundary E = 8, H = 6400 against 6656),
  and the logits of xtb_gate_route_dispatch (tensor cores) at E = 1 to 8, H = 128 to 4224, in exact, one-hot and random
  modes, with T tails around 16, 32 and 64.  Exact and one-hot modes bit for bit; random within the kernel's bound.
* Greedy router: every XTB_ROUTER_DISPATCH instantiation (E = 1 to 512), K = 1 to min(E, 8), softmax and sigmoid,
  normalising on and off, scaling 1 and 2.5, with and without the dispatch workspace (chunk histograms and
  expert_start against a CPU scan).  Exact checks on the kernel's own router_weights, router_weights within the expf
  bound, ids equal to float64 on decided rows.  Tie rows, rows of tied zeros, NaN and +-inf rows.  Refusals.
* Fused gate + route + dispatch bit-equal to xtb_router_greedy_dispatch on its own logits, and the rows
  xtb_moe_permute_prepared gathers from either workspace bit-equal, at E = 1 to 8, K = 1 to E and at the benchmark
  shape (T = 8192, H = 2048, E = 8, K = 2), and on logits with tie, NaN, partial-NaN and +-inf rows at E = 4 and 8.
* Backward: xtb_router_greedy_bwd against float64 autograd with every null combination of the three gradients;
  xtb_router_gate_bwd bit-equal to the two calls it replaces at E = 1 to 8, K = 1 to E and at the benchmark shape,
  with every null combination of the three gradients; the
  gate backward (both small kernels, the strided pair, colsum) against float64 on both sides of 768 tokens per block.
* No-aux router: E = 32 to 512, K up to 32, lanes per group 1 to 8, no mask, tied group scores, negative-bias kept
  experts against masked zeros, the zero-score kept expert's gradient, whole groups with a -inf bias (fewer than
  topk_group groups above -inf: exactly topk_group are still kept, routed and replayed), NaN rows, refusals.
* Determinism and T = 0.

Outputs go to views with 16 NaN-filled guard rows on each side; the guards must stay as they were."""
import pytest
import torch

from tests import router_reference as R
from tests.gpu_harness import Guarded, Worst
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu

WORST = Worst("router_edges")
_report = WORST.fixture()


# ---- entries ---------------------------------------------------------------------------------------------------------


def gate_logits(x, w, b):
    T, H = x.shape
    E = w.shape[0]
    out = Guarded(T, E, torch.float32)
    check(ensure_init().xtb_gate_logits(ptr(x), ptr(w), ptr(b), ptr(out.v), T, H, E, current_stream()),
          "xtb_gate_logits")
    return out.check("logits")


def router(logits, K, scoring, norm, scaling, ws=False):
    T, E = logits.shape
    rw, tw = Guarded(T, E, torch.float32), Guarded(T, K, torch.float32)
    ids, i32 = Guarded(T, K, torch.int64), Guarded(T, K, torch.int32)
    tpe = torch.full((E,), -1, dtype=torch.int64, device="cuda")
    lib = ensure_init()
    sc = 1 if scoring == "sigmoid" else 0
    if ws:
        w = torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8, device="cuda")
        check(lib.xtb_router_greedy_dispatch(ptr(logits), T, E, K, sc, int(norm), scaling, ptr(rw.v), ptr(tw.v),
                                             ptr(ids.v), ptr(i32.v), ptr(tpe), ptr(w), current_stream()),
              "xtb_router_greedy_dispatch")
    else:
        w = None
        check(lib.xtb_router_greedy(ptr(logits), T, E, K, sc, int(norm), scaling, ptr(rw.v), ptr(tw.v), ptr(ids.v),
                                    ptr(i32.v), ptr(tpe), current_stream()), "xtb_router_greedy")
    out = dict(rw=rw.check("router_weights"), tw=tw.check("topk_weights"), ids=ids.check("topk_ids"),
               i32=i32.check("topk_ids_i32"), tpe=tpe, ws=w)
    assert torch.equal(out["i32"].long(), out["ids"])
    return out


def check_workspace(ws, ids, E):
    """chunk histograms (after the scan: exclusive prefixes over chunks) and expert_start against a CPU scan."""
    T, K = ids.shape
    nc = (T + 31) // 32
    off = 256 + ((E * 4 + 255) // 256) * 256
    es = ws[256 : 256 + 4 * E].view(torch.int32).cpu().long()
    counts = ws[off : off + 4 * nc * E].view(torch.int32).view(nc, E).cpu().long()
    ic = ids.cpu()
    hist = torch.zeros(nc, E, dtype=torch.int64)
    hist.index_put_((torch.arange(T).repeat_interleave(K) // 32, ic.reshape(-1)), torch.ones(T * K, dtype=torch.int64),
                    accumulate=True)
    want_counts = torch.cumsum(hist, 0) - hist
    tot = hist.sum(0)
    assert torch.equal(counts, want_counts), "chunk histogram scan"
    assert torch.equal(es, torch.cumsum(tot, 0) - tot), "expert_start"


# ---- gate forward ----------------------------------------------------------------------------------------------------

GATE_SHAPES = [(256, 1), (256, 3), (512, 8), (768, 9), (256, 16), (320, 8), (320, 17), (2048, 40), (256, 64),
               (6400, 8), (6656, 8)]


@pytest.mark.parametrize("mode", ["exact", "onehot", "random"])
@pytest.mark.parametrize("H,E", GATE_SHAPES)
def test_gate_logits(mode, H, E):
    kernel = R.gate_kernel(0, H, E)
    assert (H, E) != (6400, 8) or kernel == "small"
    assert (H, E) != (6656, 8) or kernel == "strided"
    Ts = [H + 17] if mode == "onehot" else [1, 15, 16, 17, 33, 63, 64, 65, 1000]
    for i, T in enumerate(Ts):
        x, w, b = R.gate_inputs(T, H, E, mode, 100 * H + E + i, "cuda", with_bias=(mode != "onehot") and i % 2 == 0)
        got = gate_logits(x, w, b)
        ref, S = R.gate_ref(x, w, b)
        if mode == "random":
            WORST.note(f"gate logits ({kernel})", R.check_bound(got, ref, R.gate_bound(kernel, H, S),
                                                                f"{kernel} T={T}"))
        else:
            assert torch.equal(got.double(), ref), f"{mode} {kernel} T={T}: not exact"


def fused(x, w, K, scoring, norm, scaling):
    T, H = x.shape
    E = w.shape[0]
    lib = ensure_init()
    lg, rw, tw = Guarded(T, E, torch.float32), Guarded(T, E, torch.float32), Guarded(T, K, torch.float32)
    ids, i32 = Guarded(T, K, torch.int64), Guarded(T, K, torch.int32)
    tpe = torch.full((E,), -1, dtype=torch.int64, device="cuda")
    ws = torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8, device="cuda")
    rc = lib.xtb_gate_route_dispatch(ptr(x), ptr(w), T, H, E, K, 1 if scoring == "sigmoid" else 0, int(norm), scaling,
                                     ptr(lg.v), ptr(rw.v), ptr(tw.v), ptr(ids.v), ptr(i32.v), ptr(tpe), ptr(ws),
                                     current_stream())
    check(rc, "xtb_gate_route_dispatch")
    return dict(logits=lg.check("fused logits"), rw=rw.check("fused rw"), tw=tw.check("fused tw"),
                ids=ids.check("fused ids"), i32=i32.check("fused i32"), tpe=tpe, ws=ws)


@pytest.mark.parametrize("mode", ["exact", "onehot", "random"])
@pytest.mark.parametrize("H", [128, 384, 2048, 4096, 4224])
def test_fused_gate_logits(mode, H):
    for E in range(1, 9):
        T = H + 17 if mode == "onehot" else (16, 31, 33, 64, 65, 1000)[E % 6]
        x, w, _ = R.gate_inputs(T, H, E, mode, 7 * H + E, "cuda", with_bias=False)
        out = fused(x, w, 1, "softmax", True, 1.0)
        ref, S = R.gate_ref(x, w, None)
        if mode == "random":
            WORST.note("gate logits (mma)", R.check_bound(out["logits"], ref, R.gate_bound("mma", H, S), f"E={E}"))
        else:
            assert torch.equal(out["logits"].double(), ref), f"{mode} H={H} E={E}: not exact"


def test_fused_gate_refuses_h_4352_and_accepts_4224():
    from xtuner_b200._capi import XtbError

    x, w, _ = R.gate_inputs(40, 4352, 8, "random", 1, "cuda")
    with pytest.raises(XtbError, match="H <= 4224"):
        fused(x, w, 2, "softmax", True, 1.0)
    x, w, _ = R.gate_inputs(40, 4224, 8, "random", 1, "cuda")
    fused(x, w, 2, "softmax", True, 1.0)


def permute_prepared(x, ids32, ws, E):
    """(permuted rows as int32 words, row_id_map) of xtb_moe_permute_prepared against a prepared workspace."""
    T, H = x.shape
    K = ids32.shape[1]
    perm, rmap = Guarded(T * K, H // 2, torch.int32), Guarded(T, K, torch.int32)
    check(ensure_init().xtb_moe_permute_prepared(ptr(x), ptr(ids32), T, K, E, H * 2, ptr(perm.v), ptr(rmap.v), None,
                                                 ptr(ws), current_stream()), "xtb_moe_permute_prepared")
    return perm.check("permuted"), rmap.check("row_id_map")


def _edge_gate_inputs(T, H, E):
    """Two gate inputs (x, w) and (x, w') whose logits hold the router's edge rows.  The tensor-core gate splits the fp32
    weight into three bf16 planes: powers of two leave the lower two planes zero, and w' = w but inf at experts 1 and 3
    of column 0, which leaves inf - inf = NaN in them, so those two logits are NaN in every row of w'.  Row 0 of x is
    zero (tied zeros), row 1 holds a NaN (a NaN row), rows 2 and 3 overflow to -inf and +inf at experts E-2 and E-1 and
    the other way round, and row 4 has logits 3 and 2 at experts 0 and 2: [3, nan, 2, nan] under w' at E = 4."""
    x, w, _ = R.gate_inputs(T, H, E, "random", E, "cuda")
    x[:5] = 0
    x[:, 1] = 0
    x[1, 5] = float("nan")
    x[2, 1], x[3, 1] = 2.0 ** 100, -(2.0 ** 100)
    x[4, 2] = 1
    w[:, 1] = 0
    w[E - 2, 1], w[E - 1, 1] = -(2.0 ** 100), 2.0 ** 100
    w[0, 2], w[2, 2] = 3, 2
    w_nan = w.clone()
    w_nan[[1, 3], 0] = float("inf")
    return [(x, w), (x, w_nan)]


@pytest.mark.parametrize("E,T,H,Ks,edges", [
    pytest.param(E, 1000, 256, range(1, E + 1), False, id=str(E)) for E in range(1, 9)] + [
    pytest.param(8, 8192, 2048, (2,), False, id="bench")] + [
    pytest.param(E, 1000, 256, range(1, E + 1), True, id=f"edges{E}") for E in (4, 8)])
def test_fused_gate_route_equals_router_on_its_own_logits(E, T, H, Ks, edges):
    inputs = _edge_gate_inputs(T, H, E) if edges else [R.gate_inputs(T, H, E, "random", E, "cuda")[:2]]
    for i, (x, w) in enumerate(inputs):
        for K in Ks:
            for scoring, norm, scaling in [("softmax", True, 1.0), ("sigmoid", False, 2.5), ("softmax", False, 2.5)]:
                what = (i, K, scoring)
                f = fused(x, w, K, scoring, norm, scaling)
                r = router(f["logits"].clone(), K, scoring, norm, scaling, ws=True)
                for k in ("rw", "tw", "ids", "i32", "tpe", "ws"):
                    assert torch.equal(f[k].view(torch.uint8) if f[k].dtype == torch.float32 else f[k],
                                       r[k].view(torch.uint8) if r[k].dtype == torch.float32 else r[k]), (*what, k)
                (pf, mf), (pr, mr) = permute_prepared(x, f["i32"], f["ws"], E), permute_prepared(x, r["i32"], r["ws"], E)
                assert torch.equal(mf, mr) and torch.equal(pf, pr), (*what, "permuted rows")
                if edges and i == 1 and E == 4 and K == 3 and scoring == "sigmoid":
                    # NaN at experts 1 and 3: the third pick falls back to the lowest id not selected yet
                    assert f["ids"][4].tolist() == [0, 2, 1], f["ids"][4].tolist()


# ---- greedy router ---------------------------------------------------------------------------------------------------

ROUTER_E = [1, 2, 3, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256, 257, 384, 512]


def _edge_logits(T, E, seed):
    """N(0, 3) rows, with edge rows: all equal, duplicates straddling the K boundary and lanes (7 and 8, 0 and E-1),
    spreads that underflow all but a few softmax weights to exactly 0."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lg = torch.randn(T, E, generator=g, device="cuda") * 3
    if E >= 2:
        lg[0] = 0.5
        lg[1, :] = -1.0
        lg[1, [0, E - 1]] = 30.0
        lg[2] = torch.arange(E, device="cuda").float() * -200.0  # softmax: one weight 1, the rest exactly 0 (tied)
        lg[3, :] = -300.0
        lg[3, E // 2] = 0.0
    if E >= 9:
        lg[4, :] = -1.0
        lg[4, 7] = lg[4, 8] = 30.0
        lg[5, :4] = 40.0  # duplicates straddling every K <= 4 boundary
    return lg


@pytest.mark.parametrize("E", ROUTER_E)
def test_greedy_router(E):
    T = 300
    lg = _edge_logits(T, E, E)
    for K in sorted({1, min(E, 2), min(E, 3), min(E, 8)}):
        for scoring in ("softmax", "sigmoid"):
            p64, bound = R.greedy_ref(lg, scoring)
            for norm, scaling, ws in [(True, 1.0, False), (False, 2.5, True), (True, 2.5, False), (False, 1.0, True)]:
                r = router(lg, K, scoring, norm, scaling, ws)
                what = f"E={E} K={K} {scoring} norm={norm} scaling={scaling} ws={ws}"
                R.check_greedy_exact(r["rw"], r["tw"], r["ids"], r["tpe"], K, norm, scaling, what)
                WORST.note(f"router_weights ({scoring})", R.check_bound(r["rw"], p64, bound, what))
                dec = R.decided_rows(p64, bound, K)
                assert torch.equal(r["ids"][dec], R.topk_rounds(p64, K)[dec]), what
                if ws:
                    check_workspace(r["ws"], r["ids"], E)


@pytest.mark.parametrize("E", [2, 8, 9, 64, 257, 512])
def test_greedy_router_nan_and_inf_rows(E):
    T = 64
    lg = torch.randn(T, E, device="cuda")
    lg[0] = float("nan")
    lg[1, ::2] = float("nan")
    lg[2, 0] = float("inf")
    lg[3] = float("-inf")
    lg[4, 1:] = float("nan")
    lg[5, E - 1] = float("-inf")
    for K in sorted({1, min(E, 2), min(E, 8)}):
        for scoring in ("softmax", "sigmoid"):
            for ws in (False, True):
                r = router(lg, K, scoring, True, 1.0, ws)
                ids = r["ids"]
                assert bool(((ids >= 0) & (ids < E)).all()), (K, scoring)
                srt = ids.sort(-1).values
                assert bool((srt[:, 1:] != srt[:, :-1]).all()), (K, scoring, ids[:6].tolist())
                assert int(r["tpe"].sum()) == T * K
                assert torch.equal(r["tpe"], torch.bincount(ids.reshape(-1), minlength=E))


def test_greedy_router_refusals_and_empty():
    from xtuner_b200._capi import XtbError

    lib = ensure_init()
    for E, K in [(513, 2), (16, 9), (4, 5)]:
        lg = torch.zeros(4, E, device="cuda")
        with pytest.raises(XtbError):
            router(lg, K, "softmax", True, 1.0)
    tpe = torch.full((8,), -1, dtype=torch.int64, device="cuda")
    d = torch.empty(1, device="cuda")
    check(lib.xtb_router_greedy(ptr(d), 0, 8, 2, 0, 1, 1.0, ptr(d), ptr(d), ptr(d), None, ptr(tpe), current_stream()))
    assert bool((tpe == 0).all())


# ---- backward --------------------------------------------------------------------------------------------------------


def greedy_bwd(r, K, scoring, norm, scaling, g_tw, g_rw, g_dir):
    T, E = r["rw"].shape
    gl = Guarded(T, E, torch.float32)
    check(ensure_init().xtb_router_greedy_bwd(ptr(r["rw"]), ptr(r["tw"]), ptr(r["ids"]), ptr(g_tw), ptr(g_rw),
                                              ptr(g_dir), T, E, K, 1 if scoring == "sigmoid" else 0, int(norm), scaling,
                                              ptr(gl.v), current_stream()))
    return gl.check("grad_logits")


@pytest.mark.parametrize("E", [3, 8, 16, 33, 128, 257, 512])
def test_greedy_router_bwd(E):
    T = 256
    g = torch.Generator(device="cuda").manual_seed(E)
    lg = torch.randn(T, E, generator=g, device="cuda") * 2
    for K in sorted({1, min(E, 3), min(E, 8)}):
        for scoring, norm, scaling in [("softmax", True, 1.0), ("sigmoid", True, 2.5), ("softmax", False, 2.5)]:
            r = router(lg, K, scoring, norm, scaling)
            p64, pb = R.greedy_ref(lg, scoring)
            dec = R.decided_rows(p64, pb, K)
            for mask in range(8):
                g_tw = torch.randn(T, K, generator=g, device="cuda") if mask & 1 else None
                g_rw = torch.randn(T, E, generator=g, device="cuda") if mask & 2 else None
                g_dir = torch.randn(T, E, generator=g, device="cuda") if mask & 4 else None
                got = greedy_bwd(r, K, scoring, norm, scaling, g_tw, g_rw, g_dir)
                ref, ref_ids = R.greedy_bwd_ref(lg, K, scoring, norm, scaling, g_tw, g_rw, g_dir)
                d = dec & (r["ids"] == ref_ids).all(-1)
                bound = R.greedy_bwd_bound(p64, K, g_tw, g_rw, g_dir, scaling, norm)
                WORST.note("grad_logits (greedy)", R.check_bound(got[d], ref[d], bound[d], f"E={E} K={K} mask={mask}"))


@pytest.mark.parametrize("E,T,H,Ks", [pytest.param(E, 1500, 256, range(1, E + 1), id=str(E)) for E in range(1, 9)] + [
    pytest.param(8, 8192, 2048, (2,), id="bench")])
def test_router_gate_bwd_equals_the_two_calls(E, T, H, Ks):
    lib = ensure_init()
    x, w, _ = R.gate_inputs(T, H, E, "random", E, "cuda")
    lg = torch.randn(T, E, device="cuda")
    for K in Ks:
        scoring, norm, scaling = [("softmax", True, 1.0), ("sigmoid", False, 2.5)][K % 2]
        r = router(lg, K, scoring, norm, scaling)
        sc = 1 if scoring == "sigmoid" else 0
        ws = torch.empty(int(lib.xtb_gate_logits_bwd_workspace_bytes(T, H, E)), dtype=torch.uint8, device="cuda")
        for mask in range(8):
            g_tw = torch.randn(T, K, device="cuda") if mask & 1 else None
            g_rw = torch.randn(T, E, device="cuda") if mask & 2 else None
            g_dir = torch.randn(T, E, device="cuda") if mask & 4 else None
            gw1, gx1 = torch.empty(E, H, device="cuda"), torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
            check(lib.xtb_router_gate_bwd(ptr(r["rw"]), ptr(r["tw"]), ptr(r["ids"]), ptr(g_tw), ptr(g_rw), ptr(g_dir),
                                          ptr(x), ptr(w), ptr(gw1), ptr(gx1), T, H, E, K, sc, int(norm), scaling,
                                          ptr(ws), current_stream()))
            gl = greedy_bwd(r, K, scoring, norm, scaling, g_tw, g_rw, g_dir)
            gw2, gx2 = torch.empty(E, H, device="cuda"), torch.empty(T, H, dtype=torch.bfloat16, device="cuda")
            check(lib.xtb_gate_logits_bwd(ptr(gl), ptr(x), ptr(w), ptr(gw2), ptr(gx2), None, T, H, E, ptr(ws),
                                          current_stream()))
            assert torch.equal(gw1.view(torch.int32), gw2.view(torch.int32)), (K, mask)
            assert torch.equal(gx1.view(torch.int16), gx2.view(torch.int16)), (K, mask)


@pytest.mark.parametrize("T", [1, 700, 20000, 250_000])
@pytest.mark.parametrize("E", [3, 8, 16, 40])
def test_gate_bwd(T, E):
    """grad_w and grad_bias within gamma(depth) of float64; grad_x a correctly rounded bf16 of its float64 value or a
    near-midpoint flip.  T = 250000 has more than 768 tokens per block on 132 SMs."""
    from tests import norm_combine_reference as NC

    lib = ensure_init()
    H = 256 if E <= 16 else 320
    g = torch.Generator(device="cuda").manual_seed(T + E)
    x = torch.randn(T, H, generator=g, device="cuda").to(torch.bfloat16)
    w = torch.randn(E, H, generator=g, device="cuda") * 0.05
    gl = torch.randn(T, E, generator=g, device="cuda")
    ws = torch.empty(int(lib.xtb_gate_logits_bwd_workspace_bytes(T, H, E)), dtype=torch.uint8, device="cuda")
    gw, gb, gx = Guarded(E, H, torch.float32), Guarded(1, E, torch.float32), Guarded(T, H, torch.bfloat16)
    check(lib.xtb_gate_logits_bwd(ptr(gl), ptr(x), ptr(w), ptr(gw.v), ptr(gx.v), ptr(gb.v), T, H, E, ptr(ws),
                                  current_stream()))
    gxv = gx.check("grad_x", written=None)
    gld, xd = gl.double(), x.double()
    gw_ref, gw_S = gld.T @ xd, gld.abs().T @ xd.abs()
    depth = T + 64 if E > 16 else -(-T // 132) + 8 + 512
    WORST.note("grad_w (gate)", R.check_bound(gw.check("grad_w"), gw_ref, R.gamma(depth) * gw_S, f"T={T} E={E}"))
    gb_ref, gb_S = gld.sum(0), gld.abs().sum(0)
    WORST.note("grad_bias", R.check_bound(gb.check("grad_bias")[0], gb_ref, R.gamma(T // 256 + 17) * gb_S, "grad_bias"))
    gx_ref, gx_S = gld @ w.double(), gld.abs() @ w.double().abs()
    r, _ = NC.check_near_tie(gxv, gx_ref, R.gamma(E + 2) * gx_S, f"grad_x T={T} E={E}")
    WORST.note("grad_x past-midpoint / bound", r)


# ---- no-aux router ---------------------------------------------------------------------------------------------------


def noaux(lg, bias, K, NG, TG, norm=True, scaling=2.5):
    T, E = lg.shape
    rw, tw = Guarded(T, E, torch.float32), Guarded(T, K, torch.float32)
    ids, i32 = Guarded(T, K, torch.int64), Guarded(T, K, torch.int32)
    tpe = torch.full((E,), -1.0, device="cuda")
    check(ensure_init().xtb_router_noaux(ptr(lg), ptr(bias), T, E, K, NG, TG, int(norm), scaling, ptr(rw.v), ptr(tw.v),
                                         ptr(ids.v), ptr(i32.v), ptr(tpe), current_stream()), "xtb_router_noaux")
    return dict(rw=rw.check("noaux rw"), tw=tw.check("noaux tw"), ids=ids.check("noaux ids"), i32=i32.check("i32"),
                tpe=tpe)


def noaux_bwd(lg, bias, r, K, NG, TG, g_tw, g_rw, norm=True, scaling=2.5, group_spec=None):
    from xtuner_b200.router import noaux_group_spec

    T, E = lg.shape
    gl = Guarded(T, E, torch.float32)
    spec = noaux_group_spec(NG, TG) if group_spec is None else group_spec
    check(ensure_init().xtb_router_noaux_bwd(ptr(lg), ptr(bias), ptr(r["rw"]), ptr(r["tw"]), ptr(r["ids"]), ptr(g_tw),
                                             ptr(g_rw), T, E, K, spec, int(norm), scaling, ptr(gl.v), current_stream()),
          "xtb_router_noaux_bwd")
    return gl.check("noaux grad_logits")


# (E, n_group, topk_group): lanes per group E / n_group / (E / 32) = 1, 2, 4, 8; no mask
NOAUX = [(32, 8, 3), (64, 8, 4), (128, 4, 2), (256, 8, 4), (512, 32, 6), (512, 16, 4), (256, 4, 2), (64, 2, 2),
         (128, 1, 1), (512, 8, 8)]


@pytest.mark.parametrize("E,NG,TG", NOAUX)
def test_noaux_router(E, NG, TG):
    T = 200
    g = torch.Generator(device="cuda").manual_seed(E + NG)
    lg = torch.randn(T, E, generator=g, device="cuda")
    bias = (torch.randn(E // NG, generator=g, device="cuda") * 0.1).repeat(NG)  # the same pattern in every group
    lg[0] = 0.0  # every group score ties
    lg[1, : E // 2] = lg[1, E // 2 :]
    lg[2] = -8.0  # a kept group's negative-bias experts against masked zeros
    bias_neg = bias.clone()
    for K in sorted({1, 8, min(32, E // NG * TG)}):
        for b in (bias, bias_neg - 0.2):
            r = noaux(lg, b, K, NG, TG)
            ids64, kept, masked = R.noaux_ref(lg, b, K, NG, TG)
            s64 = torch.sigmoid(lg.double())
            bound = 8 * R.U32 * (s64 + b.double().abs())
            dec = R.decided_rows(masked, bound, K)
            assert torch.equal(r["ids"][dec], ids64[dec]), (K, (~dec).sum())
            assert torch.equal(r["i32"].long(), r["ids"])
            assert torch.equal(r["tpe"], torch.bincount(r["ids"].reshape(-1), minlength=E).float())
            # each kept choice score carries the sigmoid's 6u and the bias add's u; the row sum adds gamma(E)
            S64 = masked.sum(-1, keepdim=True)
            rw64 = masked / S64
            ec = torch.where(kept, 8 * R.U32 * (s64 + b.double().abs()), torch.zeros_like(s64))
            rb = (ec + rw64.abs() * (ec.sum(-1, keepdim=True) + R.gamma(E + 8) * masked.abs().sum(-1, keepdim=True))) \
                / S64.abs() + 2 * R.U32 * rw64.abs()
            WORST.note("router_weights (noaux)", R.check_bound(r["rw"][dec], rw64[dec], rb[dec] + 1e-30,
                                                               f"E={E} K={K}"))
            # the backward against float64 autograd through the oracle
            g_tw, g_rw = torch.randn(T, K, generator=g, device="cuda"), torch.randn(T, E, generator=g, device="cuda")
            got = noaux_bwd(lg, b, r, K, NG, TG, g_tw, g_rw)
            ref = _noaux_autograd(lg, b, K, NG, TG, g_tw, g_rw, r["ids"])
            gb = _noaux_bwd_bound(lg, masked, r["ids"], K, g_tw, g_rw, ref)
            WORST.note("grad_logits (noaux)", R.check_bound(got[dec], ref[dec], gb[dec], f"noaux bwd E={E} K={K}"))


def _noaux_bwd_bound(lg, c, ids, K, g_tw, g_rw, ref):
    """gamma(4E + 64) times the magnitudes of (g - dot) / S (scaled by the conditioning sum |c| / |S| of the row sum)
    and of (scaling g_k - gw) / D, times s (1 - s); plus 8u |ref| for the sigmoid's own error."""
    E = c.shape[1]
    s = torch.sigmoid(lg.double())
    S = c.sum(-1, keepdim=True)
    kappa = c.abs().sum(-1, keepdim=True) / S.abs()
    rw = c / S
    a = kappa * (g_rw.double().abs() + 2 * (g_rw.double().abs() * rw.abs()).sum(-1, keepdim=True)) / S.abs()
    sk = s.gather(1, ids)
    D = sk.sum(-1, keepdim=True)
    tw = 2.5 * sk / D
    gt = g_tw.double().abs()
    b = (2.5 * gt.max(-1, keepdim=True).values + (gt * tw).sum(-1, keepdim=True)) / D
    return R.gamma(4 * E + 64) * (a + b) * s * (1 - s) + 8 * R.U32 * ref.abs() + 1e-30


def _noaux_autograd(lg, bias, K, NG, TG, g_tw, g_rw, ids):
    """float64 autograd through the no-aux router with the given ids and the reference's tie rules."""
    ld = lg.double().clone().requires_grad_(True)
    s = torch.sigmoid(ld)
    ch = s + bias.double()
    from oracle import moe_oracle as O

    kept = O.noaux_kept_experts(ch.detach(), NG, TG)
    c = torch.where(kept, ch, torch.zeros_like(ch))
    rw = c / c.sum(-1, keepdim=True)
    tw = s.gather(1, ids)
    if K > 1:
        tw = tw / (tw.sum(-1, keepdim=True) + 1e-20)
    tw = tw * 2.5
    (gl,) = torch.autograd.grad([tw, rw], ld, [g_tw.double(), g_rw.double()])
    return gl


def test_noaux_zero_score_kept_expert_gradient():
    E, NG, TG, K = 64, 8, 4, 4
    lg = torch.randn(8, E, device="cuda")
    bias = torch.zeros(E, device="cuda")
    lg[:, 0:8] = 4.0
    lg[:, 3] = 0.0
    bias[3] = -0.5
    r = noaux(lg, bias, K, NG, TG)
    assert bool((r["rw"][:, 3] == 0).all())
    g_tw, g_rw = torch.randn(8, K, device="cuda"), torch.randn(8, E, device="cuda")
    got = noaux_bwd(lg, bias, r, K, NG, TG, g_tw, g_rw)
    ref = _noaux_autograd(lg, bias, K, NG, TG, g_tw, g_rw, r["ids"])
    assert bool((ref[:, 3] != 0).all())
    torch.testing.assert_close(got.double(), ref, rtol=1e-4, atol=1e-6)


def noaux_replay(lg, bias, ids, NG, TG, norm=True, scaling=2.5):
    T, E = lg.shape
    K = ids.shape[1]
    rw, tw = Guarded(T, E, torch.float32), Guarded(T, K, torch.float32)
    oids, i32 = Guarded(T, K, torch.int64), Guarded(T, K, torch.int32)
    tpe = torch.full((E,), -1.0, device="cuda")
    check(ensure_init().xtb_router_noaux_replay(ptr(lg), ptr(bias), ptr(ids), ids.stride(0), T, E, K, NG, TG, int(norm),
                                                scaling, ptr(rw.v), ptr(tw.v), ptr(oids.v), ptr(i32.v), ptr(tpe),
                                                current_stream()), "xtb_router_noaux_replay")
    return dict(rw=rw.check("noaux replay rw"), tw=tw.check("noaux replay tw"))


@pytest.mark.parametrize("E,NG,TG,K,finite", [(256, 8, 4, 8, (0, 1)), (256, 8, 4, 8, (6,)), (64, 8, 3, 12, (5,)),
                                              (512, 16, 4, 8, ()), (32, 16, 3, 2, (3, 9))])
def test_noaux_groups_scoring_minus_inf(E, NG, TG, K, finite):
    """Every group but ``finite`` has a -inf bias, so fewer than topk_group groups score above -inf.  The forward still
    keeps exactly topk_group groups: those above -inf, then the lowest-index others (oracle.noaux_kept_experts), as the
    backward does.  A kept -inf group makes the row sum -inf, so router_weights are NaN at its experts and 0 elsewhere;
    replaying the forward's ids gives the same router_weights and topk weights."""
    T = 64
    g = torch.Generator(device="cuda").manual_seed(E + TG + len(finite))
    # distinct logits 6 / E apart in every row: the top-k is decided in fp32 as in float64
    lg = (torch.rand(T, E, generator=g, device="cuda").argsort(-1).float() - E / 2) * (6 / E)
    bias = torch.full((NG, E // NG), -torch.inf, device="cuda")
    bias[list(finite)] = 0.0
    bias = bias.view(E)
    r = noaux(lg, bias, K, NG, TG)
    ids64, kept, masked = R.noaux_ref(lg, bias, K, NG, TG)
    others = [i for i in range(NG) if i not in finite]
    want_groups = torch.zeros(NG, dtype=torch.bool)
    want_groups[list(finite) + others[: TG - len(finite)]] = True
    assert bool((kept.view(T, NG, -1).all(-1).cpu() == want_groups).all())
    assert torch.equal(r["ids"], ids64)
    assert torch.equal(r["tpe"], torch.bincount(r["ids"].reshape(-1), minlength=E).float())
    torch.testing.assert_close(r["rw"].double(), masked / masked.sum(-1, keepdim=True), rtol=0, atol=0, equal_nan=True)
    rp = noaux_replay(lg, bias, r["ids"], NG, TG)
    assert torch.equal(rp["rw"].view(torch.int32), r["rw"].view(torch.int32))
    assert torch.equal(rp["tw"].view(torch.int32), r["tw"].view(torch.int32))


def test_noaux_nan_rows_and_refusals():
    from xtuner_b200._capi import XtbError

    E, K = 256, 8
    lg = torch.randn(16, E, device="cuda")
    lg[0] = float("nan")
    lg[1, :250] = float("nan")
    bias = torch.zeros(E, device="cuda")
    for NG, TG in [(8, 8), (8, 4)]:
        r = noaux(lg, bias, K, NG, TG)
        ids = r["ids"]
        assert bool(((ids >= 0) & (ids < E)).all())
        srt = ids.sort(-1).values
        assert bool((srt[:, 1:] != srt[:, :-1]).all())
        assert int(r["tpe"].sum()) == 16 * K
    # (32, 32, 4): a group mask over groups of one expert, whose second-best score would be -inf in every group
    for E2, K2, NG, TG in [(96, 4, 1, 1), (192, 4, 3, 1), (64, 33, 1, 1), (32, 2, 32, 4)]:
        with pytest.raises(XtbError):
            noaux(torch.zeros(4, E2, device="cuda"), torch.zeros(E2, device="cuda"), K2, NG, TG)
    # the backward refuses a group_spec that is not the forward's geometry (1 was the old "has a group mask" flag)
    r = noaux(lg, bias, K, 8, 4)
    g_rw = torch.randn(16, E, device="cuda")
    for spec in (1, 3 | 2 << 8, 8 | 8 << 8, 8 | 0 << 8):
        with pytest.raises(XtbError):
            noaux_bwd(lg, bias, r, K, 8, 4, None, g_rw, group_spec=spec)
    lg32, b32 = torch.randn(16, 32, device="cuda"), torch.zeros(32, device="cuda")
    r32 = noaux(lg32, b32, 2, 32, 32)  # groups of one expert without a mask are accepted
    with pytest.raises(XtbError):
        noaux_bwd(lg32, b32, r32, 2, 32, 4, None, torch.randn(16, 32, device="cuda"), group_spec=32 | 4 << 8)


# ---- general ---------------------------------------------------------------------------------------------------------


def test_determinism_and_empty_inputs():
    lib = ensure_init()
    x, w, b = R.gate_inputs(5000, 2048, 8, "random", 5, "cuda")
    a1, a2 = fused(x, w, 2, "softmax", True, 1.0), fused(x, w, 2, "softmax", True, 1.0)
    for k in a1:
        assert torch.equal(a1[k], a2[k]), k
    assert torch.equal(gate_logits(x, w, b), gate_logits(x, w, b))
    d = torch.empty(16, device="cuda")
    tpe = torch.full((8,), -1, dtype=torch.int64, device="cuda")
    ws = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    check(lib.xtb_gate_logits(ptr(d), ptr(w), None, ptr(d), 0, 2048, 8, current_stream()))
    check(lib.xtb_gate_route_dispatch(ptr(d), ptr(w), 0, 2048, 8, 2, 0, 1, 1.0, ptr(d), ptr(d), ptr(d), ptr(d), ptr(d),
                                      ptr(tpe), ptr(ws), current_stream()))
    assert bool((tpe == 0).all())
    tpf = torch.full((32,), -1.0, device="cuda")
    check(lib.xtb_router_noaux(ptr(d), ptr(d), 0, 32, 2, 1, 1, 1, 1.0, ptr(d), ptr(d), ptr(d), None, ptr(tpf),
                               current_stream()))
    assert bool((tpf == 0).all())
    check(lib.xtb_router_greedy_bwd(ptr(d), ptr(d), ptr(d), None, None, None, 0, 8, 2, 0, 1, 1.0, ptr(d),
                                    current_stream()))
    check(lib.xtb_router_noaux_bwd(ptr(d), ptr(d), ptr(d), ptr(d), ptr(d), None, None, 0, 32, 2, 0, 1, 1.0, ptr(d),
                                   current_stream()))
    gw = torch.full((8, 2048), 7.0, device="cuda")
    check(lib.xtb_gate_logits_bwd(None, None, ptr(w), ptr(gw), None, None, 0, 2048, 8, None, current_stream()))
    assert bool((gw == 0).all())
