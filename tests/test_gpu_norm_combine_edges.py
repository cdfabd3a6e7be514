"""The norm, combine and dispatch-backward kernels of the block path (csrc/norm.cu, csrc/permute.cu) against the exact
restatements and float64 references of tests/norm_combine_reference.py, at the edges the end-to-end tests cannot see.

* xtb_moe_combine / xtb_moe_unpermute: K in {1..8, 16} (every compile-time K and the runtime-K loop), H from 8 to 7168
  (lanes without a vector, unroll tails), T from 1 to 4099, probs and residual given or not, hidden_factor 1, 0.5, 0.7,
  1.5, rows mapped to -1: bit for bit against the restatement.  One case past 2^31 elements.
* xtb_moe_unpermute_bwd: act_grad bit for bit, each referenced row written once and the others never, prob_grad within
  its bound (exactly 0 for a -1 entry), prob_grad = y_fwd = NULL accepted.
* xtb_rmsnorm_gate: both kernels (norm only; with the gate at E = 1, 3, 8) at every supported H, T with 4-token block
  and 2-token warp tails, rows from 2^-60 to 2^40, zero rows and eps-dominated rows: rstd and the gate logits within
  their bounds, x bit for bit given the kernel's rstd and a correct rounding of float64 (near ties aside).  Refusals.
* xtb_moe_dispatch_bwd_rmsnorm: K in {1, 2, 3, 4, 6, 8} (pipelined kernel for K = 2 and 8, generic one otherwise), H
  in {8, 256, 264, 2048}, T from 1 to 65537 (one, two, ~four and unequal numbers of token groups per CTA), every
  combination of the nullable g_x_gate, g_res and g_norm_w.  g_x bit for bit, g_h near-tie against float64, the
  residual as a bf16 add on the kernel's own g_h, g_norm_w within its bound; pipelined == generic; NaN in every row no
  entry references; a large last token under a partial group; determinism; T = 0.

Every output is written into a view with 16 guard rows on each side, pre-filled with NaN: the guards must stay NaN, so
must every permuted row no entry references, and no other output element may keep the fill."""
import math

import pytest
import torch

from tests import norm_combine_reference as R
from tests.gpu_harness import XTB_ERR_INVALID, Guarded, Worst, sm_count
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu

WORST = Worst("norm_combine_edges")
_report = WORST.fixture()


# ---- the C entries -----------------------------------------------------------------------------------------------------


def combine(y, rmap, p, res, hf, T, K, H, out):
    if res is None and hf == 1.0:
        return ensure_init().xtb_moe_unpermute(ptr(y), ptr(rmap), ptr(p), T, K, H, ptr(out), current_stream())
    return ensure_init().xtb_moe_combine(ptr(y), ptr(rmap), ptr(p), ptr(res), hf, T, K, H, ptr(out), current_stream())


def unpermute_bwd(g, y, rmap, p, T, K, H, act, pg):
    return ensure_init().xtb_moe_unpermute_bwd(ptr(g), ptr(y), ptr(rmap), ptr(p), T, K, H, ptr(act), ptr(pg),
                                               current_stream())


def rmsnorm_gate(h, w, gate_w, T, H, E, x, rstd, logits, eps=R.EPS):
    return ensure_init().xtb_rmsnorm_gate(ptr(h), ptr(w), ptr(gate_w), eps, T, H, E, ptr(x), ptr(rstd), ptr(logits),
                                          current_stream())


def dispatch_bwd(g_xp, rmap, gate, h, rstd, w, g_res, T, K, H, g_h, g_nw):
    lib = ensure_init()
    ws = None
    if g_nw is not None:
        ws = torch.empty(int(lib.xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(T, H)), dtype=torch.uint8, device="cuda")
    return lib.xtb_moe_dispatch_bwd_rmsnorm(ptr(g_xp), ptr(rmap), ptr(gate), ptr(h), ptr(rstd), ptr(w), ptr(g_res), T,
                                            K, H, ptr(g_h), ptr(g_nw), ptr(ws), current_stream())


def _n_cta(T):
    return max(1, min(2 * sm_count(), (T + 3) // 4))


# ---- combine / unpermute -----------------------------------------------------------------------------------------------

COMBINE_H = (8, 248, 256, 264, 1032, 2048, 7168)
COMBINE_T = (1, 7, 8, 9, 4099)
HFS = (1.0, 0.5, 0.7, 1.5)


def _combine_case(K, H, T, mode, with_p, with_res, hf, seed):
    rmap, owner = R.row_map(T, K, seed, 0.1, "cuda")
    sc = R.token_scales(T, seed + 1, "cuda")
    y = R.permuted_rows(owner, H, sc, mode, seed + 2)  # rows no entry references are NaN
    p = R.probs(T, K, mode, seed + 3, "cuda") if with_p else None
    res = R.token_rows(sc, H, "random", seed + 4) if with_res else None
    out = Guarded(T, H, torch.bfloat16)
    check(combine(y, rmap, p, res, hf, T, K, H, out.v), "combine")
    torch.cuda.synchronize()
    what = f"combine K={K} H={H} T={T} {mode} probs={with_p} residual={with_res} hf={hf}"
    out.check(what)
    want = R.combine(y, rmap, p, res, hf, K)
    R.assert_bits_equal(out.v, want, what)
    ref, bnd = R.combine_ref(y, rmap, p, res, hf, K)
    WORST.note("combine restatement vs fp64", R.check_bound(want, ref, bnd, what))


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 6, 7, 8, 16])
def test_combine_exact(K):
    for i, H in enumerate(COMBINE_H):
        j = i + K
        _combine_case(K, H, COMBINE_T[j % 5], "exact" if i % 2 == 0 else "random", with_p=(j % 3 != 2),
                      with_res=(i % 2 == 1), hf=HFS[j % 4], seed=100 * K + i)
    for T in COMBINE_T:  # every T with probs, residual and a factor that is not a power of two
        _combine_case(K, 264, T, "random", True, True, 0.7, seed=7 * T + K)


def test_combine_past_2g_elements():
    """T K H > 2^31: the last 64 permuted rows start past element 2^31.  Sampled tokens only."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    T, K, H = 32776, 8, 8192
    M = T * K
    assert (M - 64) * H >= 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(5)
    rmap = torch.randperm(M, generator=g, device="cuda").to(torch.int32)
    y = torch.empty((M, H), dtype=torch.bfloat16, device="cuda")
    for s in range(0, M, 16384):
        y[s : s + 16384] = torch.randn((min(16384, M - s), H), generator=g, device="cuda")
    p = torch.rand((T, K), generator=g, device="cuda")
    res = torch.randn((T, H), generator=g, device="cuda").to(torch.bfloat16)
    out = torch.empty((T, H), dtype=torch.bfloat16, device="cuda")
    check(combine(y, rmap, p, res, 0.7, T, K, H, out), "combine")
    gout = torch.randn((T, H), generator=g, device="cuda").to(torch.bfloat16)
    act = torch.empty((M, H), dtype=torch.bfloat16, device="cuda")
    pg = torch.empty((T, K), dtype=torch.float32, device="cuda")
    check(unpermute_bwd(gout, y, rmap, p, T, K, H, act, pg), "unpermute_bwd")
    torch.cuda.synchronize()
    far = (rmap.view(T, K).long() >= 2 ** 31 // H).any(1).nonzero().flatten()
    assert far.numel() > 0
    toks = torch.cat([torch.arange(64, device="cuda"), torch.arange(T - 64, T, device="cuda"), far]).unique()
    sub = rmap.view(T, K)[toks]
    rows = sub.reshape(-1).long()
    # the sampled tokens' rows, renumbered 0 .. n-1
    ys = y[rows]
    local = torch.arange(rows.numel(), device="cuda", dtype=torch.int32)
    R.assert_bits_equal(out[toks], R.combine(ys, local, p[toks], res[toks], 0.7, K), "combine past 2^31 elements")
    want, _ = R.act_grad(gout[toks], local, p[toks], K, rows.numel())
    R.assert_bits_equal(act[rows], want, "act_grad past 2^31 elements")
    ref, bnd = R.prob_grad_ref(gout[toks], ys, local, K)
    WORST.note("prob_grad", R.check_bound(pg[toks], ref, bnd, "prob_grad past 2^31 elements"))
    WORST["peak GiB, 2^31-element case"] = torch.cuda.max_memory_allocated() / 2 ** 30
    del y, act, out, gout, res, ys
    torch.cuda.empty_cache()


def test_combine_refusals_name_the_entry():
    lib = ensure_init()
    y = torch.zeros((8, 16), dtype=torch.bfloat16, device="cuda")
    m = torch.zeros(8, dtype=torch.int32, device="cuda")
    out = torch.empty((8, 16), dtype=torch.bfloat16, device="cuda")
    assert lib.xtb_moe_combine(ptr(y), ptr(m), None, None, 1.0, 8, 1, 12, ptr(out), current_stream()) == XTB_ERR_INVALID
    assert b"xtb_moe_combine" in lib.xtb_last_error()
    assert lib.xtb_moe_combine(ptr(y), None, None, None, 1.0, 8, 1, 16, ptr(out), current_stream()) == XTB_ERR_INVALID
    assert b"xtb_moe_combine" in lib.xtb_last_error()
    assert lib.xtb_moe_unpermute(ptr(y), ptr(m), None, 8, 1, 12, ptr(out), current_stream()) == XTB_ERR_INVALID
    msg = lib.xtb_last_error()
    assert b"xtb_moe_unpermute" in msg and b"xtb_moe_combine" not in msg


# ---- unpermute backward ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 6, 7, 8, 16])
def test_unpermute_bwd(K):
    for i, H in enumerate(COMBINE_H):
        T = COMBINE_T[(i + K) % 5]
        mode = "exact" if i % 2 == 0 else "random"
        seed = 300 * K + i
        what = f"unpermute_bwd K={K} H={H} T={T} {mode}"
        rmap, owner = R.row_map(T, K, seed, 0.1, "cuda")
        sc = R.token_scales(T, seed + 1, "cuda")
        y = R.permuted_rows(owner, H, sc, mode, seed + 2)
        p = R.probs(T, K, mode, seed + 3, "cuda") if i % 3 != 1 else None
        g = R.token_rows(R.token_scales(T, seed + 4, "cuda"), H, mode, seed + 5)
        M = T * K
        act, pg = Guarded(M, H, torch.bfloat16), Guarded(T, K, torch.float32)
        check(unpermute_bwd(g, y, rmap, p, T, K, H, act.v, pg.v), what)
        act2 = Guarded(M, H, torch.bfloat16)
        check(unpermute_bwd(g, None, rmap, p, T, K, H, act2.v, None), what + " without prob_grad")
        torch.cuda.synchronize()
        want, written = R.act_grad(g, rmap, p, K, M)
        act.check(what, written)
        act2.check(what + " without prob_grad", written)
        pg.check(what + " prob_grad")
        R.assert_bits_equal(act.v[written], want[written], what)
        assert torch.equal(act.buf, act2.buf), f"{what}: act_grad depends on whether prob_grad is asked for"
        ref, bnd = R.prob_grad_ref(g, y, rmap, K)
        WORST.note("prob_grad", R.check_bound(pg.v, ref, bnd, what))
        neg = rmap.view(T, K) < 0
        assert bool((pg.v[neg] == 0).all()), f"{what}: prob_grad of a -1 entry is not 0"


# ---- rmsnorm (+ gate) --------------------------------------------------------------------------------------------------


def _norm_case(H, T, E, seed):
    h = R.norm_rows(T, H, seed, "cuda")
    w = R.norm_weight(H, seed + 1, "cuda")
    gate_w = (torch.randn((E, H), generator=torch.Generator(device="cuda").manual_seed(seed + 2), device="cuda") * H ** -0.5
              if E else None)
    what = f"rmsnorm_gate H={H} T={T} E={E}"
    xg, rg, lg = Guarded(T, H, torch.bfloat16), Guarded(T, 1, torch.float32), Guarded(T, max(E, 1), torch.float32)
    check(rmsnorm_gate(h, w, gate_w, T, H, E, xg.v, rg.v, lg.v if E else None), what)
    xg2, lg2 = Guarded(T, H, torch.bfloat16), Guarded(T, max(E, 1), torch.float32)
    check(rmsnorm_gate(h, w, gate_w, T, H, E, xg2.v, None, lg2.v if E else None), what + " without rstd")
    torch.cuda.synchronize()
    x = xg.check(what + " x")
    rs = rg.check(what + " rstd")[:, 0]
    if E:
        lg.check(what + " logits")
        assert torch.equal(lg.buf, lg2.buf), f"{what}: logits depend on whether rstd is written"
    assert torch.equal(xg.buf, xg2.buf), f"{what}: x depends on whether rstd is written"
    ref = R.rstd_ref(h, R.EPS)
    WORST.note("rstd", R.check_bound(rs, ref, R.rstd_rel(H) * ref, what + " rstd"))
    R.assert_bits_equal(x, R.rmsnorm_x(h, rs, w), what + " x given the kernel's rstd")
    xr, xb = R.x_ref(h, R.EPS, w)
    WORST.note("x (bf16, past the midpoint)", R.check_near_tie(x, xr, xb, what + " x")[0])
    if E:
        lr, lb = R.logits_ref(x, gate_w)
        WORST.note("gate logits", R.check_bound(lg.v, lr, lb, what + " logits"))


@pytest.mark.parametrize("H", [256, 512, 1024, 2048])
def test_rmsnorm(H):
    for T in (1, 2, 3, 4, 5, 4099):
        _norm_case(H, T, 0, seed=H + T)
    for E in (1, 3, 8):
        for T in (1, 3, 4099):
            _norm_case(H, T, E, seed=H + 10 * E + T)


def test_rmsnorm_refusals():
    lib = ensure_init()
    T = 4
    h = torch.zeros((T, 4096), dtype=torch.bfloat16, device="cuda")
    w = torch.ones(4096, dtype=torch.float32, device="cuda")
    gw = torch.zeros((9, 4096), dtype=torch.float32, device="cuda")
    x = torch.empty_like(h)
    rstd = torch.empty(T, dtype=torch.float32, device="cuda")
    lg = torch.empty((T, 9), dtype=torch.float32, device="cuda")
    for H in (384, 4096, 260):
        for gate in (None, gw):
            assert rmsnorm_gate(h, w, gate, T, H, 8, x, rstd, lg) == XTB_ERR_INVALID, f"H={H} accepted"
            assert b"xtb_rmsnorm_gate" in lib.xtb_last_error()
    assert rmsnorm_gate(h, w, gw, T, 256, 9, x, rstd, lg) == XTB_ERR_INVALID, "E=9 accepted with the gate"


# ---- dispatch backward + RMSNorm backward ------------------------------------------------------------------------------

BWD_H = (8, 256, 264, 2048)
BWD_T = (1, 2, 3, 5, 263, 1056, 1057, 8192, 65537)


def _bwd_inputs(T, K, H, seed, mode="exact", rmap=None, owner=None):
    if rmap is None:
        rmap, owner = R.row_map(T, K, seed, 0.1, "cuda")
    sc = R.token_scales(T, seed + 1, "cuda", exp_range=(-4, 4))
    g_xp = R.permuted_rows(owner, H, sc, mode, seed + 2)  # rows no entry references are NaN
    gate = R.token_rows(sc, H, "random", seed + 3)
    h = R.norm_rows(T, H, seed + 4, "cuda")
    rstd = R.rstd_ref(h, R.EPS).float()
    w = R.norm_weight(H, seed + 5, "cuda")
    g_res = R.token_rows(sc, H, "random", seed + 6)
    return rmap, g_xp, gate, h, rstd, w, g_res


def _bwd_run(T, K, H, rmap, g_xp, gate, h, rstd, w, g_res, with_nw, what):
    """Runs without and with g_res; checks guards, the residual composition and that g_norm_w ignores g_res.
    Returns (g_h without g_res, g_norm_w or None)."""
    gh0, gh1 = Guarded(T, H, torch.bfloat16), Guarded(T, H, torch.bfloat16)
    nw0, nw1 = Guarded(1, H, torch.float32), Guarded(1, H, torch.float32)
    check(dispatch_bwd(g_xp, rmap, gate, h, rstd, w, None, T, K, H, gh0.v, nw0.v[0] if with_nw else None), what)
    check(dispatch_bwd(g_xp, rmap, gate, h, rstd, w, g_res, T, K, H, gh1.v, nw1.v[0] if with_nw else None),
          what + " +g_res")
    torch.cuda.synchronize()
    gh0.check(what + " g_h")
    gh1.check(what + " g_h +g_res")
    R.assert_bits_equal(gh1.v, (gh0.v.float() + g_res.float()).to(torch.bfloat16),
                        what + " g_h(res) vs bf16(g_h + g_res)")
    if not with_nw:
        nw0.check(what + " g_norm_w, NULL", written=False)
        nw1.check(what + " g_norm_w, NULL +g_res", written=False)
        return gh0.v, None
    nw0.check(what + " g_norm_w")
    assert torch.equal(nw0.buf, nw1.buf), f"{what}: g_norm_w depends on g_res"
    return gh0.v, nw0.v[0]


def _check_bwd(T, K, H, rmap, g_xp, gate, h, rstd, w, gh, nw, what):
    g_x = R.dispatch_gx(g_xp, rmap, gate, K)
    ref, bnd = R.g_h_ref(g_x, h, rstd, w)
    WORST.note("g_h (bf16, past the midpoint)", R.check_near_tie(gh, ref, bnd, what + " g_h")[0])
    if nw is not None:
        gr, gb = R.g_norm_w_ref(g_x, h, rstd, _n_cta(T))
        WORST.note("g_norm_w", R.check_bound(nw, gr, gb, what + " g_norm_w"))


@pytest.mark.parametrize("K", [1, 2, 3, 4, 6, 8])
def test_dispatch_bwd_rmsnorm(K):
    i = 0
    for H in BWD_H:
        for T in BWD_T:
            if T * H > 2 ** 26:
                continue  # T = 65537 runs at the narrow widths
            with_gate, with_nw = (i % 2 == 0), (i // 2 % 2 == 0)
            what = f"dispatch_bwd K={K} H={H} T={T} gate={with_gate} g_norm_w={with_nw}"
            rmap, g_xp, gate, h, rstd, w, g_res = _bwd_inputs(T, K, H, 1000 * K + i)
            gate = gate if with_gate else None
            gh, nw = _bwd_run(T, K, H, rmap, g_xp, gate, h, rstd, w, g_res, with_nw, what)
            _check_bwd(T, K, H, rmap, g_xp, gate, h, rstd, w, gh, nw, what)
            i += 1


@pytest.mark.parametrize("K", [1, 2, 3, 4, 6, 8])
def test_dispatch_bwd_g_x_exact(K):
    """h = 0, rstd = 1, w = 1 makes g_h = g_x exactly: the dispatch backward's sum and gate add, bit for bit."""
    i = 0
    for H in BWD_H:
        for T in (1, 5, 1057, 8192):
            what = f"dispatch_bwd g_x K={K} H={H} T={T}"
            rmap, g_xp, gate, h, rstd, w, g_res = _bwd_inputs(T, K, H, 2000 * K + i, mode="random")
            gate = gate if i % 2 == 0 else None
            h = torch.zeros_like(h)
            rstd = torch.ones_like(rstd)
            w = torch.ones_like(w)
            gh, nw = _bwd_run(T, K, H, rmap, g_xp, gate, h, rstd, w, g_res, True, what)
            R.assert_bits_equal(gh, R.dispatch_gx(g_xp, rmap, gate, K), what)
            assert bool((nw == 0).all()), f"{what}: g_norm_w of h = 0 is not 0"
            i += 1


def _pad_map(rmap, T, K, pad, seed):
    """[T, K + pad] with ``pad`` -1 entries per token at random positions, the real entries in their order."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    keys = torch.rand((T, K + pad), generator=g, device="cuda")
    slots = keys.argsort(1)[:, :K].sort(1).values  # K sorted positions per token
    out = torch.full((T, K + pad), -1, dtype=torch.int32, device="cuda")
    out.scatter_(1, slots, rmap.view(T, K))
    return out.view(-1)


@pytest.mark.parametrize("K,pad", [(2, 2), (8, 1)])
def test_dispatch_bwd_pipe_equals_generic(K, pad):
    """K = 2 and 8 take the pipelined kernel; the same entries padded with -1 to K + pad take the generic one."""
    for H in (264, 2048):
        for T in (263, 1057, 8192):
            what = f"pipe K={K} vs generic K={K + pad}, H={H} T={T}"
            rmap, g_xp, gate, h, rstd, w, g_res = _bwd_inputs(T, K, H, 3000 + T + H, mode="random")
            padded = _pad_map(rmap, T, K, pad, T)
            gh_p, nw_p = _bwd_run(T, K, H, rmap, g_xp, gate, h, rstd, w, g_res, True, what + " (pipe)")
            gh_g, nw_g = _bwd_run(T, K + pad, H, padded, g_xp, gate, h, rstd, w, g_res, True, what + " (generic)")
            R.assert_bits_equal(gh_p, gh_g, what)
            _check_bwd(T, K, H, rmap, g_xp, gate, h, rstd, w, gh_p, nw_p, what + " (pipe)")
            _check_bwd(T, K + pad, H, padded, g_xp, gate, h, rstd, w, gh_g, nw_g, what + " (generic)")


@pytest.mark.parametrize("K", [2, 3])
def test_dispatch_bwd_large_last_token(K):
    """With T odd the last token group is partial and its empty slots load row T-1; they must add nothing to g_norm_w."""
    for T in (5, 263, 1057):
        H = 256
        what = f"dispatch_bwd last token K={K} T={T}"
        rmap, owner = R.row_map(T, K, T, 0.0, "cuda")
        sc = torch.ones(T, device="cuda")
        sc[-1] = 2.0 ** 10
        g_xp = R.permuted_rows(owner, H, sc, "random", T + 1)
        h = (torch.randn((T, H), generator=torch.Generator(device="cuda").manual_seed(T), device="cuda")
             * torch.where(torch.arange(T, device="cuda") == T - 1, 2.0 ** 10, 1.0)[:, None]).to(torch.bfloat16)
        rstd = torch.ones(T, device="cuda")
        w = R.norm_weight(H, T + 2, "cuda")
        g_res = torch.zeros((T, H), dtype=torch.bfloat16, device="cuda")
        gh, nw = _bwd_run(T, K, H, rmap, g_xp, None, h, rstd, w, g_res, True, what)
        _check_bwd(T, K, H, rmap, g_xp, None, h, rstd, w, gh, nw, what)


def test_dispatch_bwd_bench_shape_deterministic():
    """The benchmark's layer: T = 8192, H = 2048, top-2 of 8 experts, rows in expert order as permute makes them."""
    T, H, K, E = 8192, 2048, 2, 8
    g = torch.Generator(device="cuda").manual_seed(11)
    ids = torch.randint(0, E, (T * K,), generator=g, device="cuda")
    order = ids.argsort(stable=True)
    rmap = torch.empty(T * K, dtype=torch.int32, device="cuda")
    rmap[order] = torch.arange(T * K, dtype=torch.int32, device="cuda")
    owner = torch.arange(T * K, device="cuda") // K
    owner = owner[order]
    rm, g_xp, gate, h, rstd, w, g_res = _bwd_inputs(T, K, H, 12, mode="random", rmap=rmap, owner=owner)
    what = "dispatch_bwd bench shape"
    gh, nw = _bwd_run(T, K, H, rmap, g_xp, gate, h, rstd, w, g_res, True, what)
    _check_bwd(T, K, H, rmap, g_xp, gate, h, rstd, w, gh, nw, what)
    gh2, nw2 = _bwd_run(T, K, H, rmap, g_xp, gate, h, rstd, w, g_res, True, what + " (again)")
    assert torch.equal(gh.view(torch.int16), gh2.view(torch.int16)) and torch.equal(nw.view(torch.int32), nw2.view(torch.int32)), \
        f"{what}: two calls differ"


def test_dispatch_bwd_refuses_wide_rows():
    T, H = 4, 2056
    z = torch.zeros((T * 2, H), dtype=torch.bfloat16, device="cuda")
    m = torch.zeros(T * 2, dtype=torch.int32, device="cuda")
    r = torch.ones(T, device="cuda")
    w = torch.ones(H, device="cuda")
    out = torch.empty((T, H), dtype=torch.bfloat16, device="cuda")
    assert dispatch_bwd(z, m, None, z, r, w, None, T, 2, H, out, None) == XTB_ERR_INVALID
    assert b"xtb_moe_dispatch_bwd_rmsnorm" in ensure_init().xtb_last_error()


def test_empty_batch_writes_nothing():
    H, K = 256, 2
    z = torch.zeros((4, H), dtype=torch.bfloat16, device="cuda")
    m = torch.zeros(4, dtype=torch.int32, device="cuda")
    f = torch.ones(H, device="cuda")
    # one row each, so that the pointers are not NULL
    out, fout, nw = Guarded(1, H, torch.bfloat16), Guarded(1, 1, torch.float32), Guarded(1, H, torch.float32)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    lib = ensure_init()
    assert lib.xtb_moe_combine(ptr(z), ptr(m), None, ptr(z), 0.7, 0, K, H, ptr(out.v), current_stream()) == 0
    assert lib.xtb_moe_unpermute_bwd(ptr(z), ptr(z), ptr(m), None, 0, K, H, ptr(out.v), ptr(fout.v),
                                     current_stream()) == 0
    assert rmsnorm_gate(z, f, None, 0, H, 0, out.v, fout.v, None) == 0
    assert lib.xtb_moe_dispatch_bwd_rmsnorm(ptr(z), ptr(m), None, ptr(z), ptr(f), ptr(f), None, 0, K, H, ptr(out.v),
                                            ptr(nw.v[0]), ptr(ws), current_stream()) == 0
    torch.cuda.synchronize()
    for g, name in ((out, "bf16 out"), (fout, "fp32 out"), (nw, "g_norm_w")):
        g.check(f"T = 0 wrote {name}", written=False)
    assert math.isnan(float(nw.v[0, 0]))
