"""Grouped expert GEMMs (csrc/group_gemm.cu) against float64 references at the edges the parity tests do not reach.

* Exact: exact-mode inputs (tests/gemm_reference.py) make every fp32 sum exact, so every output of xtb_group_gemm_nt,
  _nt_swiglu, _nn, _tn and _tn_pair must be bf16(fp64 reference) bit for bit — at every tile width each entry selects,
  with 1, 8, 33, 128 and 1024 experts (the device prefix scan over tokens_per_expert walks 32 experts per step), ragged
  counts from {0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257} (16-row store boxes, 64-row TN k-blocks,
  128-row tiles), empty first, last and consecutive experts.  Every output is written into a view of a buffer with 16
  guard rows on each side, all pre-filled with a NaN pattern: the guards must stay untouched and no output element may
  keep the fill (a masked store writing outside its rows, or a skipped tile, shows).
* Bound: random-mode inputs at the benchmark geometry and at a 128-expert one, against |out - ref| <= 2^-8 |ref| + tau S.
* Isolation: NaN in every row and weight that is not the victim expert's leaves the victim's outputs bit-identical.
* ops.group_gemm refuses inconsistent shapes on the host, before any launch."""
import pytest
import torch

from oracle import moe_oracle as O
from tests import gemm_reference as R
from tests.gpu_harness import XTB_ERR_INVALID, Guarded
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu


# ---- the C entries -----------------------------------------------------------------------------------------------------


def nt(x, w, tpe, out):
    E, N, Kd = w.shape
    return ensure_init().xtb_group_gemm_nt(ptr(x), ptr(w), ptr(tpe), x.shape[0], N, Kd, E, ptr(out), current_stream())


def nn(dy, w, tpe, out):
    E, N, Kd = w.shape
    return ensure_init().xtb_group_gemm_nn(ptr(dy), ptr(w), ptr(tpe), dy.shape[0], N, Kd, E, ptr(out), current_stream())


def swiglu_gemm(x, w13, tpe, h, a):
    E, twoI, Kd = w13.shape
    return ensure_init().xtb_group_gemm_nt_swiglu(ptr(x), ptr(w13), ptr(tpe), x.shape[0], twoI // 2, Kd, E, ptr(h),
                                                  ptr(a), current_stream())


def tn(dy, x, tpe, dw, E):
    return ensure_init().xtb_group_gemm_tn(ptr(dy), ptr(x), ptr(tpe), x.shape[0], dy.shape[1], x.shape[1], E, ptr(dw),
                                           current_stream())


def tn_pair(dya, xa, dwa, dyb, xb, dwb, tpe, E):
    return ensure_init().xtb_group_gemm_tn_pair(ptr(dya), ptr(xa), dya.shape[1], xa.shape[1], ptr(dwa), ptr(dyb),
                                                ptr(xb), dyb.shape[1], xb.shape[1], ptr(dwb), ptr(tpe), xa.shape[0], E,
                                                current_stream())


def _xtb_swiglu(h):
    a = torch.empty(h.shape[0], h.shape[1] // 2, dtype=torch.bfloat16, device="cuda")
    check(ensure_init().xtb_swiglu(ptr(h), ptr(a), h.shape[0], h.shape[1] // 2, current_stream()), "xtb_swiglu")
    return a


def _tpe(counts):
    return torch.tensor(counts, dtype=torch.int64, device="cuda")


def _counts(E, pattern, seed):
    return R.counts_pattern(E, pattern, seed, total={"single": 16381, "zipf": 4096}.get(pattern, 0))


def _assert_swiglu_a(a, h, what):
    """a = xtb_swiglu(h) bit for bit (same silu_fast, same roundings); the oracle's swiglu within rare 1-ulp flips."""
    ref = _xtb_swiglu(h)
    diff = a.view(torch.int16) != ref.view(torch.int16)
    if bool(diff.any()):
        r, c = (int(i) for i in diff.nonzero()[0])
        raise AssertionError(f"{what}: a differs from xtb_swiglu(h) in {int(diff.sum())} elements; first at row {r}, "
                             f"column {c}: {a[r, c].item()!r} vs {ref[r, c].item()!r} (h_gate {h[r, c].item()!r})")
    d = R.ulp_distance(a.cpu(), O.swiglu(h.cpu()))
    assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 1e-3, (what, int(d.max()), float((d > 0).float().mean()))


# ---- B: exact ------------------------------------------------------------------------------------------------------------

# (E, count pattern, N, Kd).  NT picks its tile width from N, NN and TN from Kd: N / Kd mod 256 in {0, 128} for each.
NT_CASES = [(1, "single", 384, 256), (8, "ragged", 512, 384), (33, "ragged", 1792, 128), (33, "ragged", 384, 256),
            (128, "zipf", 256, 512), (128, "zipf", 128, 128), (1024, "sparse", 128, 128)]
NN_TN_CASES = [(1, "single", 256, 384), (8, "ragged", 384, 512), (33, "ragged", 128, 1792), (33, "ragged", 256, 384),
               (128, "zipf", 512, 256), (128, "zipf", 128, 128), (1024, "sparse", 128, 128)]


def _id(c):
    return "-".join(str(v) for v in c)


def test_some_case_walks_more_than_two_waves_of_tiles():
    """Every persistent CTA (132 on an H100 SXM) walks tiles of several experts in at least one exact case."""
    E, pattern, N, _ = NT_CASES[2]
    assert R.m_tiles(_counts(E, pattern, 0)) * (N // 256) > 2 * 132


@pytest.mark.parametrize("case", NT_CASES, ids=_id)
def test_nt_exact(case):
    E, pattern, N, Kd = case
    counts = _counts(E, pattern, 0)
    M = sum(counts)
    x = R.rows_operand(counts, Kd, "exact", 1, "cuda")
    w = R.weight_operand(E, N, Kd, "exact", 2, "cuda")
    out = Guarded(M, N, torch.bfloat16)
    check(nt(x, w, _tpe(counts), out.v), "nt")
    torch.cuda.synchronize()
    R.assert_exact(out.check(f"nt {case}"), "nt", x, w, counts, f"{case}")


@pytest.mark.parametrize("case", NN_TN_CASES, ids=_id)
def test_nn_exact(case):
    E, pattern, N, Kd = case
    counts = _counts(E, pattern, 1)
    M = sum(counts)
    dy = R.rows_operand(counts, N, "exact", 3, "cuda")
    w = R.weight_operand(E, N, Kd, "exact", 4, "cuda")
    out = Guarded(M, Kd, torch.bfloat16)
    check(nn(dy, w, _tpe(counts), out.v), "nn")
    torch.cuda.synchronize()
    R.assert_exact(out.check(f"nn {case}"), "nn", dy, w, counts, f"{case}")


@pytest.mark.parametrize("case", NN_TN_CASES, ids=_id)
def test_tn_exact(case):
    E, pattern, N, Kd = case
    counts = _counts(E, pattern, 2)
    dy = R.rows_operand(counts, N, "exact", 5, "cuda")
    x = R.rows_operand(counts, Kd, "exact", 6, "cuda")
    dw = Guarded(E * N, Kd, torch.bfloat16)
    check(tn(dy, x, _tpe(counts), dw.v, E), "tn")
    torch.cuda.synchronize()
    R.assert_exact(dw.check(f"tn {case}").view(E, N, Kd), "tn", dy, x, counts, f"{case}")


# (E, pattern, N_a, Kd_a, N_b, Kd_b): equal tile widths run as one launch, unequal ones as two
TN_PAIR_CASES = [(8, "ragged", 256, 512, 384, 256), (33, "ragged", 128, 384, 256, 128), (128, "zipf", 256, 256, 128, 384),
                 (1, "single", 128, 128, 256, 256), (1024, "sparse", 128, 128, 128, 128)]


@pytest.mark.parametrize("case", TN_PAIR_CASES, ids=_id)
def test_tn_pair_exact(case):
    E, pattern, Na, Ka, Nb, Kb = case
    counts = _counts(E, pattern, 3)
    dya, xa = R.rows_operand(counts, Na, "exact", 7, "cuda"), R.rows_operand(counts, Ka, "exact", 8, "cuda")
    dyb, xb = R.rows_operand(counts, Nb, "exact", 9, "cuda"), R.rows_operand(counts, Kb, "exact", 10, "cuda")
    ga, gb = Guarded(E * Na, Ka, torch.bfloat16), Guarded(E * Nb, Kb, torch.bfloat16)
    check(tn_pair(dya, xa, ga.v, dyb, xb, gb.v, _tpe(counts), E), "tn_pair")
    torch.cuda.synchronize()
    dwa, dwb = ga.check(f"tn_pair a {case}"), gb.check(f"tn_pair b {case}")
    R.assert_exact(dwa.view(E, Na, Ka), "tn", dya, xa, counts, f"pair a {case}")
    R.assert_exact(dwb.view(E, Nb, Kb), "tn", dyb, xb, counts, f"pair b {case}")


# (E, pattern, I, Kd): I = 64 and 192 take the 128-wide tiles (64 gate + 64 up columns), the rest the 256-wide ones;
# I >= 192 has tiles with n_blk > 0 at both widths
SWIGLU_CASES = [(1, "single", 64, 256), (8, "ragged", 192, 384), (33, "ragged", 128, 128), (128, "zipf", 256, 256),
                (8, "ragged", 768, 512), (1024, "sparse", 64, 128)]


@pytest.mark.parametrize("case", SWIGLU_CASES, ids=_id)
def test_nt_swiglu_exact(case):
    E, pattern, I, Kd = case
    counts = _counts(E, pattern, 4)
    M = sum(counts)
    x = R.rows_operand(counts, Kd, "exact", 11, "cuda")
    w13 = R.weight_operand(E, 2 * I, Kd, "exact", 12, "cuda")
    hg, ag = Guarded(M, 2 * I, torch.bfloat16), Guarded(M, I, torch.bfloat16)
    check(swiglu_gemm(x, w13, _tpe(counts), hg.v, ag.v), "nt_swiglu")
    torch.cuda.synchronize()
    h, a = hg.check(f"nt_swiglu h {case}"), ag.check(f"nt_swiglu a {case}")
    R.assert_exact(h, "nt", x, w13, counts, f"swiglu h {case}")
    _assert_swiglu_a(a, h, f"swiglu {case}")


@pytest.mark.parametrize("I", [64, 192, 128, 256, 768])
def test_nt_swiglu_h_is_the_plain_nt_product(I):
    """Random-mode data: the SwiGLU GEMM's h is xtb_group_gemm_nt's output on the same operands bit for bit (same tile
    width, same wgmma shape, same k order; only the column placement of the tiles differs)."""
    counts = R.counts_pattern(8, "ragged", 5)
    M, Kd = sum(counts), 512
    x = R.rows_operand(counts, Kd, "random", 13, "cuda", exp_range=(-2, 2))
    w13 = R.weight_operand(8, 2 * I, Kd, "random", 14, "cuda", exp_range=(-6, -3))
    tpe = _tpe(counts)
    h = torch.empty(M, 2 * I, dtype=torch.bfloat16, device="cuda")
    a = torch.empty(M, I, dtype=torch.bfloat16, device="cuda")
    h_nt = torch.empty_like(h)
    check(swiglu_gemm(x, w13, tpe, h, a), "nt_swiglu")
    check(nt(x, w13, tpe, h_nt), "nt")
    torch.cuda.synchronize()
    diff = h.view(torch.int16) != h_nt.view(torch.int16)
    if bool(diff.any()):
        r, c = (int(i) for i in diff.nonzero()[0])
        raise AssertionError(f"I={I}: h differs from nt in {int(diff.sum())} elements; first at row {r}, column {c}: "
                             f"{h[r, c].item()!r} vs {h_nt[r, c].item()!r}")
    R.check_bound(h, "nt", x, w13, counts, what=f"swiglu h I={I}")
    _assert_swiglu_a(a, h, f"random I={I}")


def test_more_than_1024_experts_is_rejected():
    """kMaxExperts = 1024 sizes the kernel's shared-memory prefix tables: E = 1025 is refused by every entry, before any
    launch and without touching the output."""
    lib = ensure_init()
    E, M = 1025, 128
    counts = [0] * E
    counts[3] = M
    tpe = _tpe(counts)
    x = torch.zeros(M, 128, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(E, 128, 128, dtype=torch.bfloat16, device="cuda")
    out = torch.full((E * 128, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    out2 = torch.full((M, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    torch.cuda.synchronize()
    before = lib.xtb_launch_count()
    rcs = {
        "nt": nt(x, w, tpe, out),
        "nn": nn(x, w, tpe, out),
        "nt_swiglu": swiglu_gemm(x, w, tpe, out, out2),
        "tn": tn(x, x, tpe, out, E),
        "tn_pair": tn_pair(x, x, out, x, x, out, tpe, E),
    }
    torch.cuda.synchronize()
    assert rcs == {k: XTB_ERR_INVALID for k in rcs}, rcs
    assert b"E=1025" in lib.xtb_last_error()
    assert lib.xtb_launch_count() == before
    assert bool(out.isnan().all() and out2.isnan().all())


# ---- C: bound at production shapes ---------------------------------------------------------------------------------------


def _expert_mlp_bounds(counts, H, I, seed):
    """Every entry at one expert-MLP geometry, random mode: the forward (nt_swiglu, then nt through w2), dX through both
    weights (nn), both dW (tn, and tn_pair bit for bit against a tn launch per product); returns the largest
    |out - ref| / bound per product."""
    E, M = len(counts), sum(counts)
    tpe = _tpe(counts)
    bf = dict(dtype=torch.bfloat16, device="cuda")
    x = R.rows_operand(counts, H, "random", seed, "cuda", exp_range=(-2, 2))
    w13 = R.weight_operand(E, 2 * I, H, "random", seed + 1, "cuda", exp_range=(-8, -4))
    w2 = R.weight_operand(E, H, I, "random", seed + 2, "cuda", exp_range=(-8, -4))
    dy = R.rows_operand(counts, H, "random", seed + 3, "cuda", exp_range=(-4, 0))
    ratios = {}
    h, a = torch.empty(M, 2 * I, **bf), torch.empty(M, I, **bf)
    check(swiglu_gemm(x, w13, tpe, h, a), "nt_swiglu")
    ratios["nt_swiglu.h"] = R.check_bound(h, "nt", x, w13, counts, what="h")
    _assert_swiglu_a(a, h, "production a")
    y = torch.empty(M, H, **bf)
    check(nt(a, w2, tpe, y), "nt")
    ratios["nt"] = R.check_bound(y, "nt", a, w2, counts, what="y")
    del y
    da = torch.empty(M, I, **bf)
    check(nn(dy, w2, tpe, da), "nn w2")
    ratios["nn.w2"] = R.check_bound(da, "nn", dy, w2, counts, what="da")
    dh = R.rows_operand(counts, 2 * I, "random", seed + 4, "cuda", exp_range=(-4, 0))
    dx = torch.empty(M, H, **bf)
    check(nn(dh, w13, tpe, dx), "nn w13")
    ratios["nn.w13"] = R.check_bound(dx, "nn", dh, w13, counts, what="dx")
    del dx, da
    gw2 = torch.empty(E, H, I, **bf)
    check(tn(dy, a, tpe, gw2, E), "tn")
    ratios["tn"] = R.check_bound(gw2, "tn", dy, a, counts, what="gw2")
    gw2p, gw13p = torch.empty(E, H, I, **bf), torch.empty(E, 2 * I, H, **bf)
    check(tn_pair(dy, a, gw2p, dh, x, gw13p, tpe, E), "tn_pair")
    torch.cuda.synchronize()
    assert torch.equal(gw2p.view(torch.int16), gw2.view(torch.int16)), "tn_pair differs from tn (gw2)"
    del gw2, gw2p
    ratios["tn_pair"] = R.check_bound(gw13p, "tn", dh, x, counts, what="gw13 pair")
    gw13 = torch.empty(E, 2 * I, H, **bf)
    check(tn(dh, x, tpe, gw13, E), "tn w13")
    torch.cuda.synchronize()
    assert torch.equal(gw13p.view(torch.int16), gw13.view(torch.int16)), "tn_pair differs from tn (gw13)"
    del gw13, gw13p
    return ratios, dict(x=x, w13=w13, w2=w2, a=a, dy=dy, tpe=tpe)


@pytest.mark.parametrize("skew", [False, True], ids=["balanced", "zipf"])
def test_bound_benchmark_geometry(skew):
    """H = 2048, I = 768, 8 experts, 16384 rows: the expert MLP of bench.py, SwiGLU epilogue included.
    Largest |out - ref| / bound measured on an NVIDIA H100 80GB HBM3 (700 W limit): 0.98 (nt through w2), 0.96-0.98 for
    the others.  The rounding to bf16 alone brings the ratio just under 1 (half an ulp at a mantissa of 1.0 is 2^-8 |ref|);
    the margin left is what tau S leaves for the fp32 accumulation."""
    E, M = 8, 16384
    counts = R.counts_pattern(E, "zipf" if skew else "balanced", 21, M)
    ratios, _ = _expert_mlp_bounds(counts, 2048, 768, 100 + int(skew))
    print("BOUND_RATIO", "bench", "zipf" if skew else "balanced", " ".join(f"{k}={v:.4f}" for k, v in ratios.items()))


def test_bound_128_experts_and_ops_group_gemm():
    """H = 2048, I = 768, 128 experts with top-8 routing of 4096 tokens (32768 rows), Zipf counts and empty experts —
    the geometry of the models the plugin's group_gemm seam serves — through every C entry and through ops.group_gemm's
    forward and backward, which must be the C entries' bits.
    Largest |out - ref| / bound measured on an NVIDIA H100 80GB HBM3 (700 W limit): 0.992 (tn, reductions up to 9227
    rows), 0.96-0.99 for the others."""
    from xtuner_b200 import ops

    counts = R.counts_pattern(128, "zipf", 22, 32768)
    ratios, t = _expert_mlp_bounds(counts, 2048, 768, 200)
    print("BOUND_RATIO", "e128", " ".join(f"{k}={v:.4f}" for k, v in ratios.items()))
    a, w2, dy, tpe = t["a"], t["w2"], t["dy"], t["tpe"]
    ar, wr = a.clone().requires_grad_(True), w2.clone().requires_grad_(True)
    y = ops.group_gemm(ar, wr, tpe)
    da, dw = torch.autograd.grad(y, (ar, wr), dy)
    bf = dict(dtype=torch.bfloat16, device="cuda")
    y_c, da_c, dw_c = torch.empty_like(y), torch.empty(a.shape, **bf), torch.empty(w2.shape, **bf)
    check(nt(a, w2, tpe, y_c), "nt")
    check(nn(dy, w2, tpe, da_c), "nn")
    check(tn(dy, a, tpe, dw_c, 128), "tn")
    torch.cuda.synchronize()
    for got, want in ((y, y_c), (da, da_c), (dw, dw_c)):
        assert torch.equal(got.detach().view(torch.int16), want.view(torch.int16))
    assert not dw[0].any() and not dw[127].any()  # empty experts


# ---- D: isolation ----------------------------------------------------------------------------------------------------------

ISO_COUNTS = [65, 0, 128, 200, None, 64, 0, 257, 33]  # None: the victim (expert 4)
VICTIM = 4


@pytest.mark.parametrize("victim_rows", [17, 129])
@pytest.mark.parametrize("entry", ["nt", "nn", "nt_swiglu", "tn", "tn_pair"])
def test_poisoned_neighbours_do_not_reach_the_victim(entry, victim_rows):
    """NaN in every row of the row operands outside the victim expert's range and in every other expert's weight: the
    victim's outputs are the bits of a clean run.  NT / NN / SwiGLU A tiles over-read the next expert's rows (masked at
    the store); TN must zero both operands' rows past the expert's end in its last k-block, or 0 * NaN poisons dW."""
    counts = [victim_rows if c is None else c for c in ISO_COUNTS]
    E, M = len(counts), sum(counts)
    o = R.offsets(counts)
    lo, hi = o[VICTIM], o[VICTIM + 1]
    tpe = _tpe(counts)
    N, Kd, I = 384, 256, 192
    nan = float("nan")

    def rows(cols, seed):
        clean = R.rows_operand(counts, cols, "random", seed, "cuda")
        bad = torch.full_like(clean, nan)
        bad[lo:hi] = clean[lo:hi]
        return clean, bad

    def weights(n, k, seed):
        clean = R.weight_operand(E, n, k, "random", seed, "cuda", exp_range=(-6, -3))
        bad = torch.full_like(clean, nan)
        bad[VICTIM] = clean[VICTIM]
        return clean, bad

    def run(poisoned):
        pick = (lambda pair: pair[1]) if poisoned else (lambda pair: pair[0])
        bf = dict(dtype=torch.bfloat16, device="cuda")
        if entry == "nt":
            out = torch.empty(M, N, **bf)
            check(nt(pick(X), pick(W), tpe, out), entry)
            return [out[lo:hi]]
        if entry == "nn":
            out = torch.empty(M, Kd, **bf)
            check(nn(pick(DY), pick(W), tpe, out), entry)
            return [out[lo:hi]]
        if entry == "nt_swiglu":
            h, a = torch.empty(M, 2 * I, **bf), torch.empty(M, I, **bf)
            check(swiglu_gemm(pick(X), pick(W13), tpe, h, a), entry)
            return [h[lo:hi], a[lo:hi]]
        if entry == "tn":
            dw = torch.empty(E, N, Kd, **bf)
            check(tn(pick(DY), pick(X), tpe, dw, E), entry)
            return [dw[VICTIM], dw[1], dw[6]]
        dwa, dwb = torch.empty(E, N, Kd, **bf), torch.empty(E, 2 * I, Kd, **bf)
        check(tn_pair(pick(DY), pick(X), dwa, pick(DH), pick(X), dwb, tpe, E), entry)
        return [dwa[VICTIM], dwb[VICTIM], dwa[1], dwb[6]]

    X, DY, DH = rows(Kd, 31), rows(N, 32), rows(2 * I, 33)
    W, W13 = weights(N, Kd, 34), weights(2 * I, Kd, 35)
    clean, poisoned = run(False), run(True)
    torch.cuda.synchronize()
    for i, (c, p) in enumerate(zip(clean, poisoned)):
        assert torch.isfinite(c.float()).all()
        assert torch.equal(c.view(torch.int16), p.view(torch.int16)), f"{entry}: output {i} of the victim changed"
    if entry in ("tn", "tn_pair"):
        for z in poisoned[-2:] if entry == "tn_pair" else poisoned[1:]:
            assert not z.view(torch.int16).any(), "an empty expert's dW must be exactly zero"


# ---- F: ops.group_gemm shape checks ----------------------------------------------------------------------------------------


def test_ops_group_gemm_rejects_inconsistent_shapes_before_launching():
    from xtuner_b200 import ops
    from xtuner_b200._capi import XtbError

    lib = ensure_init()
    bf = dict(dtype=torch.bfloat16, device="cuda")
    x = torch.randn(300, 256, **bf)
    w = torch.randn(4, 128, 256, **bf)
    tpe = _tpe([100, 0, 150, 50])
    ops.group_gemm(x, w, tpe)  # consistent: runs
    torch.cuda.synchronize()
    bad = {
        "weights not 3-D": (x, w[0], tpe),
        "x.shape[1] != weights.shape[2]": (torch.randn(300, 384, **bf), w, tpe),
        "x not 2-D": (x.view(300, 2, 128), w, tpe),
        "fewer split sizes than experts": (x, w, tpe[:3]),
        "more split sizes than experts": (x, w, _tpe([100, 0, 150, 50, 0])),
        "split sizes not 1-D": (x, w, tpe.view(2, 2)),
        "zero rows, x.shape[1] != weights.shape[2]": (torch.empty(0, 384, **bf), w, tpe),
    }
    for what, args in bad.items():
        before = lib.xtb_launch_count()
        with pytest.raises(XtbError):
            ops.group_gemm(*args)
        assert lib.xtb_launch_count() == before, what
