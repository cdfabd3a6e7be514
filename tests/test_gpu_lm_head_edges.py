"""The lm_head kernels (csrc/lm_head_ce.cu and the EPI_CE epilogue of csrc/group_gemm.cu) against float64 formulas
(tests/lm_head_ce_reference.py) and exact restatements, at the vocabulary sizes people train with and at their edges.

* Vocabulary matrix: V from one 128- or 256-column tile to the DeepSeek-V3 (129 280, H 7168) and Qwen3 (151 936, H 2048)
  heads, each V reaching another path of ``row_max_sum`` (one or two passes of its strided loops over the tile pairs)
  and of ``grad_row_in_place`` (chunk slots u = 0..3, one or more 4 x 256-chunk passes, a partial last pass).
* Row and width tails: T from 1 to 129 (16-row store boxes ragged in either 8-row half, 128-row tiles one short or one
  over), H = 128 (one k-block) and 2048, both tile widths.
  Each case of these two groups checks, on the kernel's own bf16 logits z:
  - z itself with exact-mode operands: bf16(fp64) bit for bit (``tests/gemm_reference.py``);
  - every per-tile pair (max, sum exp(z - max)) of the workspace: max bit-equal, sum within width * 2^-23 relative;
  - per-row CE, logp and the row statistics' log-sum within 1e-6 relative to max(1, |value|); the max bit-equal;
  - the loss within LOSS_REL of sum |ce64 * w| (see below);
  - every element of G, of the CE entry and of the logprob backward, within 1 bf16 ulp of bf16(fp64), and at most
    0.1 % of them (plus 4, for cases of a few hundred elements) not exact.  The fp32 path (expf of the fp32
    log-softmax, times w) errs by about 1e-7..1e-6 relative, while bf16's rounding boundaries are 2^-8 relative apart:
    an element rounds to the other side only when it lies that close to a boundary, a share of order 1e-4 (the printed
    shares are the measured ones);
  - dh and dW of both entries bit-equal to xtb_group_gemm_nn / _tn called on the entry's own G.
* Long reductions, exact: the NN product over K = V = 151 936 and 129 280 and the TN product over 16 384 and 32 768 rows
  into [151 936, 2048], with exact-mode operands (integers in [-4, 4] times a power of two; partial sums stay below
  16 * 151 936 < 2^22 units, so an fp32 accumulator is exact in any order): bf16(fp64) bit for bit.
* Labels and weights: ignore_index -100, -1, 0 and V-1; a negative label that is not ignore_index (NaN in that row of
  the CE entry only, clipped to 0 by the logprob entries); label V-1 in the last column of either tile width; loss
  weights 0, negative and 1e30; an ignored row with a NaN weight (NaN loss, as ``(ce * lw).sum()``); grad_logp of 0,
  negative and NaN in one row.
* Non-finite isolation: NaN in one row of h stays in that row (every other row bit-identical to the finite run); NaN in
  one row of W makes every counted row NaN and leaves ignored rows at CE 0 and G exactly 0; an all-zero h row (every
  logit ties across every tile); logits ~1e4 with one dominant tile, so every other tile's rescale factor underflows.
* Zero rows: the raw entries with T = 0 write only what their contract says; ``ops.lm_head_cross_entropy`` gives the
  reference's zero loss, empty dh and zero dW without calling the entry.

Every output is written into a view with 16 guard rows on each side (the workspace: 16 pairs after its T * n_vt pairs),
pre-filled with a NaN pattern no kernel produces: the guards must keep the fill and no output element may keep it.  Each
quantity's worst |err| / bound and each V's exact share of G are printed at the end of the module."""
import contextlib
import math

import pytest
import torch

from tests import gemm_reference as R
from tests.gpu_harness import FILL32, GUARD, Guarded, Worst
from tests.lm_head_ce_reference import grad64, lm_head_ce, logp64, logprob_grad64, row_ce64, row_stats64
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu

DEV = "cuda"
IGN = -100
WS_HEADER = 256  # bytes of the workspace ahead of its tile pairs
REL = 1e-6  # CE, logp and log-sum: relative to max(1, |value|)
# the loss: each row's CE within REL, the products rounded once, and an fp32 sum of at most 40 dependent adds (one term
# per thread below 1024 rows, a 5-level warp butterfly, 32 warp results in order)
LOSS_REL = REL + 40 * 2.0 ** -24
WORST = Worst("lm_head_edges")
SHARE = {}  # case -> exact share of G


@contextlib.contextmanager
def _shares():
    yield
    for k, v in SHARE.items():
        print(f"lm_head_edges: G exact share {k}: {v:.6f}")


_report = WORST.fixture(_shares)


def _workspace(T, V):
    """int32 workspace of xtb_lm_head_ce_workspace_bytes(T, V) bytes plus 16 guard pairs, all filled"""
    n = int(ensure_init().xtb_lm_head_ce_workspace_bytes(T, V))
    assert n % 8 == 0
    return n, torch.full((n // 4 + 2 * GUARD,), FILL32, dtype=torch.int32, device=DEV)


def _width(V):
    return 256 if V % 256 == 0 else 128


def _pairs(ws, T, V):
    n_vt = V // _width(V)
    return ws[WS_HEADER // 4:WS_HEADER // 4 + 2 * T * n_vt].view(torch.float32).view(T, n_vt, 2)


def _check_ws(n, ws, T, V, what):
    assert bool((ws[n // 4:] == FILL32).all()), f"{what}: written past the workspace's {T} x {V // _width(V)} pairs"
    if T:
        assert n == WS_HEADER + 8 * T * (V // _width(V))
        assert not bool((_pairs(ws, T, V).view(torch.int32) == FILL32).any()), f"{what}: a tile pair was never written"


class Out:
    pass


def ce(h, w, lab, lw, need_grad, ignore=IGN):
    """one xtb_lm_head_ce call into guarded buffers (guards checked) -> Out with z (z or G), ce, loss, dh, dw, pairs"""
    T, H = h.shape
    V = w.shape[0]
    o = Out()
    z, c, l = Guarded(T, V, torch.bfloat16), Guarded(T, 1, torch.float32), Guarded(1, 1, torch.float32)
    dh, dw = (Guarded(T, H, torch.bfloat16), Guarded(V, H, torch.bfloat16)) if need_grad else (None, None)
    n, ws = _workspace(T, V)
    check(ensure_init().xtb_lm_head_ce(ptr(h), ptr(w), ptr(lab), ptr(lw), T, H, V, ignore, int(need_grad), ptr(z.v),
                                       ptr(ws), ptr(c.v), ptr(l.v), ptr(dh.v) if need_grad else None,
                                       ptr(dw.v) if need_grad else None, current_stream()), "xtb_lm_head_ce")
    torch.cuda.synchronize()
    o.z, o.ce, o.loss = z.check("z / G"), c.check("row_ce")[:, 0], l.check("loss")[0, 0]
    o.dh, o.dw = (dh.check("dh"), dw.check("dW")) if need_grad else (None, None)
    _check_ws(n, ws, T, V, "xtb_lm_head_ce workspace")
    o.pairs = _pairs(ws, T, V)
    return o


def logprob(h, w, lab):
    """one xtb_lm_head_logprob call -> Out with z, logp, rs, pairs"""
    T, H = h.shape
    V = w.shape[0]
    o = Out()
    z, lp, rs = Guarded(T, V, torch.bfloat16), Guarded(T, 1, torch.float32), Guarded(T, 2, torch.float32)
    n, ws = _workspace(T, V)
    check(ensure_init().xtb_lm_head_logprob(ptr(h), ptr(w), ptr(lab), T, H, V, ptr(z.v), ptr(ws), ptr(lp.v), ptr(rs.v),
                                            current_stream()), "xtb_lm_head_logprob")
    torch.cuda.synchronize()
    o.z, o.logp, o.rs = z.check("logprob z"), lp.check("logp")[:, 0], rs.check("row_stats")
    _check_ws(n, ws, T, V, "xtb_lm_head_logprob workspace")
    o.pairs = _pairs(ws, T, V)
    return o


def logprob_bwd(z, rs, lab, c, h, w):
    """one xtb_lm_head_logprob_bwd call over z (a guarded view, overwritten with G) -> (dh, dW)"""
    T, H = h.shape
    V = w.shape[0]
    dh, dw = Guarded(T, H, torch.bfloat16), Guarded(V, H, torch.bfloat16)
    n, ws = _workspace(0, V)
    check(ensure_init().xtb_lm_head_logprob_bwd(ptr(z), ptr(rs), ptr(lab), ptr(c), ptr(h), ptr(w), T, H, V, ptr(ws),
                                                ptr(dh.v), ptr(dw.v), current_stream()), "xtb_lm_head_logprob_bwd")
    torch.cuda.synchronize()
    assert bool((ws[n // 4:] == FILL32).all()), "logprob_bwd: written past the workspace"
    return dh.check("logprob dh"), dw.check("logprob dW")


def gemm(kind, a, b, T):
    """xtb_group_gemm_nn (a = G [T, V], b = w [V, H] -> [T, H]) or _tn (a = G, b = h [T, H] -> [V, H]), one group"""
    V, H = a.shape[1], b.shape[1]
    tpe = torch.tensor([T], dtype=torch.int64, device=DEV)
    out = Guarded(T if kind == "nn" else V, H, torch.bfloat16)
    f = ensure_init().xtb_group_gemm_nn if kind == "nn" else ensure_init().xtb_group_gemm_tn
    check(f(ptr(a), ptr(b), ptr(tpe), T, V, H, 1, ptr(out.v), current_stream()), f"xtb_group_gemm_{kind}")
    torch.cuda.synchronize()
    return out.check(f"{kind} output")


def _labels(T, V, seed, ignored=0.3, ign=IGN):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lab = torch.randint(0, V, (T,), generator=g, device=DEV)
    lab[torch.rand(T, generator=g, device=DEV) < ignored] = ign
    if T > 3:
        lab[1], lab[2] = 0, V - 1
    return lab


def _random(T, H, V, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = (torch.randn(T, H, generator=g, device=DEV) * scale).to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device=DEV) * H ** -0.5).to(torch.bfloat16)
    return h, w


# ---- checks against float64 ------------------------------------------------------------------------------------------


def _rel(got, want, name, rows=None):
    """asserts |got - want| <= REL * max(1, |want|) on ``rows`` (all if None)"""
    if rows is not None:
        got, want = got[rows], want[rows]
    r = ((got.double() - want).abs() / want.abs().clamp_min(1.0)).nan_to_num(math.inf) / REL
    if r.numel():
        WORST.note(name, r.max())
        assert float(r.max()) <= 1.0, f"{name}: error {float(r.max()) * REL:.3g} relative, row {int(r.argmax())}"


def _ulp(G, g64, name, share_key=None, rows=None):
    """every element within 1 bf16 ulp of bf16(g64); at most 0.1 % of them, plus 4 for the cases of a few hundred
    elements (where one element is already more than 0.1 %), off by that ulp"""
    if rows is not None:
        G, g64 = G[rows], g64[rows]
    d = R.ulp_distance(G, R.bf16_rn(g64))
    share = (d == 0).double().mean().item()
    WORST.note(f"{name} max ulp (bound 1)", d.max())
    if share_key is not None:
        SHARE[share_key] = min(share, SHARE.get(share_key, 1.0))
    assert int(d.max()) <= 1, f"{name}: {int((d > 1).sum())} elements more than 1 ulp from bf16(fp64)"
    assert int((d != 0).sum()) <= 1e-3 * d.numel() + 4, f"{name}: exact share {share:.6f} of {d.numel()} elements"


def _check_pairs(pairs, z, what):
    """per row and vocab tile: max bit-equal to the tile's max, sum exp(z - max) within width * 2^-23 relative"""
    T, V = z.shape
    zt = z.double().view(T, V // _width(V), _width(V))
    m = zt.amax(2)
    assert torch.equal(pairs[..., 0].double(), m), f"{what}: a tile max differs"
    s = torch.exp(zt - m[..., None]).sum(2)
    r = (pairs[..., 1].double() - s).abs() / (s * _width(V) * 2.0 ** -23)
    WORST.note("tile sum exp / bound", r.max())
    assert float(r.max()) <= 1.0, f"{what}: tile sum off by {float(r.max())} x its bound"


def _check_loss(loss, ce64, lw, name="loss / bound"):
    prod = ce64 * lw.double()
    r = abs(loss.item() - prod.sum().item()) / (LOSS_REL * prod.abs().sum().item())
    WORST.note(name, r)
    assert r <= 1.0, f"loss {loss.item()!r} against fp64 {prod.sum().item()!r}"


def _check_ce_entry(h, w, lab, lw, key=None, ignore=IGN):
    """need_grad 0 then 1: z, CE, loss and G against fp64 on the kernel's own z -> (z, Out of the grad call)"""
    T = h.shape[0]
    o0 = ce(h, w, lab, lw, False, ignore)
    z = o0.z.clone()
    _check_pairs(o0.pairs, z, "xtb_lm_head_ce pairs")
    o = ce(h, w, lab, lw, True, ignore)
    assert torch.equal(o.ce, o0.ce) and torch.equal(o.loss, o0.loss)
    keep = lab != ignore
    ce64 = row_ce64(z, lab, ignore)
    assert bool((o.ce[~keep] == 0).all()) and bool((o.z[~keep] == 0).all())
    _rel(o.ce, ce64, "CE rel / 1e-6", keep)
    _check_loss(o.loss, ce64, lw)
    _ulp(o.z, grad64(z, lab, lw, ignore), "G (CE)", key)
    assert torch.equal(o.dh, gemm("nn", o.z, w, T)) and torch.equal(o.dw, gemm("tn", o.z, h, T)), \
        "dh / dW differ from the NN / TN GEMMs on the entry's own G"
    return z, o


def _check_logprob(h, w, lab, c, z_ce=None, key=None):
    """forward: logp and row stats against fp64; backward: G against fp64 and dh / dW against the GEMMs on it"""
    T = h.shape[0]
    o = logprob(h, w, lab)
    z = o.z.clone()
    if z_ce is not None:
        assert torch.equal(z, z_ce), "the two entries' logits differ"
    _check_pairs(o.pairs, z, "xtb_lm_head_logprob pairs")
    _rel(o.logp, logp64(z, lab), "logp rel / 1e-6")
    m64, ls64 = row_stats64(z)
    assert torch.equal(o.rs[:, 0].double(), m64), "row_stats max differs from the row's max"
    _rel(o.rs[:, 1], ls64, "row_stats log-sum rel / 1e-6")
    dh, dw = logprob_bwd(o.z, o.rs, lab, c, h, w)
    _ulp(o.z, logprob_grad64(z, lab, c), "G (logprob)", key)
    assert torch.equal(dh, gemm("nn", o.z, w, T)) and torch.equal(dw, gemm("tn", o.z, h, T)), \
        "logprob dh / dW differ from the NN / TN GEMMs on the entry's own G"
    return z, o, dh, dw


def _case(T, H, V, seed):
    # exact-mode logits
    he = R.rows_operand([T], H, "exact", seed=seed, device=DEV)
    we = R.weight_operand(1, V, H, "exact", seed=seed, device=DEV)
    o = ce(he, we[0], _labels(T, V, seed), torch.ones(T, device=DEV), False)
    R.assert_exact(o.z, "nt", he, we, [T], what=f"lm_head logits T={T} H={H} V={V}")
    del he, we, o
    # random-mode: everything from the kernel's own logits
    h, w = _random(T, H, V, seed)
    lab = _labels(T, V, seed)
    lw = torch.rand(T, device=DEV) + 0.5
    z, _ = _check_ce_entry(h, w, lab, lw, key=f"CE V={V}")
    _check_logprob(h, w, lab, torch.randn(T, device=DEV), z_ce=z, key=f"logprob V={V}")


# ---- 1. vocabulary matrix --------------------------------------------------------------------------------------------


VOCAB = [  # (V, H): tile width, n_vt tiles, n16 = V / 8 chunks of a row of G
    (128, 256),  # 128 x 1, 16: one tile
    (256, 256),  # 256 x 1, 32: one tile
    (2048, 256),  # 256 x 8, 256: slot u = 0 full
    (2176, 256),  # 128 x 17, 272: slot u = 1 partial
    (8192, 256),  # 256 x 32, 1024: one whole 4 x 256 pass
    (8320, 256),  # 128 x 65, 1040: second pass, 16 chunks
    (32896, 256),  # 128 x 257, 4112: row_max_sum's second pass
    (65536, 256),  # 256 x 256, 8192: 256 tile pairs, one per thread
    (65792, 256),  # 256 x 257, 8224: one pair over
    (129280, 7168),  # 256 x 505, 16160: the DeepSeek-V3 head
    (151936, 2048),  # 128 x 1187, 18992: the Qwen3 head
]


@pytest.mark.parametrize("V,H", VOCAB)
def test_vocabulary_matrix(V, H):
    _case(300, H, V, seed=V % 9973)


# ---- 2. row and width tails ------------------------------------------------------------------------------------------


@pytest.mark.parametrize("V", [128, 1152])
@pytest.mark.parametrize("H", [128, 2048])
@pytest.mark.parametrize("T", [1, 8, 9, 16, 17, 63, 64, 65, 127, 129])
def test_row_and_width_tails(T, H, V):
    _case(T, H, V, seed=T * 31 + H + V)


# ---- 3. long reductions, exact ---------------------------------------------------------------------------------------


@pytest.mark.parametrize("V,H", [(151936, 2048), (129280, 7168)])
def test_dh_product_over_the_whole_vocabulary_is_exact(V, H):
    T = 300
    G = R.rows_operand([T], V, "exact", seed=V % 997, device=DEV)
    w = R.weight_operand(1, V, H, "exact", seed=V % 991, device=DEV)
    dh = gemm("nn", G, w[0], T)
    R.assert_exact(dh, "nn", G, w, [T], what=f"NN K={V}")


@pytest.mark.parametrize("T", [16384, 32768])
def test_dw_product_over_long_row_counts_is_exact(T):
    V, H = 151936, 2048
    g = torch.Generator(device=DEV).manual_seed(T)
    G = torch.randint(-4, 5, (T, V), generator=g, device=DEV, dtype=torch.int8).to(torch.bfloat16).mul_(2.0 ** -3)
    h = torch.randint(-4, 5, (T, H), generator=g, device=DEV, dtype=torch.int8).to(torch.bfloat16).mul_(4.0)
    dw = gemm("tn", G, h, T)
    h64 = h.double()
    for v0 in range(0, V, 8192):  # the float64 reference in vocabulary slices
        want = R.bf16_rn(G[:, v0:v0 + 8192].double().T @ h64)
        bad = dw[v0:v0 + 8192] != want
        if bool(bad.any()):
            r, c = (int(i) for i in bad.nonzero()[0])
            raise AssertionError(f"TN over {T} rows: {int(bad.sum())} elements differ from bf16(fp64); first at "
                                 f"[{v0 + r}, {c}]: got {dw[v0 + r, c].item()!r}, want {want[r, c].item()!r}")


# ---- 4. labels and weights -------------------------------------------------------------------------------------------


@pytest.mark.parametrize("ignore", [-100, -1, 0, "V-1"])
def test_ignore_index(ignore):
    T, H, V = 300, 256, 1152
    ign = V - 1 if ignore == "V-1" else ignore
    h, w = _random(T, H, V, seed=41)
    lab = _labels(T, V, seed=41, ign=ign)
    lab[3:6] = torch.tensor([0, V - 1, ign], device=DEV)
    assert int((lab == ign).sum()) > 10
    _check_ce_entry(h, w, lab, torch.rand(T, device=DEV) + 0.5, ignore=ign)


def test_negative_label_that_is_not_ignored():
    T, H, V = 300, 256, 1152
    h, w = _random(T, H, V, seed=43)
    lab = _labels(T, V, seed=43)
    lab[10], lab[11] = -5, -1
    lw = torch.rand(T, device=DEV) + 0.5
    o = ce(h, w, lab, lw, True)
    bad = torch.zeros(T, dtype=torch.bool, device=DEV)
    bad[10:12] = True
    assert bool(o.ce[bad].isnan().all()) and bool(o.z[bad].float().isnan().all()) and bool(o.dh[bad].float().isnan().all())
    assert math.isnan(o.loss.item())
    # every other row as in a run where those two rows carry a valid label
    lab_ok = lab.clone()
    lab_ok[10], lab_ok[11] = 3, 4
    ok = ce(h, w, lab_ok, lw, True)
    assert torch.equal(o.ce[~bad], ok.ce[~bad]) and torch.equal(o.z[~bad], ok.z[~bad]) and torch.equal(o.dh[~bad], ok.dh[~bad])
    # the logprob entries clip it to 0
    _check_logprob(h, w, lab, torch.randn(T, device=DEV))


@pytest.mark.parametrize("V", [1024, 1152])  # the last column of a 256- and of a 128-column tile
def test_label_in_the_last_column(V):
    T, H = 64, 256
    h, w = _random(T, H, V, seed=V)
    lab = torch.full((T,), V - 1, dtype=torch.int64, device=DEV)
    z, _ = _check_ce_entry(h, w, lab, torch.rand(T, device=DEV) + 0.5)
    _check_logprob(h, w, lab, torch.randn(T, device=DEV), z_ce=z)


def test_loss_weights_zero_negative_and_huge():
    T, H, V = 300, 256, 1152
    h, w = _random(T, H, V, seed=47)
    lab = _labels(T, V, seed=47)
    # apart, so that the 1e30 rows do not swamp the bound of the others
    for pattern in ([0.0, -0.75, 1.5, -2.0, 0.25], [1e30, 1.0, -1e30, 0.0, 2.0]):
        _check_ce_entry(h, w, lab, torch.tensor(pattern, device=DEV).repeat(T // 5))


def test_ignored_row_with_a_nan_weight_gives_a_nan_loss():
    """as the reference's (ce * lw).sum(): the ignored row's CE is 0, and 0 * NaN is NaN"""
    T, H, V = 300, 256, 1152
    h, w = _random(T, H, V, seed=53)
    lab = _labels(T, V, seed=53)
    lw = torch.rand(T, device=DEV) + 0.5
    lab[7], lw[7] = IGN, float("nan")
    o = ce(h, w, lab, lw, True)
    assert math.isnan(o.loss.item()) and o.ce[7].item() == 0.0 and bool((o.z[7] == 0).all())
    keep = lab != IGN
    assert bool(torch.isfinite(o.ce).all()) and bool(torch.isfinite(o.z[keep].float()).all())


def test_grad_logp_zero_negative_and_nan():
    T, H, V = 300, 256, 1152
    h, w = _random(T, H, V, seed=59)
    lab = _labels(T, V, seed=59)
    c = torch.randn(T, device=DEV)
    c[3], c[4], c[5] = 0.0, -2.5, float("nan")
    o = logprob(h, w, lab)
    z = o.z.clone()
    dh, dw = logprob_bwd(o.z, o.rs, lab, c, h, w)
    rows = torch.ones(T, dtype=torch.bool, device=DEV)
    rows[5] = False
    _ulp(o.z, logprob_grad64(z, lab, c), "G (logprob)", rows=rows)
    assert bool((o.z[3] == 0).all()) and bool(o.z[5].float().isnan().all()) and bool(dh[5].float().isnan().all())
    assert bool(dw.float().isnan().all())  # every element of dW sums over row 5
    # every other row of dh as in a run where row 5's coefficient is finite
    o2 = logprob(h, w, lab)
    c2 = c.clone()
    c2[5] = 1.0
    dh2, _ = logprob_bwd(o2.z, o2.rs, lab, c2, h, w)
    assert torch.equal(dh[rows], dh2[rows])


# ---- 5. non-finite isolation -----------------------------------------------------------------------------------------


def test_nan_in_one_row_of_h_stays_in_that_row():
    T, H, V = 300, 256, 1152
    h, w = _random(T, H, V, seed=61)
    lab = _labels(T, V, seed=61)
    lab[7] = 5
    lw = torch.rand(T, device=DEV) + 0.5
    c = torch.randn(T, device=DEV)
    hn = h.clone()
    hn[7, 3] = float("nan")
    rows = torch.ones(T, dtype=torch.bool, device=DEV)
    rows[7] = False
    a, b = ce(h, w, lab, lw, True), ce(hn, w, lab, lw, True)
    for name in ("ce", "z", "dh"):
        x, y = getattr(a, name), getattr(b, name)
        assert bool(y[7].float().isnan().all()), f"CE entry: row 7 of {name} is not NaN"
        assert torch.equal(x[rows], y[rows]), f"CE entry: NaN in row 7 of h changed another row of {name}"
    pa, pb = logprob(h, w, lab), logprob(hn, w, lab)
    assert math.isnan(pb.logp[7].item()) and torch.equal(pa.logp[rows], pb.logp[rows])
    assert torch.equal(pa.rs[rows], pb.rs[rows])
    da, _ = logprob_bwd(pa.z, pa.rs, lab, c, h, w)
    db, _ = logprob_bwd(pb.z, pb.rs, lab, c, hn, w)
    assert bool(pb.z[7].float().isnan().all()) and bool(db[7].float().isnan().all())
    assert torch.equal(pa.z[rows], pb.z[rows]) and torch.equal(da[rows], db[rows])


def test_nan_in_one_row_of_w_spares_only_the_ignored_rows():
    """Every counted row's CE and G are NaN; an ignored row keeps CE 0 and G exactly 0 (the kernel never reads its
    logits).  Torch differs on purpose here: its log_softmax backward computes 0 - exp(NaN) * 0 on an ignored row and
    gives NaN there."""
    T, H, V = 300, 256, 1152
    h, w = _random(T, H, V, seed=67)
    w[100, 5] = float("nan")
    lab = _labels(T, V, seed=67)
    keep = lab != IGN
    o = ce(h, w, lab, torch.rand(T, device=DEV) + 0.5, True)
    assert bool(o.ce[keep].isnan().all()) and bool(o.z[keep].float().isnan().all())
    assert bool((o.ce[~keep] == 0).all()) and bool((o.z[~keep] == 0).all())
    assert math.isnan(o.loss.item())


@pytest.mark.parametrize("V,H", [(1152, 256), (151936, 2048)])
def test_all_zero_row_ties_across_every_tile(V, H):
    T = 64
    h, w = _random(T, H, V, seed=71)
    h[5], h[6] = 0, 0
    lab = _labels(T, V, seed=71)
    lab[5], lab[6] = 17, V - 1
    lw = torch.rand(T, device=DEV) + 0.5
    z, o = _check_ce_entry(h, w, lab, lw)
    assert bool((z[5:7] == 0).all())
    _rel(o.ce[5:7], torch.full((2,), math.log(V), dtype=torch.float64, device=DEV), "CE rel / 1e-6")
    want = R.bf16_rn(lw[5:7].double()[:, None] / V).expand(2, V).clone()  # G = bf16(w / V) off the label
    G = o.z[5:7].clone()
    G[0, 17], G[1, V - 1] = want[0, 0], want[1, 0]
    assert int(R.ulp_distance(G, want).max()) <= 1
    _, ol, _, _ = _check_logprob(h, w, lab, torch.randn(T, device=DEV), z_ce=z)
    _rel(ol.rs[5:7, 1], torch.full((2,), math.log(V), dtype=torch.float64, device=DEV), "row_stats log-sum rel / 1e-6")


def test_one_dominant_tile_underflows_every_other_tile():
    T, H, V = 64, 256, 8320  # 65 tiles of 128 columns
    h, w = _random(T, H, V, seed=73)
    h[:, 0] = 64.0
    g = torch.Generator(device=DEV).manual_seed(73)
    w[40 * 128:41 * 128, 0] = (150.0 + torch.randn(128, generator=g, device=DEV)).to(torch.bfloat16)
    lab = _labels(T, V, seed=73)
    lab[3:6] = torch.tensor([40 * 128 + 7, 41 * 128 - 1, 9], device=DEV)
    z, o = _check_ce_entry(h, w, lab, torch.rand(T, device=DEV) + 0.5)
    zd = z.float()
    assert float(zd.abs().max()) > 5e3
    other = torch.cat([zd[:, :40 * 128], zd[:, 41 * 128:]], 1)
    assert bool((other.amax(1) - zd.amax(1) < -200).all()), "the other tiles do not underflow"
    assert bool((o.pairs[:, 40, 0] == zd.amax(1)).all())
    _check_logprob(h, w, lab, torch.randn(T, device=DEV), z_ce=z)


# ---- 6. zero rows ----------------------------------------------------------------------------------------------------


def test_zero_rows_at_the_entries_write_only_their_contract():
    H, V = 256, 1024
    h, w = _random(1, H, V, seed=79)
    lab = torch.zeros(1, dtype=torch.int64, device=DEV)
    lw = torch.ones(1, device=DEV)
    lib = ensure_init()
    for need_grad in (1, 0):  # one row of every buffer, so that no pointer is NULL
        z, c, l = Guarded(1, V, torch.bfloat16), Guarded(1, 1, torch.float32), Guarded(1, 1, torch.float32)
        dh, dw = Guarded(1, H, torch.bfloat16), Guarded(V, H, torch.bfloat16)
        wsb = torch.full((1024,), FILL32, dtype=torch.int32, device=DEV)
        check(lib.xtb_lm_head_ce(ptr(h), ptr(w), ptr(lab), ptr(lw), 0, H, V, IGN, need_grad, ptr(z.v), ptr(wsb),
                                 ptr(c.v), ptr(l.v), ptr(dh.v), ptr(dw.v), current_stream()), "xtb_lm_head_ce")
        torch.cuda.synchronize()
        what = f"T = 0, need_grad {need_grad}"
        assert l.check(f"{what}: loss", written=None).view(torch.int32)[0, 0].item() == 0, "the loss is not +0"
        for g, name in ((z, "z"), (c, "row_ce"), (dh, "dh")):
            g.check(f"{what}: {name}", written=False)
        assert bool((wsb == FILL32).all()), f"{what}: workspace written"
        if need_grad:
            assert bool((dw.check(f"{what}: dW", written=None).view(torch.int16) == 0).all())
        else:
            dw.check(f"{what}: dW", written=False)
    z, lp, rs = Guarded(1, V, torch.bfloat16), Guarded(1, 1, torch.float32), Guarded(1, 2, torch.float32)
    wsb = torch.full((1024,), FILL32, dtype=torch.int32, device=DEV)
    check(lib.xtb_lm_head_logprob(ptr(h), ptr(w), ptr(lab), 0, H, V, ptr(z.v), ptr(wsb), ptr(lp.v), ptr(rs.v),
                                  current_stream()), "xtb_lm_head_logprob")
    torch.cuda.synchronize()
    for g, name in ((z, "z"), (lp, "logp"), (rs, "row_stats")):
        g.check(f"logprob T = 0: {name}", written=False)
    assert bool((wsb == FILL32).all()), "logprob T = 0: workspace written"
    dh, dw = Guarded(1, H, torch.bfloat16), Guarded(V, H, torch.bfloat16)
    check(lib.xtb_lm_head_logprob_bwd(ptr(z.v), ptr(rs.v), ptr(lab), ptr(lw), ptr(h), ptr(w), 0, H, V, ptr(wsb),
                                      ptr(dh.v), ptr(dw.v), current_stream()), "xtb_lm_head_logprob_bwd")
    torch.cuda.synchronize()
    for g, name in ((z, "z"), (rs, "row_stats"), (dh, "dh")):
        g.check(f"logprob_bwd T = 0: {name}", written=False)
    assert bool((wsb == FILL32).all()), "logprob_bwd T = 0: workspace written"
    assert bool((dw.check("logprob_bwd T = 0: dW", written=None).view(torch.int16) == 0).all())


@pytest.mark.parametrize("chunk", [None, 1024])
def test_zero_rows_through_the_op(chunk):
    from xtuner_b200 import ops

    H, V = 256, 1024
    _, w = _random(1, H, V, seed=83)
    h = torch.empty((0, H), dtype=torch.bfloat16, device=DEV)
    lab, lw = torch.empty((0,), dtype=torch.int64, device=DEV), torch.empty((0,), device=DEV)
    want = lm_head_ce(h, w, lab, lw, IGN, chunk)
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    loss = ops.lm_head_cross_entropy(hh, ww, lab, lw, IGN, chunk)
    loss.backward()
    assert torch.equal(loss.detach(), want[0]) and loss.item() == 0.0
    assert hh.grad.shape == (0, H) and torch.equal(ww.grad, want[2]) and ww.grad.count_nonzero() == 0
    with torch.no_grad():
        assert ops.lm_head_cross_entropy(h, w, lab, lw, IGN, chunk).item() == 0.0
