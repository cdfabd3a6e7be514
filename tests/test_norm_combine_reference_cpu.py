"""The checkers of tests/norm_combine_reference.py on the CPU: they accept correct fp32 emulations whose row reductions
are summed in another order than the kernels', and each rejects a planted mutation of the rounding order or of the
data flow that the GPU edge tests (tests/test_gpu_norm_combine_edges.py) exist to catch."""
import pytest
import torch

from tests import norm_combine_reference as R

T, K, H = 203, 4, 256
HF = 0.7  # not a power of two: the rounding after the factor is not exact


def _trunc(t: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 by truncation instead of round-to-nearest."""
    return (t.float().contiguous().view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


def _combine_inputs(mode, seed=0, neg_frac=0.1):
    rmap, owner = R.row_map(T, K, seed, neg_frac)
    sc = R.token_scales(T, seed + 1)
    y = R.permuted_rows(owner, H, sc, mode, seed + 2)
    p = R.probs(T, K, mode, seed + 3)
    res = R.token_rows(sc, H, "random", seed + 4)
    return rmap, y, p, res


def _acc32(y, rmap, p):
    """The fp32 accumulator of combine before its first bf16 round."""
    m = rmap.view(T, K).long()
    acc = None
    for k in range(K):
        ok = (m[:, k] >= 0)[:, None]
        prod = torch.where(ok, y[m[:, k].clamp_min(0)].float() * p[:, k : k + 1], torch.zeros(1))
        acc = prod if acc is None else acc + prod
    return acc


def _combine_fma(y, rmap, p, hf):
    """Products fused into the adds (fma) instead of rounded to fp32 first."""
    m = rmap.view(T, K).long()
    acc = None
    for k in range(K):
        ok = (m[:, k] >= 0)[:, None]
        prod = torch.where(ok, y[m[:, k].clamp_min(0)].double() * p[:, k : k + 1].double(), torch.zeros(1, dtype=torch.float64))
        acc = prod.float() if acc is None else (acc.double() + prod).float()
    return (acc.to(torch.bfloat16).float() * hf).to(torch.bfloat16)


# ---- acceptance ----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("hf,with_p,with_res", [(1.0, True, False), (0.5, True, True), (HF, False, True), (HF, True, False), (1.5, True, True)])
def test_combine_restatement_within_fp64_bound(mode, hf, with_p, with_res):
    rmap, y, p, res = _combine_inputs(mode)
    p = p if with_p else None
    res = res if with_res else None
    out = R.combine(y, rmap, p, res, hf, K)
    assert not torch.isnan(out.float()).any(), "a row mapped to -1 leaked its NaN"
    ref, bnd = R.combine_ref(y, rmap, p, res, hf, K)
    assert R.check_bound(out, ref, bnd, "combine") <= 1.0


def test_combine_exact_mode_sum_is_exact():
    rmap, y, p, _ = _combine_inputs("exact")
    ref, _ = R.combine_ref(y, rmap, p, None, 1.0, K)
    # the fp32 sum is exact: bf16(acc) is the correctly rounded fp64 sum
    R.assert_bits_equal(R.combine(y, rmap, p, None, 1.0, K), ref.float().to(torch.bfloat16), "exact-mode combine")


def test_norm_forward_emulation_in_another_order_passes():
    h = R.norm_rows(64, H, 5)
    w = R.norm_weight(H, 6)
    gate_w = torch.randn(8, H, generator=torch.Generator().manual_seed(7)) * H ** -0.5
    hf = h.float()
    ss = hf.square().view(64, 32, H // 32).flip(1).sum(1).sum(-1)  # another fp32 order than the kernels'
    eps32 = torch.tensor(R.EPS, dtype=torch.float32)
    rstd = torch.rsqrt((ss / H + eps32).double()).float()
    assert R.check_bound(rstd, R.rstd_ref(h, R.EPS), R.rstd_rel(H) * R.rstd_ref(h, R.EPS), "rstd") <= 1.0
    x = R.rmsnorm_x(h, rstd, w)
    xr, xb = R.x_ref(h, R.EPS, w)
    R.check_near_tie(x, xr, xb, "x")
    assert bool((x[torch.arange(64) % 13 == 5] == 0).all())
    lg = (x.float().view(64, 1, 32, H // 32) * gate_w.view(1, 8, 32, H // 32)).sum(-1).flip(-1).sum(-1)
    lr, lb = R.logits_ref(x, gate_w)
    assert R.check_bound(lg, lr, lb, "logits") <= 1.0


def _bwd_inputs(seed=0, Tb=T):
    rmap, owner = R.row_map(Tb, K, seed)
    sc = R.token_scales(Tb, seed + 1, exp_range=(-4, 4))
    g_xp = R.permuted_rows(owner, H, sc, "random", seed + 2)
    gate = R.token_rows(sc, H, "random", seed + 3)
    h = R.norm_rows(Tb, H, seed + 4)
    rstd = R.rstd_ref(h, R.EPS).float()
    w = R.norm_weight(H, seed + 5)
    return rmap, g_xp, gate, h, rstd, w


def _g_h_emulation(g_x, h, rstd, w, c_power=2):
    wg = g_x.float() * w
    hf = h.float()
    dot = (wg * hf).flip(-1).sum(-1, keepdim=True)
    r = rstd[:, None]
    c = dot * r ** c_power / H if c_power == 2 else dot * r / H
    return ((wg - hf * c) * r).to(torch.bfloat16)


def _g_norm_w_emulation(g_x, h, rstd, n_cta=264, last_twice=False):
    terms = (g_x.float() * rstd[:, None]) * h.float()
    part = torch.zeros((n_cta, H))
    for t in reversed(range(h.shape[0])):
        part[t % n_cta] += terms[t]
    if last_twice:
        part[(h.shape[0] - 1) % n_cta] += terms[-1]
    return part.sum(0)


def test_dispatch_bwd_emulation_in_another_order_passes():
    rmap, g_xp, gate, h, rstd, w = _bwd_inputs()
    g_x = R.dispatch_gx(g_xp, rmap, gate, K)
    assert not torch.isnan(g_x.float()).any()
    ref, bnd = R.g_h_ref(g_x, h, rstd, w)
    worst, _ = R.check_near_tie(_g_h_emulation(g_x, h, rstd, w), ref, bnd, "g_h")
    assert worst <= 1.0
    gr, gb = R.g_norm_w_ref(g_x, h, rstd)
    assert R.check_bound(_g_norm_w_emulation(g_x, h, rstd), gr, gb, "g_norm_w") <= 1.0


def test_unpermute_bwd_emulation_passes():
    rmap, y, p, _ = _combine_inputs("random")
    g = R.token_rows(R.token_scales(T, 9), H, "random", 10)
    rows, written = R.act_grad(g, rmap, p, K, T * K)
    assert int(written.sum()) == int((rmap >= 0).sum())
    pg = (g.float()[:, None, :] * torch.where((rmap.view(T, K) >= 0)[:, :, None],
                                                y[rmap.view(T, K).long().clamp_min(0)].float(), torch.zeros(1))).sum(-1)
    ref, bnd = R.prob_grad_ref(g, y, rmap, K)
    assert R.check_bound(pg, ref, bnd, "prob_grad") <= 1.0


# ---- rejection -------------------------------------------------------------------------------------------------------


def test_rejects_hf_before_first_round():
    rmap, y, p, res = _combine_inputs("random")
    want = R.combine(y, rmap, p, res, HF, K)
    accf = _acc32(y, rmap, p)
    bad = ((accf * HF).to(torch.bfloat16).float() + res.float()).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(bad, want, "hf before the first round")


def test_rejects_residual_before_round():
    rmap, y, p, res = _combine_inputs("random")
    accf = _acc32(y, rmap, p)
    bad = (accf + res.float()).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(bad, R.combine(y, rmap, p, res, 1.0, K), "residual before the round")


def test_rejects_fma_products():
    rmap, y, p, _ = _combine_inputs("random", neg_frac=0.0)
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(_combine_fma(y, rmap, p, HF), R.combine(y, rmap, p, None, HF, K), "fma")


@pytest.mark.parametrize("mode", ["exact", "random"])
def test_rejects_dropped_row(mode):
    rmap, y, p, res = _combine_inputs(mode)
    dropped = rmap.clone().view(T, K)
    dropped[:, K - 1] = -1
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(R.combine(y, dropped.view(-1), p, res, HF, K), R.combine(y, rmap, p, res, HF, K), "combine")
    rm, g_xp, gate, h, rstd, w = _bwd_inputs()
    dr = rm.clone().view(T, K)
    dr[:, 1] = -1
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(R.dispatch_gx(g_xp, dr.view(-1), gate, K), R.dispatch_gx(g_xp, rm, gate, K), "g_x")
    g = R.token_rows(R.token_scales(T, 9), H, mode, 10)
    ref, bnd = R.prob_grad_ref(g, y, rmap, K)
    bad, _ = R.prob_grad_ref(g, y, dropped.view(-1), K)
    with pytest.raises(AssertionError, match="outside the bound"):
        R.check_bound(bad.float(), ref, bnd, "prob_grad")


def test_rejects_unrounded_g_x_before_gate_add():
    rmap, g_xp, gate, h, rstd, w = _bwd_inputs()
    m = rmap.view(T, K).long()
    acc = torch.zeros((T, H))
    for k in range(K):
        ok = (m[:, k] >= 0)[:, None]
        acc = torch.where(ok, acc + g_xp[m[:, k].clamp_min(0)].float(), acc)
    bad = (acc + gate.float()).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(bad, R.dispatch_gx(g_xp, rmap, gate, K), "g_x")


def test_rejects_c_with_rstd_instead_of_rstd_squared():
    rmap, g_xp, gate, h, rstd, w = _bwd_inputs()
    g_x = R.dispatch_gx(g_xp, rmap, gate, K)
    ref, bnd = R.g_h_ref(g_x, h, rstd, w)
    with pytest.raises(AssertionError, match="near tie"):
        R.check_near_tie(_g_h_emulation(g_x, h, rstd, w, c_power=1), ref, bnd, "g_h")


def test_rejects_last_token_counted_twice():
    Tb = 1057
    rmap, g_xp, gate, h, rstd, w = _bwd_inputs(seed=3, Tb=Tb)
    h = h.clone()
    h[-1] = (torch.randn(H, generator=torch.Generator().manual_seed(1)) * 64).to(torch.bfloat16)
    rstd = R.rstd_ref(h, R.EPS).float()
    rstd[-1] = 1.0  # the last row's terms are large next to the sum of the others
    g_x = R.dispatch_gx(g_xp, rmap, gate, K)
    ref, bnd = R.g_norm_w_ref(g_x, h, rstd)
    assert R.check_bound(_g_norm_w_emulation(g_x, h, rstd), ref, bnd, "g_norm_w") <= 1.0
    with pytest.raises(AssertionError, match="outside the bound"):
        R.check_bound(_g_norm_w_emulation(g_x, h, rstd, last_twice=True), ref, bnd, "g_norm_w")


def test_rejects_truncation():
    rmap, y, p, res = _combine_inputs("random")
    accf = _acc32(y, rmap, p)
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(_trunc(accf), R.combine(y, rmap, p, None, 1.0, K), "combine")
    g = R.token_rows(R.token_scales(T, 9), H, "random", 10)
    want, written = R.act_grad(g, rmap, p, K, T * K)
    tok = torch.arange(T * K) // K
    ok = rmap.long() >= 0
    bad = want.clone()
    bad[rmap.long()[ok]] = _trunc(g[tok[ok]].float() * p.reshape(-1)[ok][:, None])
    with pytest.raises(AssertionError, match="differ"):
        R.assert_bits_equal(bad[written], want[written], "act_grad")
    h = R.norm_rows(64, H, 5)
    w = R.norm_weight(H, 6)
    rstd = R.rstd_ref(h, R.EPS).float()
    xr, xb = R.x_ref(h, R.EPS, w)
    R.check_near_tie(R.rmsnorm_x(h, rstd, w), xr, xb, "x")
    with pytest.raises(AssertionError, match="near tie"):
        R.check_near_tie(_trunc((h.float() * rstd[:, None]) * w), xr, xb, "x")
    rm, g_xp, gate, hb, rs, wb = _bwd_inputs()
    g_x = R.dispatch_gx(g_xp, rm, gate, K)
    ref, bnd = R.g_h_ref(g_x, hb, rs, wb)
    wg = g_x.float() * wb
    c = (wg * hb.float()).sum(-1, keepdim=True) * rs[:, None] ** 2 / H
    with pytest.raises(AssertionError, match="near tie"):
        R.check_near_tie(_trunc((wg - hb.float() * c) * rs[:, None]), ref, bnd, "g_h")
