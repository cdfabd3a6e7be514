"""The checkers of tests/router_reference.py on the CPU: they accept correct emulations (fp32 sums in another order
included) and reject each planted mistake.  Also CPU models of the routers' arg-max rounds on NaN rows, which show the
duplicate-id fallback and the out-of-range id the kernels used to produce there (the fixed kernels are checked on the
GPU by tests/test_gpu_router_edges.py)."""
import pytest
import torch

from tests import router_reference as R

INT_MAX = 2**31 - 1


# ---- gate ------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("H", [128, 384, 2048])
def test_gate_onehot_is_exact_only_with_all_three_planes(H):
    x, w, _ = R.gate_inputs(3 * H, H, 8, "onehot", H, with_bias=False)
    ref, _ = R.gate_ref(x, w, None)
    assert torch.equal(R.emulate_gate_mma(x, w).double(), ref)
    # the lo plane dropped / w rounded to bf16: not exact
    assert not torch.equal(R.emulate_gate_mma(x, w, planes=2).double(), ref)
    assert not torch.equal(R.emulate_gate_mma(x, w, planes=1).double(), ref)
    hi, mid, lo = R.split3(w)
    assert torch.equal(hi.double() + mid.double() + lo.double(), w.double())
    assert bool((lo != 0).any())  # the lo plane carries bits on these inputs


@pytest.mark.parametrize("H", [128, 2048, 4224])
def test_gate_random_bound_accepts_fp32_and_rejects_bf16_weights(H):
    """A dropped lo plane moves a random-mode logit by about 2^-17 |w| sqrt(H), under the worst-case bound: only the
    one-hot mode (exact comparison) sees it."""
    x, w, b = R.gate_inputs(64, H, 8, "random", H)
    ref, S = R.gate_ref(x, w, b)
    bound = R.gate_bound("mma", H, S)
    got = R.emulate_gate_mma(x, w) + b
    assert R.check_bound(got, ref, bound) <= 1.0
    rev = (x.float().flip(1) @ w.flip(1).T) + b  # another fp32 order
    assert R.check_bound(rev, ref, bound) <= 1.0
    with pytest.raises(AssertionError):
        R.check_bound(x.float() @ w.to(torch.bfloat16).float().T + b, ref, bound)
    for k in ("small", "strided"):
        assert R.check_bound(got, ref, R.gate_bound(k, H, S)) <= 1.0


def test_gate_exact_mode_sums_are_exact():
    x, w, b = R.gate_inputs(64, 6656, 8, "exact", 1)
    ref, _ = R.gate_ref(x, w, b)
    assert torch.equal((x.float() @ w.T + b).double(), ref)
    assert torch.equal((x.float().flip(1) @ w.flip(1).T + b).double(), ref)


# ---- greedy router ---------------------------------------------------------------------------------------------------


def _route32(logits, K, scoring, norm, scaling):
    """fp32 emulation of the greedy router (torch's softmax / sigmoid, (value desc, index asc) rounds)."""
    rw = torch.softmax(logits, -1) if scoring == "softmax" else torch.sigmoid(logits)
    ids = R.topk_rounds(rw, K)
    tw = R.topk_weights_restated(rw, ids, norm, scaling)
    return rw, tw, ids, torch.bincount(ids.reshape(-1), minlength=logits.shape[1])


@pytest.mark.parametrize("scoring", ["softmax", "sigmoid"])
def test_greedy_checkers_accept_an_emulation_and_reject_planted_mistakes(scoring):
    T, E, K, scaling = 300, 64, 6, 2.5
    logits = torch.randn(T, E) * 3
    logits[0] = 1.0  # all equal
    logits[1, 7] = logits[1, 8] = 30.0  # a duplicate straddling lanes
    logits[2, 0] = logits[2, E - 1] = 30.0
    rw, tw, ids, tpe = _route32(logits, K, scoring, True, scaling)
    R.check_greedy_exact(rw, tw, ids, tpe, K, True, scaling)
    assert ids[0].tolist() == list(range(K)) and ids[1, :2].tolist() == [7, 8] and ids[2, :2].tolist() == [0, E - 1]
    p64, bound = R.greedy_ref(logits, scoring)
    assert R.check_bound(rw, p64, bound) <= 1.0
    dec = R.decided_rows(p64, bound, K)
    assert torch.equal(ids[dec], R.topk_rounds(p64, K)[dec])

    # ties resolved to the highest index
    hi_ids = ids.clone()
    hi_ids[0] = torch.arange(E - 1, E - 1 - K, -1)
    with pytest.raises(AssertionError):
        R.check_greedy_exact(rw, R.topk_weights_restated(rw, hi_ids, True, scaling), hi_ids,
                             torch.bincount(hi_ids.reshape(-1), minlength=E), K, True, scaling)
    # scaling applied before normalising
    sel = rw.gather(1, ids) * scaling
    bad_tw = sel / sel.sum(-1, keepdim=True)
    with pytest.raises(AssertionError):
        R.check_greedy_exact(rw, bad_tw, ids, tpe, K, True, scaling)
    # a miscounted histogram
    bad_tpe = tpe.clone()
    bad_tpe[0] += 1
    bad_tpe[1] -= 1
    with pytest.raises(AssertionError):
        R.check_greedy_exact(rw, tw, ids, bad_tpe, K, True, scaling)


def _greedy_bwd32(rw, tw, ids, g_tw, g_rw, scoring, norm, scaling, with_dot=True, softmax_sq=False):
    """fp32 restatement of router_greedy_bwd_kernel (one lane per token)."""
    gp = g_rw.clone() if g_rw is not None else torch.zeros_like(rw)
    if g_tw is not None:
        s = rw.gather(1, ids).sum(-1, keepdim=True)
        dot = (g_tw * (tw / scaling if scaling != 1.0 else tw)).sum(-1, keepdim=True) if with_dot else 0.0
        gv = scaling * (g_tw - dot) / s if norm else scaling * g_tw
        gp = gp.scatter_add(1, ids, gv)
    if scoring == "softmax":
        if softmax_sq:
            return gp * rw * rw
        d = (gp * rw).sum(-1, keepdim=True)
        return rw * (gp - d)
    return gp * rw * (1 - rw)


@pytest.mark.parametrize("scoring", ["softmax", "sigmoid"])
def test_greedy_bwd_bound_accepts_fp32_and_rejects_planted_mistakes(scoring):
    T, E, K, scaling = 200, 32, 4, 2.5
    logits = torch.randn(T, E) * 2
    g_tw, g_rw = torch.randn(T, K), torch.randn(T, E)
    rw, tw, ids, _ = _route32(logits, K, scoring, True, scaling)
    p64, _ = R.greedy_ref(logits, scoring)
    ref, ref_ids = R.greedy_bwd_ref(logits, K, scoring, True, scaling, g_tw, g_rw, None)
    dec = R.decided_rows(p64, R.greedy_ref(logits, scoring)[1], K)
    assert torch.equal(ids[dec], ref_ids[dec])
    bound = R.greedy_bwd_bound(p64, K, g_tw, g_rw, None, scaling, True)
    good = _greedy_bwd32(rw, tw, ids, g_tw, g_rw, scoring, True, scaling)
    assert R.check_bound(good[dec], ref[dec], bound[dec]) <= 1.0
    with pytest.raises(AssertionError):  # the dot term missing from the g_tw backward
        R.check_bound(_greedy_bwd32(rw, tw, ids, g_tw, g_rw, scoring, True, scaling, with_dot=False)[dec], ref[dec],
                      bound[dec])
    if scoring == "softmax":
        with pytest.raises(AssertionError):  # rw^2 in place of rw (g - d)
            R.check_bound(_greedy_bwd32(rw, tw, ids, g_tw, g_rw, scoring, True, scaling, softmax_sq=True)[dec],
                          ref[dec], bound[dec])


# ---- arg-max rounds on NaN rows --------------------------------------------------------------------------------------


def _rounds_model(p, K, fallback):
    """The kernels' K arg-max rounds over one row (plain Python floats; NaN never compares greater).  ``fallback``
    chooses the id of a round that finds no candidate: "k" (the old greedy fallback), "none" (the old no-aux kernel:
    the sentinel stays), "lowest_free" (the fix)."""
    taken, sel = set(), []
    for k in range(K):
        bv, be = -float("inf"), INT_MAX
        for j, v in enumerate(p):
            if j not in taken and v > bv:
                bv, be = v, j
        if not (0 <= be < len(p)):
            if fallback == "k":
                be = k
            elif fallback == "lowest_free":
                be = min(set(range(len(p))) - set(sel))
        taken.add(be)
        sel.append(be)
    return sel


def test_nan_row_fallbacks():
    nan = float("nan")
    sig = [nan, 1 / (1 + torch.exp(torch.tensor(-5.0)).item()), nan, nan]  # sigmoid of [NaN, 5, NaN, NaN]
    assert _rounds_model(sig, 2, "k") == [1, 1]  # the old greedy fallback repeats expert 1
    assert _rounds_model(sig, 2, "lowest_free") == [1, 0]
    assert _rounds_model([nan] * 8, 3, "none") == [INT_MAX] * 3  # the old no-aux kernel: an out-of-range id
    for row, K in [([nan] * 8, 8), ([nan, 0.3, nan, 0.1, nan, nan, nan, nan], 5), ([float("-inf"), nan, 2.0], 3)]:
        sel = _rounds_model(row, K, "lowest_free")
        assert len(set(sel)) == K and all(0 <= e < len(row) for e in sel), sel
