"""Lane-level model of ``router_noaux_bwd_kernel<LPT, VPL>`` (csrc/route.cu): LPT lanes per token, each holding VPL
consecutive experts, xor-shuffle reductions for the row sums, the group mask recomputed from the choice scores
(``noaux_kept_experts``: per-lane top-2, xor merges across the lanes of a group, topk_group butterfly arg-max rounds),
the top-k gradient scattered by id.  Restates the kernel's per-lane arithmetic and checks it against the reference-made
gradient fixture.  ``noaux_kept_experts`` is also the forward's group mask (``router_noaux_kernel`` calls it with
LPT = 32, VPL = E / 32), so its model is checked against the oracle's group choice under both lane mappings, on rows
where whole groups score -inf too.  The kernels themselves are covered on the GPU by tests/test_gpu_router.py and
tests/test_gpu_router_edges.py."""
import numpy as np
import pytest
import torch

from tests.conftest import load_golden


def top2_insert(a, b, v):
    if v > a:
        return v, a
    if v > b:
        return a, v
    return a, b


def kept_lane_model(ch, n_group, topk_group, LPT, VPL):
    """``noaux_kept_experts<LPT, VPL>`` for one token: ``ch`` float32 [E] -> bool [E].  The backward's group mask at
    ``dispatch(E)``, the forward's at ``(32, E // 32)``.  With LPT = 32 (the forward, and the backward at E = 256 and
    512) the kernel takes its one-candidate-per-lane path; otherwise the slot loop."""
    E = ch.shape[0]
    f32 = np.float32
    gs = E // n_group
    ninf = f32(-np.inf)
    if LPT == 32:  # one candidate per lane: the lane's group g, scored on the group's first lane
        assert VPL == E // 32 and gs % VPL == 0
        a = np.full(LPT, ninf, f32)
        b = np.full(LPT, ninf, f32)
        for sub in range(LPT):
            for j in range(VPL):
                a[sub], b[sub] = top2_insert(a[sub], b[sub], ch[sub * VPL + j])
        o = 1
        while o < gs // VPL:
            oa, ob = a[np.arange(LPT) ^ o], b[np.arange(LPT) ^ o]
            a, b = np.maximum(a, oa), np.maximum(np.minimum(a, oa), np.maximum(b, ob))
            o *= 2
        gv = (a + b).astype(f32)
        grp = np.arange(LPT) * VPL // gs
        cand = np.arange(LPT) * VPL % gs == 0
        kept = set()
        for _ in range(topk_group):
            ok = cand & ~np.isin(grp, list(kept)) & (gv >= ninf)
            bv = np.where(ok, gv, ninf).astype(f32)
            bi = np.where(ok, grp, 2**31 - 1).astype(np.int64)
            o = 16
            while o > 0:
                ov, oi = bv[np.arange(LPT) ^ o], bi[np.arange(LPT) ^ o]
                take = (ov > bv) | ((ov == bv) & (oi < bi))
                bv, bi = np.where(take, ov, bv), np.where(take, oi, bi)
                o //= 2
            assert (bi == bi[0]).all()
            if bi[0] < n_group:
                kept.add(int(bi[0]))
        return np.array([(e // gs) in kept for e in range(E)])
    gv = np.full((LPT, VPL), ninf, f32)
    cand = np.zeros((LPT, VPL), bool)
    a = np.full(LPT, ninf, f32)
    b = np.full(LPT, ninf, f32)
    for sub in range(LPT):
        for j in range(VPL):
            a[sub], b[sub] = top2_insert(a[sub], b[sub], ch[sub * VPL + j])
            if gs <= VPL and (j + 1) % gs == 0:
                gv[sub, j] = f32(a[sub] + b[sub])
                cand[sub, j] = True
                a[sub] = b[sub] = ninf
    if gs > VPL:
        o = 1
        while o < gs // VPL:
            oa, ob = a[np.arange(LPT) ^ o], b[np.arange(LPT) ^ o]
            a, b = np.maximum(a, oa), np.maximum(np.minimum(a, oa), np.maximum(b, ob))
            o *= 2
        for sub in range(LPT):
            gv[sub, VPL - 1] = f32(a[sub] + b[sub])
            cand[sub, VPL - 1] = (sub * VPL) % gs == 0
    kept = set()
    for _ in range(topk_group):
        bv = np.full(LPT, ninf, f32)
        bi = np.full(LPT, 2**31 - 1, np.int64)
        for sub in range(LPT):
            for j in range(VPL):
                gi = (sub * VPL + j) // gs
                if cand[sub, j] and gi not in kept and (gv[sub, j] > bv[sub] or (gv[sub, j] == bv[sub] and gi < bi[sub])):
                    bv[sub], bi[sub] = gv[sub, j], gi
        o = LPT // 2
        while o > 0:
            ov, oi = bv[np.arange(LPT) ^ o], bi[np.arange(LPT) ^ o]
            take = (ov > bv) | ((ov == bv) & (oi < bi))
            bv, bi = np.where(take, ov, bv), np.where(take, oi, bi)
            o //= 2
        assert (bi == bi[0]).all()  # every lane of the token agrees
        kept.add(int(bi[0]))
    return np.array([(e // gs) in kept for e in range(E)])


def lane_model(logits, bias, rw, tw, ids, g_tw, g_rw, n_group, topk_group, norm_topk, scaling, LPT, VPL):
    T, E = logits.shape
    K = ids.shape[1]
    out = np.zeros((T, E), np.float32)
    f32 = np.float32
    for tok in range(T):
        lanes = []
        for sub in range(LPT):
            e0 = sub * VPL
            sg = np.zeros(VPL, f32)
            for j in range(VPL):
                x = logits[tok, e0 + j] if e0 + j < E else f32(0)
                sg[j] = f32(1) / (f32(1) + np.exp(-x, dtype=f32))
            lanes.append(dict(e0=e0, sg=sg, ds=np.zeros(VPL, f32)))
        if g_rw is not None:
            if n_group != topk_group:
                ch = np.concatenate([ln["sg"] for ln in lanes]) + bias.astype(f32)
                kept = kept_lane_model(ch.astype(f32), n_group, topk_group, LPT, VPL)
            else:
                kept = np.ones(E, bool)
            S = np.zeros(LPT, f32)
            dot = np.zeros(LPT, f32)
            for sub, ln in enumerate(lanes):
                ln["g"] = np.zeros(VPL, f32)
                ln["keep"] = np.zeros(VPL, bool)
                for j in range(VPL):
                    e = ln["e0"] + j
                    r = rw[tok, e] if e < E else f32(0)
                    ln["g"][j] = g_rw[tok, e] if e < E else f32(0)
                    ln["keep"][j] = (e < E) and kept[e]
                    if ln["keep"][j]:
                        S[sub] += ln["sg"][j] + bias[e]
                    dot[sub] = f32(ln["g"][j] * r + dot[sub])
            o = LPT // 2
            while o > 0:  # butterfly: every lane ends with the full sum
                S = S + S[np.arange(LPT) ^ o]
                dot = dot + dot[np.arange(LPT) ^ o]
                o //= 2
            for sub, ln in enumerate(lanes):
                for j in range(VPL):
                    if ln["keep"][j]:
                        ln["ds"][j] = (ln["g"][j] - dot[sub]) / S[sub]
        if g_tw is not None:
            norm = K > 1 and norm_topk
            for sub, ln in enumerate(lanes):  # every lane recomputes D and gw from all K ids (no shuffles)
                D = f32(0)
                gw = f32(0)
                if norm:
                    for k in range(K):
                        x = logits[tok, ids[tok, k]]
                        D += f32(1) / (f32(1) + np.exp(-x, dtype=f32))
                        gw = f32(g_tw[tok, k] * tw[tok, k] + gw)
                    D += f32(1e-20)
                for k in range(K):
                    i = int(ids[tok, k])
                    if ln["e0"] <= i < ln["e0"] + VPL:
                        gk = g_tw[tok, k]
                        v = (f32(scaling) * gk - gw) / D if norm else f32(scaling) * gk
                        ln["ds"][i - ln["e0"]] += v
        for ln in lanes:
            for j in range(VPL):
                e = ln["e0"] + j
                if e < E:
                    out[tok, e] = ln["ds"][j] * ln["sg"][j] * (f32(1) - ln["sg"][j])
    return out


def dispatch(E):  # XTB_ROUTER_DISPATCH of route.cu
    for lim, cfg in [(8, (1, 8)), (16, (2, 8)), (32, (4, 8)), (64, (8, 8)), (128, (16, 8)), (256, (32, 8)), (512, (32, 16))]:
        if E <= lim:
            return cfg
    raise ValueError(E)


@pytest.mark.parametrize("tag", ["grouped", "ungrouped", "nonorm"])
def test_noaux_bwd_lane_model(tag):
    g = load_golden("noaux_router_bwd")[tag]
    n = 12  # tokens (the model is a Python loop)
    a = lambda k: g[k][:n].numpy()
    LPT, VPL = dispatch(g["logits"].shape[1])
    common = (a("logits"), g["e_score_correction_bias"].numpy(), a("router_weights"), a("topk_weights"), a("topk_ids"))
    tail = (g["n_group"], g["topk_group"], g["norm_topk_prob"], g["router_scaling_factor"], LPT, VPL)
    with np.errstate(over="ignore"):
        both = lane_model(*common, a("grad_topk_weights"), a("grad_router_weights"), *tail)
        only_tw = lane_model(*common, a("grad_topk_weights"), None, *tail)
        only_rw = lane_model(*common, None, a("grad_router_weights"), *tail)
    np.testing.assert_allclose(both, a("grad_logits"), rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(only_tw, a("grad_logits_from_topk"), rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(only_rw, a("grad_logits_from_router_weights"), rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize("E,n_group,topk_group", [(32, 4, 2), (32, 16, 3), (64, 8, 3), (128, 32, 5), (256, 8, 4),
                                                  (256, 2, 1), (512, 16, 4), (512, 4, 3), (512, 32, 7)])
def test_kept_experts_lane_model_equals_the_forward_choice(E, n_group, topk_group):
    """The recomputed group mask, under the backward's lane mapping (groups inside one lane and groups spanning 2 to 32
    lanes) and under the forward's (one warp per token), equals the group choice of the forward: the oracle's mask,
    and the experts the forward's router_weights leave non-zero.  Rows include tied group scores (lowest group index
    first) and whole groups scoring -inf, down to every group: exactly topk_group groups are kept all the same, the
    groups above -inf first, then the lowest-index remaining ones."""
    from oracle import moe_oracle as O

    g = torch.Generator().manual_seed(E + n_group)
    T = 6
    logits = torch.randn(T, E, generator=g)
    logits[0] = 0.0  # every group ties
    logits[1, : E // 2] = logits[1, E // 2 :]  # the two halves' groups tie pairwise
    bias = torch.randn(E, generator=g) * 0.1
    ch = torch.sigmoid(logits) + bias
    ch[0] = 0.25
    gs = E // n_group
    ninf = ch[2:6].clone().view(4, n_group, gs)
    ninf[0, :-1] = -torch.inf  # only the last group above -inf
    ninf[1] = -torch.inf  # every group -inf
    ninf[2, 1::2] = -torch.inf  # every odd group -inf
    ninf[3, :, 1:] = -torch.inf  # one score per group above -inf: every group score is -inf
    ch = torch.cat([ch, ninf.view(4, E)])
    want = O.noaux_kept_experts(ch, n_group, topk_group)
    for LPT, VPL in (dispatch(E), (32, E // 32)):
        for t in range(ch.shape[0]):
            got = kept_lane_model(ch[t].numpy(), n_group, topk_group, LPT, VPL)
            assert (got == want[t].numpy()).all(), (LPT, VPL, t)
    kept_groups = want.view(-1, n_group, gs).all(-1)
    assert (kept_groups.sum(-1) == topk_group).all()
    assert torch.equal(kept_groups[0].nonzero().flatten(), torch.arange(topk_group))
    first = torch.arange(topk_group)
    assert torch.equal(kept_groups[6].nonzero().flatten(), torch.cat([first[:-1], torch.tensor([n_group - 1])]))
    assert torch.equal(kept_groups[7].nonzero().flatten(), first)
    assert torch.equal(kept_groups[9].nonzero().flatten(), first)
    fwd = O.noaux_router(logits[2:], bias, min(8, E // n_group * topk_group), n_group, topk_group, 1.0)
    assert torch.equal(fwd["router_weights"] != 0, want[2:6])


def test_zero_score_kept_expert_keeps_its_router_weight_gradient():
    """A kept expert whose choice score is exactly 0 (logit 0 gives sigmoid 0.5, bias -0.5): its router weight is 0,
    and autograd still gives it (g - dot) / S sigma'.  A mask read back from router_weights != 0 drops that gradient;
    the recomputed mask keeps it."""
    from oracle import moe_oracle as O

    E, NG, TG, K = 64, 8, 4, 4
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(2, E, generator=g)
    bias = torch.zeros(E)
    logits[:, 0:8] = 4.0  # group 0 is kept
    logits[:, 3] = 0.0
    bias[3] = -0.5
    lg = logits.clone().requires_grad_(True)
    r = O.noaux_router(lg, bias, K, NG, TG, 1.0)
    assert float(r["router_weights"][0, 3]) == 0.0 and bool((r["router_weights"][:, 0:8].sum(-1) > 0).all())
    g_rw = torch.randn(2, E, generator=g)
    (want,) = torch.autograd.grad(r["router_weights"], lg, g_rw)
    assert float(want[0, 3]) != 0.0
    rw, tw, ids = (r[k].detach() for k in ("router_weights", "topk_weights", "topk_ids"))
    got = O.noaux_router_bwd(logits, bias, rw, tw, ids, None, g_rw, True, 1.0, n_group=NG, topk_group=TG)
    torch.testing.assert_close(got, want, rtol=2e-5, atol=2e-6)
    LPT, VPL = dispatch(E)
    lane = lane_model(logits.numpy(), bias.numpy(), rw.numpy(), tw.numpy(), ids.numpy(), None, g_rw.numpy(), NG, TG,
                      True, 1.0, LPT, VPL)
    np.testing.assert_allclose(lane, want.numpy(), rtol=2e-5, atol=2e-6)

    # without the geometry the oracle would have to read the mask back from router_weights != 0: it refuses this row
    with pytest.raises(ValueError, match="exactly 0"):
        O.noaux_router_bwd(logits, bias, rw, tw, ids, None, g_rw, True, 1.0)
    # the closed form the backward used before: the group mask read back from router_weights != 0
    s = torch.sigmoid(logits)
    mask = rw != 0
    c = torch.where(mask, s + bias, torch.zeros_like(s))
    dot = (g_rw * rw).sum(-1, keepdim=True)
    old = torch.where(mask, (g_rw - dot) / c.sum(-1, keepdim=True), torch.zeros_like(s)) * s * (1 - s)
    assert float(old[0, 3]) == 0.0
    assert not torch.allclose(old, want, rtol=2e-5, atol=2e-6)
