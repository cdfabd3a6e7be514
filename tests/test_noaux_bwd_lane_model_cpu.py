"""Lane-level model of ``router_noaux_bwd_kernel<LPT, VPL>`` (csrc/route.cu): LPT lanes per token, each holding VPL
consecutive experts, xor-shuffle reductions for the row sums, the group mask read back from ``router_weights != 0``, the
top-k gradient scattered by id.  Restates the kernel's per-lane arithmetic and checks it against the reference-made
gradient fixture — the kernel itself is covered on the GPU by tests/test_gpu_router.py (noaux backward vs the same fixture)."""
import numpy as np
import pytest
import torch

from tests.conftest import load_golden


def lane_model(logits, bias, rw, tw, ids, g_tw, g_rw, has_mask, norm_topk, scaling, LPT, VPL):
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
            S = np.zeros(LPT, f32)
            dot = np.zeros(LPT, f32)
            for sub, ln in enumerate(lanes):
                ln["g"] = np.zeros(VPL, f32)
                ln["keep"] = np.zeros(VPL, bool)
                for j in range(VPL):
                    e = ln["e0"] + j
                    r = rw[tok, e] if e < E else f32(0)
                    ln["g"][j] = g_rw[tok, e] if e < E else f32(0)
                    ln["keep"][j] = (e < E) and (not has_mask or r != 0)
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
    tail = (g["n_group"] != g["topk_group"], g["norm_topk_prob"], g["router_scaling_factor"], LPT, VPL)
    with np.errstate(over="ignore"):
        both = lane_model(*common, a("grad_topk_weights"), a("grad_router_weights"), *tail)
        only_tw = lane_model(*common, a("grad_topk_weights"), None, *tail)
        only_rw = lane_model(*common, None, a("grad_router_weights"), *tail)
    np.testing.assert_allclose(both, a("grad_logits"), rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(only_tw, a("grad_logits_from_topk"), rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(only_rw, a("grad_logits_from_router_weights"), rtol=2e-5, atol=2e-6)
