"""Golden vectors for routing replay (``tests/golden/router_replay.pt``), made on the CPU by the REFERENCE'S OWN routers
(imported through ``ref_shim``): ``GreedyRouter`` (module/router/greedy.py:64-98) and ``NoAuxRouter``
(module/router/noaux_router.py:78-150), each called with ``rollout_routed_experts``:

    python tests/golden/make_router_replay_golden.py

Per case: the fp32 logits [T, E], the router_weights (the same for every id pattern), the upstream gradient of
router_weights; per id pattern: the replayed ids (the router returns them as topk_ids), the upstream gradient of
topk_weights, the router's topk_weights and tokens_per_expert, and the logits gradient by the reference's autograd.
Cases (T = 8 tokens):

* GreedyRouter: softmax and sigmoid, with and without renormalisation, scaling 1.5; K = 1, 2, 8; E = 8 and 128.
* NoAuxRouter: E = 256, K = 8, scaling 2.5, with n_group 8 / topk_group 4 and with n_group == topk_group == 8; a random
  correction bias.

and for each, four id patterns:

* ``own``: the router's own top-k, columns reversed;
* ``dup``: random ids with duplicates in every third row;
* ``never``: ids the router would not choose (its K lowest scores; for NoAux with a group mask, experts of masked groups);
* ``slice``: the [:, 1, :] slice of a random int64 [T, 3, K] tensor (stored whole as ``<case>.slice.full``; the
  pattern's ids are ``full[:, 1, :]``).
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ref_shim.apply_cpu_patches()

from make_golden import save  # noqa: E402
import xtuner.v1.module.router.noaux_router as _nr  # noqa: E402
from xtuner.v1.module.router.greedy import GreedyRouter  # noqa: E402
from xtuner.v1.module.router.noaux_router import NoAuxRouter  # noqa: E402

_nr.get_device = lambda: "cpu"  # the bias buffer is created on get_device()

T = 8
PATTERNS = ("own", "dup", "never", "slice")


def greedy_cases():
    for scoring in ("softmax", "sigmoid"):
        for norm in (True, False):
            for E in (8, 128):
                for K in (1, 2, 8):
                    yield f"greedy.{scoring}.{'norm' if norm else 'raw'}.e{E}.k{K}", scoring, norm, E, K


def noaux_cases():
    yield "noaux.g8t4", 8, 4
    yield "noaux.g8t8", 8, 8


def id_patterns(g, own, scores, E, K, masked=None):
    """{pattern: (ids [T, K] int64, full [T, 3, K] or None)}"""
    out = {"own": (own.flip(1).contiguous(), None)}
    dup = torch.randint(0, E, (T, K), generator=g)
    dup[::3, 0] = dup[::3, -1]
    out["dup"] = (dup, None)
    if masked is not None:  # experts of masked groups: the router never picks them
        never = torch.stack([masked[t].nonzero().flatten()[:K] for t in range(T)])
    else:
        never = scores.argsort(1)[:, :K]
    out["never"] = (never.contiguous(), None)
    full = torch.randint(0, E, (T, 3, K), generator=g)
    out["slice"] = (full[:, 1, :], full)
    return out


def run(out, case, pat, router, logits, ids, g_tw, g_rw):
    """stores topk_weights, tokens_per_expert and grad_logits under ``<case>.<pat>``; router_weights (which do not depend
    on the ids) and topk_ids (the ids themselves) are checked and stored once per case / not at all"""
    lg = logits.clone().requires_grad_(True)
    r = router(lg, ids)
    ((r["topk_weights"] * g_tw).sum() + (r["router_weights"] * g_rw).sum()).backward()
    assert torch.equal(r["topk_ids"], ids)
    rw = out.setdefault(f"{case}.router_weights", r["router_weights"].detach().clone())
    assert torch.equal(rw, r["router_weights"])
    out[f"{case}.{pat}.topk_weights"] = r["topk_weights"].detach()
    out[f"{case}.{pat}.tokens_per_expert"] = r["topkens_per_expert"].detach()
    out[f"{case}.{pat}.grad_logits"] = lg.grad


def main():
    out = {"T": T}
    seed = 100
    for name, scoring, norm, E, K in greedy_cases():
        seed += 1
        g = torch.Generator().manual_seed(seed)
        router = GreedyRouter(n_routed_experts=E, num_experts_per_tok=K, norm_topk_prob=norm, scoring_func=scoring,
                              router_scaling_factor=1.5)
        logits = torch.randn(T, E, generator=g) * 2
        with torch.no_grad():
            own = router(logits.clone())["topk_ids"]
        out[f"{name}.logits"] = logits
        out[f"{name}.g_rw"] = torch.randn(T, E, generator=g)
        for pat, (ids, full) in id_patterns(g, own, logits, E, K).items():
            g_tw = torch.randn(T, K, generator=g)
            if full is None:
                out[f"{name}.{pat}.ids"] = ids
            else:  # the slice is taken again by the reader
                out[f"{name}.{pat}.full"] = full
            out[f"{name}.{pat}.g_tw"] = g_tw
            run(out, name, pat, router, logits, ids, g_tw, out[f"{name}.g_rw"])
    E, K = 256, 8
    for name, n_group, topk_group in noaux_cases():
        seed += 1
        g = torch.Generator().manual_seed(seed)
        router = NoAuxRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=2.5, scoring_func="sigmoid",
                             n_group=n_group, topk_group=topk_group, norm_topk_prob=True)
        with torch.no_grad():
            router.e_score_correction_bias.copy_(torch.randn(E, generator=g) * 0.1)
        logits = torch.randn(T, E, generator=g) * 2
        with torch.no_grad():
            r0 = router(logits.clone())
        # masked experts: router_weights is exactly 0 only for them or for s + b == 0 (not hit by random data)
        masked = r0["router_weights"] == 0 if n_group != topk_group else None
        out[f"{name}.logits"] = logits
        out[f"{name}.bias"] = router.e_score_correction_bias.detach().clone()
        out[f"{name}.g_rw"] = torch.randn(T, E, generator=g)
        scores = logits.sigmoid() + router.e_score_correction_bias
        for pat, (ids, full) in id_patterns(g, r0["topk_ids"], scores, E, K, masked).items():
            g_tw = torch.randn(T, K, generator=g)
            if full is None:
                out[f"{name}.{pat}.ids"] = ids
            else:  # the slice is taken again by the reader
                out[f"{name}.{pat}.full"] = full
            out[f"{name}.{pat}.g_tw"] = g_tw
            run(out, name, pat, router, logits, ids, g_tw, out[f"{name}.g_rw"])
    save("router_replay", out)


if __name__ == "__main__":
    main()
