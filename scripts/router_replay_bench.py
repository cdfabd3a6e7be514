"""Cost of routing replay (RL rollout-routed experts) against routing, timed in alternation with CUDA events after
warm-up, with the card name and power limit read in the same run:

  block      FusedMoEBlock forward + backward (fused.fused_moe_block: RMSNorm, gate, router, dispatch, grouped GEMMs,
             combine), routed against replayed, at C2 (T = 8192, H = 2048, I = 768, E = 8, K = 2) and at the Qwen3-30B-A3B
             MoE geometry (E = 128, K = 8).  The replayed ids are the node's own routing, so both arms do the same expert
             work and their outputs and gradients must be equal bit for bit (checked before timing).
  router     the router alone, forward + backward, at E = 128, K = 8, T = 8192: GreedyRouter routed, GreedyRouter
             replayed, and the reference's eager GreedyRouter replayed (greedy.py:64-98; from oracle/_ref).
  noaux      NoAuxRouter alone, forward + backward, routed and replayed, at the DeepSeek-V3 geometry (T = 16384,
             E = 256, K = 8, n_group = 8, topk_group = 4, scaling 2.5).

Prints one line per arm (ms per forward + backward, host dispatch included: median, min and max over the repeats; for
the router arms also the summed device time of their kernels, from torch.profiler in a run of its own) and a JSON line.  Needs a GPU;
the reference arm needs oracle/_ref (built by build()).

    python scripts/router_replay_bench.py [--repeats 7 --iters 20 --warmup 5] [--only block|router|noaux]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from lm_head_ce_bench import card  # noqa: E402

DEV = "cuda"


def time_arms(arms: dict, repeats: int, iters: int, warmup: int) -> dict:
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    times = {k: [] for k in arms}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(repeats):
        for name, fn in arms.items():  # alternate the arms within each repeat
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(iters):
                fn()
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) / iters)
    return {k: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)} for k, v in times.items()}


def kernel_us(arms: dict, iters: int) -> dict:
    """summed device time of the kernels one call launches, from torch.profiler in a run of its own"""
    out = {}
    for name, fn in arms.items():
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
        out[name] = sum(e.self_device_time_total for e in evs) / iters
    return out


def block_arms(T, H, I, E, K):
    from xtuner_b200 import fused

    g = torch.Generator(device=DEV).manual_seed(0)
    h = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16).requires_grad_(True)
    nw = (1 + 0.1 * torch.randn(H, generator=g, device=DEV)).requires_grad_(True)
    gw = (torch.randn(E, H, generator=g, device=DEV) * 0.02).requires_grad_(True)
    w13 = (torch.randn(E, 2 * I, H, generator=g, device=DEV) * 0.02).to(torch.bfloat16).requires_grad_(True)
    w2 = (torch.randn(E, H, I, generator=g, device=DEV) * 0.02).to(torch.bfloat16).requires_grad_(True)
    go = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    leaves = (h, nw, gw, w13, w2)
    with torch.no_grad():
        _, rr = fused.fused_moe_block(h, nw, 1e-6, gw, w13, w2, top_k=K)
    ids = rr["topk_ids"].clone()

    def arm(replay):
        def step():
            for t in leaves:
                t.grad = None
            out, _ = fused.fused_moe_block(h, nw, 1e-6, gw, w13, w2, top_k=K, rollout_routed_experts=replay)
            out.backward(go)
            return [out.detach()] + [t.grad for t in leaves]
        return step

    arms = {"routed": arm(None), "replayed": arm(ids)}
    a = [t.clone() for t in arms["routed"]()]
    b = arms["replayed"]()
    assert all(torch.equal(x, y) for x, y in zip(a, b)), "replaying the node's own routing changed its result"
    return arms


def router_arms(T, E, K):
    from xtuner_b200 import router

    g = torch.Generator(device=DEV).manual_seed(1)
    logits = torch.randn(T, E, generator=g, device=DEV).requires_grad_(True)
    ids = torch.randint(0, E, (T, 3, K), generator=g, device=DEV)[:, 1, :]  # the layer slice of an [S, L, K] tensor
    g_tw = torch.randn(T, K, generator=g, device=DEV)
    g_rw = torch.randn(T, E, generator=g, device=DEV)

    def arm(r, replay):
        def step():
            logits.grad = None
            res = r(logits, replay)
            torch.autograd.backward((res["topk_weights"], res["router_weights"]), (g_tw, g_rw))
            return res["topk_weights"].detach(), logits.grad
        return step

    ours = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K)
    arms = {"ours_routed": arm(ours, None), "ours_replayed": arm(ours, ids)}
    from tests.golden import ref_shim

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    if ref_shim.reference_available():
        ref_shim.import_reference()
        from xtuner.v1.module.router.greedy import GreedyRouter

        ref = GreedyRouter(n_routed_experts=E, num_experts_per_tok=K)
        arms["ref_eager_replayed"] = arm(ref, ids)
        a = [t.clone() for t in arms["ours_replayed"]()]
        b = arms["ref_eager_replayed"]()
        for x, y, n in zip(a, b, ("topk_weights", "grad_logits")):
            rel = float((x - y).abs().max() / y.abs().max().clamp_min(1e-30))
            assert rel <= 1e-4, f"ours vs the reference's replay: {n} differs by {rel:.2e} of max|ref|"
    else:
        print("oracle/_ref absent: the reference arm is skipped")
    return arms


def noaux_arms(T, E, K, n_group, topk_group):
    from xtuner_b200 import router

    g = torch.Generator(device=DEV).manual_seed(2)
    logits = torch.randn(T, E, generator=g, device=DEV).requires_grad_(True)
    ids = torch.randint(0, E, (T, 3, K), generator=g, device=DEV)[:, 1, :]  # the layer slice of an [S, L, K] tensor
    g_tw = torch.randn(T, K, generator=g, device=DEV)
    g_rw = torch.randn(T, E, generator=g, device=DEV)
    r = router.NoAuxRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=2.5,
                           scoring_func="sigmoid", n_group=n_group, topk_group=topk_group).to(DEV)
    r.e_score_correction_bias.copy_(torch.randn(E, generator=g, device=DEV) * 0.1)

    def arm(replay):
        def step():
            logits.grad = None
            res = r(logits, replay)
            torch.autograd.backward((res["topk_weights"], res["router_weights"]), (g_tw, g_rw))
        return step

    return {"noaux_routed": arm(None), "noaux_replayed": arm(ids)}


def router_only(arms: dict, a) -> dict:
    t = time_arms(arms, a.repeats, a.iters * 5, a.warmup)
    # the router alone is a few microseconds of device work: host dispatch sets the wall time, so the kernels' own
    # device time is reported beside it
    ku = kernel_us(arms, a.iters)
    for k in t:
        t[k]["kernel_us"] = ku[k]
    return t


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=("block", "router", "noaux"), default=None, help="one group of arms")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("router_replay_bench: needs a CUDA device")
    res = {"card": card(), "arms": {}}
    if a.only in (None, "block"):
        for name, shape in (("block_c2", (8192, 2048, 768, 8, 2)), ("block_qwen3_30b_a3b", (8192, 2048, 768, 128, 8))):
            t = time_arms(block_arms(*shape), a.repeats, a.iters, a.warmup)
            res["arms"][name] = {"shape": dict(zip("THIEK", shape)), **t}
            torch.cuda.empty_cache()
    if a.only in (None, "router"):
        res["arms"]["router_e128_k8"] = {"shape": {"T": 8192, "E": 128, "K": 8},
                                         **router_only(router_arms(8192, 128, 8), a)}
    if a.only in (None, "noaux"):
        shape = {"T": 16384, "E": 256, "K": 8, "n_group": 8, "topk_group": 4}
        res["arms"]["noaux_deepseek_v3"] = {"shape": shape, **router_only(noaux_arms(*shape.values()), a)}
    for group, d in res["arms"].items():
        for arm, v in d.items():
            if isinstance(v, dict) and "ms_median" in v:
                extra = f";  kernels {v['kernel_us']:.1f} us" if "kernel_us" in v else ""
                print(f"{group:22s} {arm:20s} {v['ms_median'] * 1e3:9.1f} us fwd+bwd (min {v['ms_min'] * 1e3:.1f}, "
                      f"max {v['ms_max'] * 1e3:.1f}){extra}")
    print(f"card: {res['card']}")
    print("ROUTERREPLAYBENCH " + json.dumps(res))


if __name__ == "__main__":
    main()
