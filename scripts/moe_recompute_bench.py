"""Time and peak memory of the fused MoE block's selective recompute (``recompute=`` of ``fused.fused_moe_block``) over a
stack of blocks, forward + backward, with the card name and power limit read in the same run.

Workloads
  c2              48 blocks at C2 (T = 8192, H = 2048, I = 768, E = 8, K = 2)
  qwen3_30b_a3b   blocks at the Qwen3-30B-A3B MoE layer shape (T = 8192, H = 2048, I = 768, E = 128, K = 8), as many as
                  the free memory holds under the most demanding arm (recompute=None), from the shapes; --qwen-layers
                  sets the count instead
Arms
  none            recompute=None: the node keeps x_perm, h, a and y
  act             recompute="act"
  experts         recompute="experts"
  ckpt_layer      recompute=None with every block under torch.utils.checkpoint(use_reentrant=False): the reference's
                  whole-layer recompute (FSDPConfig.recompute_ratio) reduced to the MoE half

Each arm's outputs, input gradient and first-block gradients are checked equal to the ``none`` arm's bit for bit before
timing.  Then every arm is warmed up and timed in alternation with CUDA events: ms per forward + backward, median and
min-max over the repeats.  Memory is taken over one step of each arm on its own, with no gradients held at its start:
peak allocated memory (torch.cuda.max_memory_allocated), whole and above what was allocated before the step (weights
and inputs: the rest is activations, gradients and the transients of the backward), and what the forward of the whole
stack leaves allocated for the backward (torch.cuda.memory_allocated between the two, above the same base).  Without
FSDP the stack's weight gradients are all held at the end of the backward, so where they outweigh the activations
they, not the activations, set the peak.  Prints one line per arm and a JSON line.  Needs
a GPU.

    python scripts/moe_recompute_bench.py [--repeats 5 --iters 3 --warmup 2] [--only c2|qwen3_30b_a3b]
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
from torch.utils.checkpoint import checkpoint  # noqa: E402

from lm_head_ce_bench import card  # noqa: E402

DEV = "cuda"
ARMS = {"none": None, "act": "act", "experts": "experts", "ckpt_layer": None}


def layer_bytes(T, H, I, E, K):
    """bytes one block holds from its forward to its backward under recompute=None, and its weights with their
    gradients"""
    M = T * K
    saved = (M * H + M * 2 * I + M * I + M * H) * 2 + 2 * T * H * 2 + 2 * T * E * 4 + T * K * (8 + 4 + 4) + M * 4
    weights = (E * 2 * I * H + E * H * I) * 2 + E * H * 4 + H * 4
    return saved, 2 * weights


def build(L, T, H, I, E, K, seed=0):
    g = torch.Generator(DEV).manual_seed(seed)
    x = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16).requires_grad_(True)
    params = []
    for _ in range(L):
        params.append([(1 + 0.1 * torch.randn(H, generator=g, device=DEV)).requires_grad_(True),
                       (torch.randn(E, H, generator=g, device=DEV) * 0.02).requires_grad_(True),
                       (torch.randn(E, 2 * I, H, generator=g, device=DEV) * H**-0.5).to(torch.bfloat16).requires_grad_(True),
                       (torch.randn(E, H, I, generator=g, device=DEV) * I**-0.5).to(torch.bfloat16).requires_grad_(True)])
    go = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    return x, params, go


def make_step(x, params, go, K, arm):
    from xtuner_b200 import fused

    recompute = ARMS[arm]

    def block(h, nw, gw, w13, w2):
        return fused.fused_moe_block(h, nw, 1e-6, gw, w13, w2, top_k=K, recompute=recompute)[0]

    leaves = [x] + [t for ps in params for t in ps]

    def step(between=None):
        for t in leaves:
            t.grad = None
        h = x
        for ps in params:
            h = checkpoint(block, h, *ps, use_reentrant=False) if arm == "ckpt_layer" else block(h, *ps)
        if between is not None:
            between()
        h.backward(go)
        return h.detach()

    return step


def check_equal(x, params, steps):
    """every arm's output, input gradient and first-block gradients equal the none arm's"""
    out = steps["none"]()
    want = [out.clone(), x.grad.clone()] + [t.grad.clone() for t in params[0]]
    for arm, step in steps.items():
        out = step()
        got = [out, x.grad] + [t.grad for t in params[0]]
        assert all(torch.equal(a, b) for a, b in zip(got, want)), f"arm {arm} changed the result"
    del want


def memory(step, leaves):
    """(peak allocated over one step, the part of it above the weights and inputs, what the forward leaves allocated
    for the backward)"""
    for t in leaves:
        t.grad = None  # the previous step's gradients are not part of the weights
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    held = []
    step(lambda: held.append(torch.cuda.memory_allocated() - base))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    return peak, peak - base, held[0]


def time_arms(steps, repeats, iters, warmup):
    for step in steps.values():
        for _ in range(warmup):
            step()
    times = {k: [] for k in steps}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(repeats):
        for name, step in steps.items():  # the arms alternate within each repeat
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(iters):
                step()
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) / iters)
    return {k: {"ms_median": statistics.median(v), "ms_min": min(v), "ms_max": max(v)} for k, v in times.items()}


def run(L, shape, a):
    T, H, I, E, K = shape
    x, params, go = build(L, T, H, I, E, K)
    steps = {arm: make_step(x, params, go, K, arm) for arm in ARMS}
    check_equal(x, params, steps)
    leaves = [x] + [t for ps in params for t in ps]
    mem = {arm: memory(step, leaves) for arm, step in steps.items()}
    t = time_arms(steps, a.repeats, a.iters, a.warmup)
    res = {"shape": dict(zip("THIEK", shape)), "layers": L,
           "arms": {arm: {**t[arm], "peak_alloc_gb": mem[arm][0] / 1e9, "peak_above_weights_gb": mem[arm][1] / 1e9,
                          "held_after_forward_gb": mem[arm][2] / 1e9} for arm in ARMS}}
    del x, params, go, steps, leaves
    torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--c2-layers", type=int, default=48)
    ap.add_argument("--qwen-layers", type=int, default=None)
    ap.add_argument("--only", choices=("c2", "qwen3_30b_a3b"), default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_recompute_bench: needs a CUDA device")
    from xtuner_b200 import _capi

    _capi.ensure_init()
    res = {"card": card(), "workloads": {}}
    if a.only in (None, "c2"):
        res["workloads"]["c2"] = run(a.c2_layers, (8192, 2048, 768, 8, 2), a)
    if a.only in (None, "qwen3_30b_a3b"):
        shape = (8192, 2048, 768, 128, 8)
        L = a.qwen_layers
        if L is None:
            saved, weights = layer_bytes(*shape)
            free, _ = torch.cuda.mem_get_info()
            # one block's backward transients (its gradients and the rebuilt tensors) on top of every block's state
            L = max(1, int((0.85 * free - 2 * saved) // (saved + weights)))
        res["workloads"]["qwen3_30b_a3b"] = run(L, shape, a)
    for wl, d in res["workloads"].items():
        for arm, v in d["arms"].items():
            print(f"{wl:14s} x{d['layers']:<3d} {arm:11s} {v['ms_median']:9.2f} ms fwd+bwd (min {v['ms_min']:.2f}, "
                  f"max {v['ms_max']:.2f});  peak {v['peak_alloc_gb']:.2f} GB, {v['peak_above_weights_gb']:.2f} GB above "
                  f"weights and inputs;  {v['held_after_forward_gb']:.2f} GB held from forward to backward")
    print(f"card: {res['card']}")
    print("MOERECOMPUTEBENCH " + json.dumps(res))


if __name__ == "__main__":
    main()
