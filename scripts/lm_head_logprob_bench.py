"""The RL trainer's lm_head calls at the Qwen3-MoE head (T = 8192 rows, H = 2048, V = 151 936, about 30 % of the labels
ignored), each through the reference's own context with ``plugin.install_rl_lm_head()`` (ours) and without it (ref),
timed in alternation with CUDA events after warm-up:

  logprob_{eager,chunk}  LogProbContext.forward under no_grad (compute_actor_logprobs / compute_ref_logprobs)
  grpo_{eager,chunk}     GRPOLossContext.forward + backward, vanilla loss (clip 0.2 / 0.28), low_var_kl on

Chunk mode runs --chunk rows at a time.  Prints one line per arm and a JSON line: ms per call (median, min and max over
repeats), TFLOP/s on the algorithmic 2 T V H FLOP (forward) and 6 T V H FLOP (forward + backward), peak allocated memory
of one call, and the card name and power limit read in the same run.  Needs a GPU and the reference package that
``oracle/make_ref.py`` places under ``oracle/_ref``.

    python scripts/lm_head_logprob_bench.py [--T 8192 --H 2048 --V 151936 --chunk 1024 --repeats 5 --iters 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.lm_head_ce_bench import card  # noqa: E402
from tests.golden import ref_shim  # noqa: E402
from xtuner_b200 import plugin  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=8192)
    ap.add_argument("--H", type=int, default=2048)
    ap.add_argument("--V", type=int, default=151936)
    ap.add_argument("--chunk", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lm_head_logprob_bench: needs a CUDA device")
    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    if not ref_shim.reference_available():
        raise SystemExit("lm_head_logprob_bench: oracle/_ref is missing (build() places it where a reference exists)")
    ref_shim.import_reference()
    from xtuner.v1.loss.rl_loss import LogProbConfig, LogProbContext, LogProbKwargs
    from xtuner.v1.rl.loss.grpo_loss import GRPOLossConfig, GRPOLossContext, GRPOLossKwargs

    dev = "cuda"
    T, H, V = a.T, a.H, a.V
    g = torch.Generator(device=dev).manual_seed(0)
    h = torch.randn(1, T, H, generator=g, device=dev).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(V, H, generator=g, device=dev) * H ** -0.5).to(torch.bfloat16).requires_grad_(True)
    lab = torch.randint(0, V, (1, T), generator=g, device=dev)
    lab[torch.rand(1, T, generator=g, device=dev) < 0.3] = -100
    adv = torch.randn(1, T, generator=g, device=dev)
    noise = 0.2 * torch.randn(1, T, generator=g, device=dev)

    def logprob(mode):
        ctx = LogProbContext(LogProbConfig(mode=mode, chunk_size=a.chunk), LogProbKwargs(shifted_labels=lab))
        with torch.no_grad():
            return ctx.forward(h, w)[0],

    with torch.no_grad():
        old = logprob("chunk")[0] + noise

    def grpo(mode):
        cfg = GRPOLossConfig(policy_loss_cfg={"loss_type": "vanilla", "cliprange_low": 0.2, "cliprange_high": 0.28},
                             use_kl_loss=True, kl_loss_coef=0.001, kl_loss_type="low_var_kl", mode=mode,
                             chunk_size=a.chunk)
        kw = GRPOLossKwargs(shifted_labels=lab, old_logprobs=old, advantages=adv, ref_logprobs=old - noise)
        (ctx,) = GRPOLossContext.build_batches([GRPOLossContext(cfg, kw)])
        loss = ctx.forward(h, w)[0]
        return (loss,) + torch.autograd.grad(loss, (h, w))

    def arm(fn, mode, ours):
        def run():
            if ours:
                plugin.install_rl_lm_head()
            try:
                return fn(mode)
            finally:
                plugin.uninstall_rl_lm_head()
        return run

    arms, flop = {}, {}
    for kind, fn, f in (("logprob", logprob, 2.0), ("grpo", grpo, 6.0)):
        for mode in ("eager", "chunk"):
            for who in ("ours", "ref"):
                arms[f"{kind}_{mode}_{who}"] = arm(fn, mode, who == "ours")
                flop[f"{kind}_{mode}_{who}"] = f * T * V * H
    base = torch.cuda.memory_allocated()
    peak, first = {}, {}
    for name, fn in arms.items():  # warm-up, then the peak memory of one call (its gradients included)
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        r = fn()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() - base
        first[name] = r[0].float().sum().item() if r[0].dim() else r[0].item()
        del r
    times = {k: [] for k in arms}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(a.repeats):
        for name, fn in arms.items():  # alternate the arms within each repeat
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(a.iters):
                fn()
            ev[1].record()
            torch.cuda.synchronize()
            times[name].append(ev[0].elapsed_time(ev[1]) / a.iters)
    c = card()
    res = {"shape": {"T": T, "H": H, "V": V, "chunk": a.chunk}, "card": c, "arms": {}}
    for name in arms:
        ms = statistics.median(times[name])
        tf = flop[name] / (ms * 1e-3) / 1e12
        res["arms"][name] = {"ms_median": ms, "ms_min": min(times[name]), "ms_max": max(times[name]), "tflops": tf,
                             "peak_alloc_gib": peak[name] / 2 ** 30, "value": first[name]}
        print(f"{name:20s} {ms:8.2f} ms/call (min {min(times[name]):.2f}, max {max(times[name]):.2f})  {tf:6.1f} TFLOP/s  "
              f"peak {peak[name] / 2 ** 30:6.2f} GiB  value {first[name]:.6f}")
    print(f"card: {c}")
    print("LMHEADLOGPROB " + json.dumps(res))


if __name__ == "__main__":
    main()
