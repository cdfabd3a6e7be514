"""Forward + backward of the lm_head cross-entropy at the Qwen3-MoE head (T = 8192 rows, H = 2048, V = 151 936), three
arms timed in alternation with CUDA events after warm-up:

  ours        ops.lm_head_cross_entropy (xtb_lm_head_ce: logits GEMM with the CE epilogue, row kernel, NN + TN GEMMs)
  ref_eager   the reference's mode "eager": F.linear -> .float() -> F.cross_entropy, torch autograd
  ref_chunk   the reference's mode "chunk" (ChunkLoss) at --chunk rows

Prints one line per arm and a JSON line: ms per call (median and spread over repeats), TFLOP/s on 6 T V H FLOP and its
share of the H100 SXM data sheet's 989 dense BF16 TFLOP/s, peak allocated memory of one call, and the card name and power
limit read in the same run.  Needs a GPU; there is no CPU fallback.

    python scripts/lm_head_ce_bench.py [--T 8192 --H 2048 --V 151936 --chunk 1024 --repeats 5 --iters 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests.lm_head_ce_reference import lm_head_ce  # noqa: E402
from xtuner_b200 import ops  # noqa: E402

PEAK_BF16_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16, 700 W card


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        p, c = (s.strip() for s in out.strip().splitlines()[0].split(","))
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(p), float(c)
    except Exception as e:  # noqa: BLE001  (reported, not guessed)
        info["error"] = f"nvidia-smi: {e}"
    return info


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
        raise SystemExit("lm_head_ce_bench: needs a CUDA device")
    dev = "cuda"
    T, H, V = a.T, a.H, a.V
    g = torch.Generator(device=dev).manual_seed(0)
    h = torch.randn(T, H, generator=g, device=dev).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(V, H, generator=g, device=dev) * H ** -0.5).to(torch.bfloat16).requires_grad_(True)
    lab = torch.randint(0, V, (T,), generator=g, device=dev)
    lab[torch.rand(T, generator=g, device=dev) < 0.3] = -100
    lw = (lab != -100).float() / (lab != -100).sum()

    def ours():
        loss = ops.lm_head_cross_entropy(h, w, lab, lw)
        return (loss,) + torch.autograd.grad(loss, (h, w))

    arms = {
        "ours": ours,
        "ref_eager": lambda: lm_head_ce(h, w, lab, lw),
        "ref_chunk": lambda: lm_head_ce(h, w, lab, lw, chunk_size=a.chunk),
    }
    flop = 6.0 * T * V * H
    base = torch.cuda.memory_allocated()
    peak, loss_val = {}, {}
    for name, fn in arms.items():  # warm-up, then the peak memory of one call (its gradients included)
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        r = fn()
        torch.cuda.synchronize()
        peak[name] = torch.cuda.max_memory_allocated() - base
        loss_val[name] = float(r[0])
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
    res = {"shape": {"T": T, "H": H, "V": V, "chunk": a.chunk}, "card": c, "flop_per_call": flop, "arms": {}}
    for name in arms:
        ms = statistics.median(times[name])
        tf = flop / (ms * 1e-3) / 1e12
        res["arms"][name] = {"ms_median": ms, "ms_min": min(times[name]), "ms_max": max(times[name]), "tflops": tf,
                             "share_of_989": tf / PEAK_BF16_TFLOPS, "peak_alloc_gib": peak[name] / 2 ** 30,
                             "loss": loss_val[name]}
        print(f"{name:10s} {ms:8.2f} ms/call (min {min(times[name]):.2f}, max {max(times[name]):.2f})  {tf:6.1f} TFLOP/s "
              f"({tf / PEAK_BF16_TFLOPS:.1%} of 989)  peak {peak[name] / 2 ** 30:6.2f} GiB  loss {loss_val[name]:.6f}")
    print(f"card: {c}")
    print("LMHEADCE " + json.dumps(res))


if __name__ == "__main__":
    main()
