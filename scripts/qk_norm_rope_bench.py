"""Forward + backward of q_norm / k_norm + the rotary embedding at the Qwen3-30B-A3B attention input (T = 8192 tokens,
Hq = 32, Hkv = 4, D = 128, bf16 norm weights as under FSDP's bf16 MixedPrecisionPolicy), three arms timed in alternation
with CUDA events after warm-up:

  ours          ops.qk_norm_rope (xtb_qk_norm_rope + xtb_qk_norm_rope_bwd)
  ref_eager     the reference's steps of MultiHeadAttention.forward (mha.py:353-363): its native_rms_norm (F.rms_norm)
                on [1, T, H, D], the transpose, apply_rotary_pos_emb_cuda; torch autograd
  ref_compiled  the same function under torch.compile, as the reference's default compile_cfg runs it

Before timing, the outputs and gradients of the three arms are compared at the timed size.  Prints one line per arm
(ms per forward + backward: median, min and max over the repeats, host dispatch included; the summed device time of the
kernels one call launches, from torch.profiler in a run of its own; achieved bytes/s of the algorithmic traffic over
each, and its share of the H100 SXM data sheet's 3.35 TB/s) and a JSON line with the card name and power limit read in the same run.
Needs a GPU and the reference package under oracle/_ref (built by build()); there is no fallback.

    python scripts/qk_norm_rope_bench.py [--T 8192 --Hq 32 --Hkv 4 --D 128 --repeats 7 --iters 20]
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
from xtuner_b200 import ops  # noqa: E402

PEAK_TBPS = 3.35  # H100 SXM data sheet, HBM3


def traffic_bytes(T: int, H: int, D: int) -> int:
    """algorithmic bytes of one forward + backward: the forward reads x, cos, sin and writes out and rstd; the backward
    reads g, x, rstd, cos, sin and writes dx (the [2, D] weight gradient is negligible)"""
    x, cs, rstd = T * H * D * 2, 2 * T * D * 2, T * H * 4
    return (x + cs + x + rstd) + (x + x + rstd + cs + x)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=8192)
    ap.add_argument("--Hq", type=int, default=32)
    ap.add_argument("--Hkv", type=int, default=4)
    ap.add_argument("--D", type=int, default=128)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("qk_norm_rope_bench: needs a CUDA device")
    from tests.golden import ref_shim

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    if not ref_shim.reference_available():
        raise SystemExit("qk_norm_rope_bench: oracle/_ref is absent (build() places the reference package there)")
    ref_shim.import_reference()
    from xtuner.v1.ops.rms_norm import native_rms_norm
    from xtuner.v1.ops.rotary_emb import apply_rotary_pos_emb_cuda

    dev = "cuda"
    T, Hq, Hkv, D, eps = a.T, a.Hq, a.Hkv, a.D, 1e-6
    g = torch.Generator(device=dev).manual_seed(0)
    qp = torch.randn(1, T, Hq * D, generator=g, device=dev).to(torch.bfloat16).requires_grad_(True)  # q_proj output
    kp = torch.randn(1, T, Hkv * D, generator=g, device=dev).to(torch.bfloat16).requires_grad_(True)
    wq = (1 + 0.3 * torch.randn(D, generator=g, device=dev)).to(torch.bfloat16).requires_grad_(True)
    wk = (1 + 0.3 * torch.randn(D, generator=g, device=dev)).to(torch.bfloat16).requires_grad_(True)
    pos = torch.arange(T, device=dev) % 4096  # packed documents of 4096 tokens
    inv = 1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64, device=dev).float() / D))
    emb = torch.cat([pos[:, None].float() * inv[None]] * 2, -1)[None]
    cos, sin = emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)  # [1, T, D]
    gq = torch.randn(1, Hq, T, D, generator=g, device=dev).to(torch.bfloat16)
    gk = torch.randn(1, Hkv, T, D, generator=g, device=dev).to(torch.bfloat16)
    leaves = (qp, kp, wq, wk)

    def reference(qp, kp, wq, wk):
        q = native_rms_norm(qp.view(1, T, Hq, D), wq, eps).transpose(1, 2)
        k = native_rms_norm(kp.view(1, T, Hkv, D), wk, eps).transpose(1, 2)
        return apply_rotary_pos_emb_cuda(q, k, cos, sin)

    def fused(qp, kp, wq, wk):
        oq, ok = ops.qk_norm_rope(qp.view(T, Hq, D), kp.view(T, Hkv, D), cos[0], sin[0], wq, wk, eps)
        return oq.view(1, T, Hq, D).transpose(1, 2), ok.view(1, T, Hkv, D).transpose(1, 2)

    compiled = torch.compile(reference)

    def arm(fn):
        def step():
            for t in leaves:
                t.grad = None
            oq, ok = fn(*leaves)
            torch.autograd.backward((oq, ok), (gq, gk))
            return oq, ok, qp.grad, kp.grad, wq.grad, wk.grad
        return step

    arms = {"ours": arm(fused), "ref_eager": arm(reference), "ref_compiled": arm(compiled)}
    results = {name: [t.detach().clone() for t in fn()] for name, fn in arms.items()}
    names = ["q_embed", "k_embed", "dq_proj", "dk_proj", "dw_q", "dw_k"]
    agreement = {}
    for name in ("ours", "ref_compiled"):
        rel = {}
        for n, x, y in zip(names, results[name], results["ref_eager"]):
            rel[n] = float((x.float() - y.float()).abs().max() / y.float().abs().max().clamp_min(1e-30))
            assert rel[n] <= 2e-2, f"{name} vs ref_eager: {n} differs by {rel[n]:.3e} of max|ref|"
        agreement[name] = rel
        print(f"{name} vs ref_eager, largest |diff| / max|ref|: " + ", ".join(f"{n} {r:.2e}" for n, r in rel.items()))
    del results
    for fn in arms.values():
        for _ in range(a.warmup):
            fn()
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
    kernel_us = {}
    for name, fn in arms.items():  # a run of its own: summed device time of the kernels one call launches
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters):
                fn()
            torch.cuda.synchronize()
        evs = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
        kernel_us[name] = sum(e.self_device_time_total for e in evs) / a.iters
        top = sorted(evs, key=lambda e: -e.self_device_time_total)[:6]
        print(f"{name} kernels per call: " + "; ".join(f"{e.key[:60]} {e.self_device_time_total / a.iters:.1f} us" for e in top))
    c = card()
    nbytes = traffic_bytes(T, Hq + Hkv, D)
    res = {"shape": {"T": T, "Hq": Hq, "Hkv": Hkv, "D": D}, "card": c, "bytes_per_call": nbytes, "agreement": agreement,
           "arms": {}}
    for name in arms:
        ms = statistics.median(times[name])
        tbps = nbytes / (ms * 1e-3) / 1e12
        ktbps = nbytes / (kernel_us[name] * 1e-6) / 1e12
        res["arms"][name] = {"ms_median": ms, "ms_min": min(times[name]), "ms_max": max(times[name]), "tb_per_s": tbps,
                             "share_of_3.35": tbps / PEAK_TBPS, "kernel_us": kernel_us[name], "kernel_tb_per_s": ktbps}
        print(f"{name:12s} {ms * 1e3:8.1f} us fwd+bwd (min {min(times[name]) * 1e3:.1f}, max {max(times[name]) * 1e3:.1f})  "
              f"{tbps:5.2f} TB/s ({tbps / PEAK_TBPS:.1%} of 3.35) on {nbytes / 1e6:.0f} MB;  kernels {kernel_us[name]:.1f} us "
              f"= {ktbps:.2f} TB/s ({ktbps / PEAK_TBPS:.1%})")
    print(f"card: {c}")
    print("QKNORMROPE " + json.dumps(res))


if __name__ == "__main__":
    main()
