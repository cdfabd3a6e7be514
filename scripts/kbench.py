#!/usr/bin/env python
"""Micro-benchmark of individual C-ABI kernels at config C2 (T=8192,H=2048,I=768,E=8,K=2) with rotating
buffers (working set > L2) and CUDA-event timing.  Usage: python scripts/kbench.py [name-substring ...]"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from xtuner_b200 import _capi, ops  # noqa: E402
from xtuner_b200._capi import check, current_stream, ptr  # noqa: E402

T, H, I, E, K = 8192, 2048, 768, 8, 2
M = T * K
R = 6  # rotating copies
dev = torch.device("cuda")
lib = _capi.ensure_init()
torch.manual_seed(0)
bf = torch.bfloat16

def rnd(*shape, dtype=bf, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(dtype)

xs = [rnd(T, H) for _ in range(R)]
gate_w = rnd(E, H, dtype=torch.float32, scale=0.02)
logits = [torch.empty(T, E, device=dev) for _ in range(R)]
rw = torch.empty(T, E, device=dev); tw = torch.empty(T, K, device=dev)
ids = torch.empty(T, K, dtype=torch.int64, device=dev); ids32 = torch.empty(T, K, dtype=torch.int32, device=dev)
tpe = torch.empty(E, dtype=torch.int64, device=dev)
st = current_stream()
check(lib.xtb_gate_logits(ptr(xs[0]), ptr(gate_w), None, ptr(logits[0]), T, H, E, st))
check(lib.xtb_router_greedy(ptr(logits[0]), T, E, K, 0, 1, 1.0, ptr(rw), ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), st))
xperm = [torch.empty(M, H, dtype=bf, device=dev) for _ in range(R)]
rmap = torch.empty(M, dtype=torch.int32, device=dev)
ws = ops.permute_workspace(T, K, E, dev)
check(lib.xtb_moe_permute(ptr(xs[0]), ptr(ids32), T, K, E, H * 2, ptr(xperm[0]), ptr(rmap), None, None, ptr(ws), st))
for i in range(1, R):
    xperm[i].copy_(xperm[0])
w13 = [rnd(E, 2 * I, H, scale=H**-0.5) for _ in range(R)]
w2 = [rnd(E, H, I, scale=I**-0.5) for _ in range(R)]
hs = [rnd(M, 2 * I) for _ in range(R)]
acts = [rnd(M, I) for _ in range(R)]
ys = [rnd(M, H) for _ in range(R)]
outs = [torch.empty(T, H, dtype=bf, device=dev) for _ in range(R)]
gl = torch.randn(T, E, device=dev)
gws = torch.empty(E, H, device=dev)
gxs = [torch.empty(T, H, dtype=bf, device=dev) for _ in range(R)]
wsb = torch.empty(int(lib.xtb_gate_logits_bwd_workspace_bytes(T, H, E)), dtype=torch.uint8, device=dev)
gtw = torch.empty(T, K, device=dev)
dw13 = torch.empty(E, 2 * I, H, dtype=bf, device=dev); dw2 = torch.empty(E, H, I, dtype=bf, device=dev)

s = 2
B_perm = T * H * s * (1 + K) + T * K * 8
KERNELS = {
    "gate_logits": (lambda i: lib.xtb_gate_logits(ptr(xs[i]), ptr(gate_w), None, ptr(logits[i]), T, H, E, st), T * H * s, "B"),
    "gate_logits_bwd": (lambda i: lib.xtb_gate_logits_bwd(ptr(gl), ptr(xs[i]), ptr(gate_w), ptr(gws), ptr(gxs[i]), None, T, H, E, ptr(wsb), st), 2 * T * H * s, "B"),
    "router_greedy": (lambda i: lib.xtb_router_greedy(ptr(logits[i]), T, E, K, 0, 1, 1.0, ptr(rw), ptr(tw), ptr(ids), ptr(ids32), ptr(tpe), st), T * E * 8, "B"),
    "router_greedy_bwd": (lambda i: lib.xtb_router_greedy_bwd(ptr(rw), ptr(tw), ptr(ids), ptr(gtw), None, None, T, E, K, 0, 1, 1.0, ptr(logits[i]), st), T * E * 8, "B"),
    "permute": (lambda i: lib.xtb_moe_permute(ptr(xs[i]), ptr(ids32), T, K, E, H * 2, ptr(xperm[i]), ptr(rmap), None, None, ptr(ws), st), B_perm, "B"),
    "combine": (lambda i: lib.xtb_moe_combine(ptr(ys[i]), ptr(rmap), ptr(tw), None, 1.0, T, K, H, ptr(outs[i]), st), B_perm, "B"),
    "combine_residual": (lambda i: lib.xtb_moe_combine(ptr(ys[i]), ptr(rmap), ptr(tw), ptr(xs[i]), 1.0, T, K, H, ptr(outs[i]), st), B_perm + T * H * s, "B"),
    "unpermute_bwd": (lambda i: lib.xtb_moe_unpermute_bwd(ptr(xs[i]), ptr(ys[i]), ptr(rmap), ptr(tw), T, K, H, ptr(xperm[i]), ptr(gtw), st), T * H * s + 2 * M * H * s, "B"),
    "swiglu": (lambda i: lib.xtb_swiglu(ptr(hs[i]), ptr(acts[i]), M, I, st), 3 * M * I * s, "B"),
    "swiglu_bwd": (lambda i: lib.xtb_swiglu_bwd(ptr(acts[i]), ptr(hs[i]), ptr(hs[(i + 1) % R]), M, I, st), 5 * M * I * s, "B"),
    "gemm_nt_w13": (lambda i: lib.xtb_group_gemm_nt(ptr(xperm[i]), ptr(w13[i]), ptr(tpe), M, 2 * I, H, E, ptr(hs[i]), st), 2 * M * 2 * I * H, "F"),
    "gemm_nt_swiglu_w13": (lambda i: lib.xtb_group_gemm_nt_swiglu(ptr(xperm[i]), ptr(w13[i]), ptr(tpe), M, I, H, E, ptr(hs[i]), ptr(acts[i]), st), 2 * M * 2 * I * H, "F"),
    "gemm_nt_w2": (lambda i: lib.xtb_group_gemm_nt(ptr(acts[i]), ptr(w2[i]), ptr(tpe), M, H, I, E, ptr(ys[i]), st), 2 * M * H * I, "F"),
    "gemm_nn_w2": (lambda i: lib.xtb_group_gemm_nn(ptr(ys[i]), ptr(w2[i]), ptr(tpe), M, H, I, E, ptr(acts[i]), st), 2 * M * H * I, "F"),
    "gemm_nn_w13": (lambda i: lib.xtb_group_gemm_nn(ptr(hs[i]), ptr(w13[i]), ptr(tpe), M, 2 * I, H, E, ptr(xperm[i]), st), 2 * M * 2 * I * H, "F"),
    "gemm_tn_w2": (lambda i: lib.xtb_group_gemm_tn(ptr(ys[i]), ptr(acts[i]), ptr(tpe), M, H, I, E, ptr(dw2), st), 2 * M * H * I, "F"),
    "gemm_tn_w13": (lambda i: lib.xtb_group_gemm_tn(ptr(hs[i]), ptr(xperm[i]), ptr(tpe), M, 2 * I, H, E, ptr(dw13), st), 2 * M * 2 * I * H, "F"),
    "gemm_tn_pair": (lambda i: lib.xtb_group_gemm_tn_pair(ptr(ys[i]), ptr(acts[i]), H, I, ptr(dw2), ptr(hs[i]), ptr(xperm[i]), 2 * I, H, ptr(dw13),
                                                          ptr(tpe), M, E, st), 2 * M * H * I + 2 * M * 2 * I * H, "F"),
}

sel = sys.argv[1:]
iters = int(os.environ.get("KB_ITERS", "30"))
torch.cuda.synchronize()
for name, (fn, work, kind) in KERNELS.items():
    if sel and not any(s_ in name for s_ in sel):
        continue
    for i in range(3):
        check(fn(i % R), name)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        check(fn(i % R), name)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    rate = work / (us * 1e-6)
    print(f"{name:22s} {us:8.2f} us   " + (f"{rate/1e9:8.1f} GB/s" if kind == "B" else f"{rate/1e12:8.1f} TFLOP/s"), flush=True)

if os.environ.get("KB_GEMM_STUDY"):
    import subprocess, threading, statistics

    def sample_clocks(fn_loop):
        p = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm,power.draw,clocks_event_reasons.sw_power_cap", "--format=csv,noheader,nounits", "-lms", "50"],
                             stdout=subprocess.PIPE, text=True)
        lines = []
        th = threading.Thread(target=lambda: [lines.append(l) for l in p.stdout], daemon=True)
        th.start()
        r = fn_loop()
        p.terminate()
        sm, pw = [], []
        for l in lines:
            f = l.split(",")
            try:
                sm.append(float(f[0])); pw.append(float(f[1]))
            except Exception:
                pass
        return r, (statistics.median(sm) if sm else None), (max(pw) if pw else None), len(sm)

    def timeit(fn, iters, rot):
        for i in range(3):
            fn(i % rot)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            fn(i % rot)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / iters

    print("\n# GEMM study: w13 forward (16384 x 1536 x 2048, 103 GFLOP): cold (6 rotating buffers) vs warm (1), burst vs sustained")
    flops = 2 * M * 2 * I * H
    ours = lambda i: check(lib.xtb_group_gemm_nt(ptr(xperm[i]), ptr(w13[i]), ptr(tpe), M, 2 * I, H, E, ptr(hs[i]), st))
    wd = [w.view(E * 2 * I, H)[: 2 * I] for w in w13]
    cublas = lambda i: torch.matmul(xperm[i], wd[i].T, out=hs[i])
    for label, fn in (("ours_nt", ours), ("cublas_dense", cublas)):
        for rot in (1, R):
            for iters in (3, 30, 4000):
                if iters >= 1000:
                    us, clk, pw, ns = sample_clocks(lambda: timeit(fn, iters, rot))
                    extra = f"  sm_clk_median={clk} MHz power_max={pw} W samples={ns}"
                else:
                    us, extra = timeit(fn, iters, rot), ""
                print(f"{label:14s} rot={rot} iters={iters:5d}  {us:8.2f} us  {flops/us/1e6:8.1f} TFLOP/s{extra}", flush=True)
