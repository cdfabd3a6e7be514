#!/usr/bin/env python
"""GPU reference of BASELINE.md §3a, measured on the same box as our kernels: the UNMODIFIED reference kernels and
modules (InternLM/xtuner, the git-ignored copy under ``oracle/_ref``, see
``oracle/make_ref.py``) at config C2.  BENCH-ONLY: nothing under ``xtuner_b200/`` imports this file.

Part A, kernel by kernel (what each of our kernels replaces), CUDA-event timed over rotating buffers (> L2):
  * Triton ``m_grouped_gemm`` forward / dX (``xtuner/v1/ops/moe/cuda/triton_kernels/m_grouped_gemm_TMA_triton3_4.py``) and
    ``k_grouped_gemm`` dW (``k_grouped_gemm_TMA_triton3_4.py``), autotuned (``XTUNER_DETERMINISTIC`` unset: deterministic
    mode pins autotune to configs[0], ``xtuner/v1/__init__.py:14-21``, and would understate the reference);
  * the in-tree torch-fallback ``cuda_token_permute_torch`` / ``cuda_token_unpermute_torch``
    (``ops/moe/cuda/permute_unpermute.py:205-248``: what the reference runs when the grouped_gemm wheel is absent, as here);
  * eager ``native_swiglu`` (``ops/act_fn.py:7-9``), the fp32 gate GEMM (``moe_decoder_layer.py:138-140``) and the router's
    eager op sequence through the reference's own ``GreedyRouter`` when the package imports.
Part B: the MoE half of ``MoEDecoderLayer._forward`` (``moe_decoder_layer.py:392-488``) assembled from the reference's own
classes (RMSNorm, MoEGate+GreedyRouter, NaiveDispatcher, MoEBlock) — forward + backward of one layer, eager (the
reference's ``compile_cfg=False`` mode).

Usage:  python baseline/gpu_reference.py [--out FILE]     (1 GPU; several minutes: ~100 Triton
autotune compilations)
"""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(os.path.dirname(HERE), "oracle", "_ref")
C2 = dict(T=8192, H=2048, I=768, E=8, K=2)


def _load(relpath: str, name: str):
    path = os.path.join(REF, relpath)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def _time(fn, iters, rot, torch):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not os.path.isdir(os.path.join(REF, "xtuner", "v1")):
        print(json.dumps({"gpu_reference": None, "unavailable": "oracle/_ref is absent (build() places it where a reference checkout is available)"}))
        return
    os.environ.pop("XTUNER_DETERMINISTIC", None)
    import torch

    torch.manual_seed(0)
    dev = torch.device("cuda")
    T, H, I, E, K = (C2[k] for k in "THIEK")
    M, R, bf = T * K, 4, torch.bfloat16
    res: dict = {"config": dict(C2), "box": torch.cuda.get_device_name(0), "torch": torch.__version__, "notes": []}
    import triton

    res["triton"] = triton.__version__
    t_all = time.time()

    mg = _load("xtuner/v1/ops/moe/cuda/triton_kernels/m_grouped_gemm_TMA_triton3_4.py", "_ref_m_grouped_gemm")
    kg = _load("xtuner/v1/ops/moe/cuda/triton_kernels/k_grouped_gemm_TMA_triton3_4.py", "_ref_k_grouped_gemm")
    pu = _load("xtuner/v1/ops/moe/cuda/permute_unpermute.py", "_ref_permute_unpermute")

    def rnd(*shape, scale=1.0, dtype=bf):
        return (torch.randn(*shape, device=dev) * scale).to(dtype)

    # routing as in the bench: near-uniform random gate
    x0 = rnd(T, H)
    gate_w = rnd(E, H, scale=0.02, dtype=torch.float32)
    logits = torch.nn.functional.linear(x0.float(), gate_w)
    probs = torch.softmax(logits, dim=1, dtype=torch.float32)
    tw, ids = torch.topk(probs, K, dim=-1)
    tw = tw / tw.sum(-1, keepdim=True)
    tpe = torch.histc(ids.float(), bins=E, min=0, max=E).to(torch.int64)
    xs = [rnd(T, H) for _ in range(R)]
    xp = [rnd(M, H) for _ in range(R)]
    w13 = [rnd(E, 2 * I, H, scale=H**-0.5) for _ in range(R)]
    w2 = [rnd(E, H, I, scale=I**-0.5) for _ in range(R)]
    hs = [rnd(M, 2 * I) for _ in range(R)]
    acts = [rnd(M, I) for _ in range(R)]
    ys = [rnd(M, H) for _ in range(R)]
    it = args.iters
    gemm_us, flops = {}, {"nt_w13": 2 * M * 2 * I * H, "nt_w2": 2 * M * H * I, "nn_w2": 2 * M * H * I, "nn_w13": 2 * M * 2 * I * H,
                          "tn_w2": 2 * M * H * I, "tn_w13": 2 * M * 2 * I * H}
    def dump():
        if args.out:
            with open(args.out, "w") as f:
                f.write(json.dumps({"gpu_reference": res}) + "\n")

    calls = {
        "nt_w13": lambda i: mg.m_grouped_gemm(xp[i], w13[i], tpe, trans_b=True),
        "nt_w2": lambda i: mg.m_grouped_gemm(acts[i], w2[i], tpe, trans_b=True),
        "nn_w2": lambda i: mg.m_grouped_gemm(ys[i], w2[i], tpe, trans_b=False),
        "nn_w13": lambda i: mg.m_grouped_gemm(hs[i], w13[i], tpe, trans_b=False),
        "tn_w2": lambda i: kg.k_grouped_gemm(ys[i], acts[i], tpe),
        "tn_w13": lambda i: kg.k_grouped_gemm(hs[i], xp[i], tpe),
    }
    for name, fn in calls.items():
        try:
            t0 = time.time()
            us = _time(fn, it, R, torch)
            gemm_us[name] = {"us": round(us, 2), "tflops": round(flops[name] / us / 1e6, 1), "autotune_s": round(time.time() - t0, 1)}
        except Exception as e:  # noqa: BLE001
            gemm_us[name] = {"error": f"{type(e).__name__}: {e}"[:300]}
        res["gemm_us"] = gemm_us
        dump()  # partial results survive a timeout (autotuning ~100 Triton configs takes minutes)
    for kern, key in ((mg.m_grouped_gemm_bKmajor_kernel, "m_bKmajor"), (mg.m_grouped_gemm_bNmajor_kernel, "m_bNmajor"),
                      (kg.k_grouped_gemm_kernel, "k")):
        try:
            res.setdefault("autotune_best", {})[key] = {str(k): str(v) for k, v in kern.cache.items()}
        except Exception:  # noqa: BLE001
            pass

    s = 2
    ids32 = ids.to(torch.int32)
    perm_out = pu.cuda_token_permute_torch(xs[0], ids32)
    row_map = perm_out[1]
    res["permute_us"] = round(_time(lambda i: pu.cuda_token_permute_torch(xs[i], ids32), it, R, torch), 2)
    res["unpermute_us"] = round(_time(lambda i: pu.cuda_token_unpermute_torch(ys[i], row_map, tw), it, R, torch), 2)
    b_perm = T * H * s * (1 + K) + T * K * 8
    res["permute_GBs"] = round(b_perm / res["permute_us"] / 1e3, 1)
    res["unpermute_GBs"] = round(b_perm / res["unpermute_us"] / 1e3, 1)
    # backward of the two (autograd of the fallback ops)
    def perm_bwd(i):
        x = xs[i].detach().requires_grad_(True)
        out, _ = pu.cuda_token_permute_torch(x, ids32)
        out.backward(xp[i])

    def unperm_bwd(i):
        y = ys[i].detach().requires_grad_(True)
        p = tw.detach().requires_grad_(True)
        pu.cuda_token_unpermute_torch(y, row_map, p).backward(xs[i])

    res["permute_fwd_bwd_us"] = round(_time(perm_bwd, it, R, torch), 2)
    res["unpermute_fwd_bwd_us"] = round(_time(unperm_bwd, it, R, torch), 2)

    def swiglu(h):
        x1, x2 = torch.chunk(h, 2, dim=-1)
        return torch.nn.functional.silu(x1) * x2

    res["swiglu_us"] = round(_time(lambda i: swiglu(hs[i]), it, R, torch), 2)

    def swiglu_fb(i):
        h = hs[i].detach().requires_grad_(True)
        swiglu(h).backward(acts[i])

    res["swiglu_fwd_bwd_us"] = round(_time(swiglu_fb, it, R, torch), 2)
    res["gate_us"] = round(_time(lambda i: torch.nn.functional.linear(xs[i].float(), gate_w.float()), it, R, torch), 2)

    def router_eager(lg):  # op sequence of router/greedy.py:64-98 (timed as issued there: 5 small eager launches)
        p = torch.softmax(lg, dim=1, dtype=torch.float32)
        w, i_ = torch.topk(p, K, dim=-1)
        w = w / w.sum(-1, keepdim=True)
        return p, w, i_, torch.histc(i_, bins=E, min=0, max=E)

    res["router_us"] = round(_time(lambda i: router_eager(logits), it, R, torch), 2)
    dump()

    # ---- Part B: the MoE half of the reference's decoder layer from its own classes ------------------------------------
    try:
        sys.path.insert(0, ROOT)
        os.environ["XTUNER_REFERENCE_ROOT"] = REF
        from tests.golden import ref_shim

        ref_shim.REFERENCE_ROOT = REF
        ref_shim.import_reference()
        import torch.distributed as dist

        if not dist.is_initialized():
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29577")
            dist.init_process_group("gloo", rank=0, world_size=1)
        from xtuner.v1.module.decoder_layer.moe_decoder_layer import MoEActFnConfig, MoEBlock, MoEGate
        from xtuner.v1.module.dispatcher import build_dispatcher
        from xtuner.v1.module.rms_norm import RMSNorm
        from xtuner.v1.module.router import GreedyRouterConfig
        from xtuner.v1.ops import moe as ref_moe_ops

        res["reference_ops_bound"] = {n: getattr(getattr(ref_moe_ops, n), "__name__", str(getattr(ref_moe_ops, n)))
                                      for n in ("group_gemm", "permute", "unpermute")}
        norm = RMSNorm(H, eps=1e-6).to(dev).to(bf)
        gate = MoEGate(hidden_size=H, n_routed_experts=E, num_experts_per_tok=K,
                       router_config=GreedyRouterConfig(scoring_func="softmax", router_scaling_factor=1.0, norm_topk_prob=True)).to(dev)
        experts = MoEBlock(hidden_size=H, moe_intermediate_size=I, n_routed_experts=E, moe_act_fn_cfg=MoEActFnConfig()).to(dev).to(bf)
        disp = build_dispatcher(dispatcher=None, n_routed_experts=E)
        with torch.no_grad():
            gate.weight.normal_(0, 0.02)
            experts.fused_w1w3.weight.normal_(0, H**-0.5)
            experts.fused_w2.weight.normal_(0, (2 * I) ** -0.5)

        def layer(h):
            residual = h
            x = norm(h)
            rr = gate(x)
            pre = disp.dispatch_preprocess(hidden_states=x.view(-1, H), topk_ids=rr["topk_ids"], topk_weights=rr["topk_weights"])
            dis = disp.dispatch(pre_dispatched=pre, topk_weights=rr["topk_weights"], decoding=False)
            post = disp.dispatch_postprocess(pre_dispatched=pre, dispatched=dis)
            eo = experts(post["hidden_states"], post["tokens_per_expert"], decoding=False)
            pc = disp.combine_preprocess(hidden_states=eo, pre_dispatched=pre, dispatched=dis, post_dispatched=post, decoding=False)
            cb = disp.combine(pre_dispatched=pre, dispatched=dis, post_dispatched=post, pre_combined=pc, decoding=False)
            out = disp.combine_postprocess(pre_dispatched=pre, dispatched=dis, post_dispatched=post, pre_combined=pc, combined=cb)
            return out["hidden_states"].view(h.shape) + residual

        hin = [rnd(1, T, H) for _ in range(R)]
        params = [p for m in (norm, gate, experts) for p in m.parameters()]

        def fwd_bwd(i):
            for p in params:
                p.grad = None
            h = hin[i].detach().requires_grad_(True)
            layer(h).float().square().mean().backward()

        res["layer_fwd_ms"] = round(_time(lambda i: layer(hin[i]), it, R, torch) / 1e3, 4)
        res["layer_fwd_bwd_ms"] = round(_time(fwd_bwd, it, R, torch) / 1e3, 4)
        res["layer_tokens_per_s_48_layers"] = round(T / (res["layer_fwd_bwd_ms"] * 48 * 1e-3), 1)
        res["notes"].append("layer = RMSNorm + MoEGate/GreedyRouter + NaiveDispatcher + MoEBlock + residual of the reference, eager "
                            "(compile_cfg=False), fp32 master weights cast to bf16 once (as after FSDP's cast)")
    except Exception as e:  # noqa: BLE001
        import traceback

        res["layer_fwd_bwd_ms"] = None
        res["layer_error"] = f"{type(e).__name__}: {e}"[:500]
        res["layer_traceback"] = traceback.format_exc()[-1500:]
    res["wall_s"] = round(time.time() - t_all, 1)
    print(json.dumps({"gpu_reference": res}), flush=True)
    dump()


if __name__ == "__main__":
    main()
