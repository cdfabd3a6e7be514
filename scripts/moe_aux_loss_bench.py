"""The MoE auxiliary losses of a 48-layer model step, with and without ``plugin.install_moe_aux_loss``: per step, 48 calls
of the reference's ``AuxLossContext.accumulate`` on fp32 router weights, logits and int64 ids (a carrier hidden state
passed through), then ``finalize``, then the backward of the balancing loss plus the carrier (which brings in every
layer's z-loss through ``AuxLossScaler``).  Shapes: C2 (N 8192, E 8, K 2) and Qwen3-30B-A3B (N 8192, E 128, K 8); arms:
balancing only (the reference's default config) and balancing + z-loss.  Global averages are off (no process group).

Per (shape, arm) and side: ms per step (median, min and max over repeats that alternate the two sides, host dispatch
included, CUDA events), then, in a separate profiled run, the device time and the number of kernels per step.  Then a
short training step of the reference's tiny MoE model (``tests/workers/router_replay_worker.py``'s greedy model, both
losses) converted with ``convert_model(fused=True)``, with and without the install.  The last line is JSON with the card
name and power limit read in the same run.  Needs a GPU and the reference package under oracle/_ref (built by build()).

    python scripts/moe_aux_loss_bench.py [--layers 48 --repeats 7 --iters 10]
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

SHAPES = {"c2": (8192, 8, 2), "qwen3_30b_a3b": (8192, 128, 8)}


def make_step(N, E, K, layers, with_z):
    from xtuner.v1.loss.aux_loss import AuxLossConfig
    from xtuner.v1.loss.moe_loss import BalancingLossConfig, ZLossConfig

    g = torch.Generator(device="cuda").manual_seed(0)
    logits = [torch.randn(N, E, device="cuda", generator=g).requires_grad_(True) for _ in range(layers)]
    rws = [torch.softmax(l.detach(), -1).requires_grad_(True) for l in logits]
    ids = [rw.detach().topk(K, -1).indices for rw in rws]
    hidden = torch.randn(N, 64, device="cuda").requires_grad_(True)
    aux = AuxLossConfig().build(n_routed_experts=E, num_experts_per_tok=K)

    def step():
        bal = BalancingLossConfig().build()
        z = ZLossConfig().build() if with_z else None
        h = hidden
        for l in range(layers):
            h = aux.accumulate(selected_router_weights=rws[l], selected_router_logits=logits[l], selected_experts=ids[l],
                               hidden_states=h, balancing_ctx=bal, z_ctx=z, num_tokens_local=N)
        bal_loss, _, _ = aux.finalize(balancing_ctx=bal, z_ctx=z, non_pad_token=N)
        (bal_loss + h.sum()).backward()
        for t in (*rws, *logits, hidden):
            t.grad = None

    return step


def timed(step, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        step()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def profiled(step, iters):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
    evs = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sum(e.self_device_time_total for e in evs) / iters / 1000, sum(e.count for e in evs) / iters


def model_step(model, cfg):
    from xtuner.v1.loss.ce_loss import CELossConfig
    from xtuner.v1.loss.moe_loss import BalancingLossConfig, ZLossConfig
    from xtuner.v1.model.moe.moe import SequenceContext

    g = torch.Generator().manual_seed(7)
    input_ids = torch.randint(0, cfg.vocab_size, (1, 4097), dtype=torch.int64, generator=g).cuda()
    seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cuda")
    loss_cfg = CELossConfig()
    lctx = loss_cfg.loss_ctx_cls.build_batches([loss_cfg.build(data={"shifted_labels": input_ids[:, 1:]}, sp_mesh=None)])[0]

    def step():
        loss_ctx = {"lm": lctx, "balancing": BalancingLossConfig().build(), "z_loss": ZLossConfig().build()}
        o = model(seq_ctx=seq_ctx, loss_ctx=loss_ctx)
        (o.loss + o.balancing_loss).backward()
        model.zero_grad(set_to_none=True)

    return step


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=48)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moe_aux_loss_bench: needs a CUDA device")
    from tests.golden import ref_shim

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    if not ref_shim.reference_available():
        raise SystemExit("moe_aux_loss_bench: oracle/_ref is missing (build() places the reference package there)")
    ref_shim.import_reference()
    from xtuner_b200 import plugin

    sides = {"reference": plugin.uninstall_moe_aux_loss, "installed": plugin.install_moe_aux_loss}
    result = {"card": card(), "layers": a.layers, "rows": {}}
    for shape, (N, E, K) in SHAPES.items():
        for arm, with_z in (("balancing", False), ("balancing+z", True)):
            step = make_step(N, E, K, a.layers, with_z)
            times = {s: [] for s in sides}
            for s, on in sides.items():  # warm-up of both sides
                on()
                for _ in range(3):
                    step()
            for _ in range(a.repeats):
                for s, on in sides.items():
                    on()
                    times[s].append(timed(step, a.iters))
            row = {}
            for s, on in sides.items():
                on()
                dev_ms, kernels = profiled(step, a.iters)
                t = times[s]
                row[s] = {"ms_median": statistics.median(t), "ms_min": min(t), "ms_max": max(t), "device_ms": dev_ms,
                          "kernels": kernels}
                print(f"{shape} {arm:12s} {s:10s} {row[s]['ms_median']:7.3f} ms/step (min {min(t):.3f}, max {max(t):.3f}); "
                      f"device {dev_ms:.3f} ms, {kernels:.0f} kernels per step", flush=True)
            result["rows"][f"{shape}/{arm}"] = row
            plugin.uninstall_moe_aux_loss()
    # the reference's tiny MoE model, fused conversion, with and without the install
    from tests.workers.router_replay_worker import build_model

    model, cfg = build_model("greedy")
    plugin.convert_model(model, fused=True)
    step = model_step(model, cfg)
    times = {s: [] for s in sides}
    for s, on in sides.items():
        on()
        for _ in range(3):
            step()
    for _ in range(a.repeats):
        for s, on in sides.items():
            on()
            times[s].append(timed(step, a.iters))
    result["tiny_model_fused"] = {s: {"ms_median": statistics.median(t), "ms_min": min(t), "ms_max": max(t)}
                                  for s, t in times.items()}
    for s, t in times.items():
        print(f"tiny model (2 layers, 4096 tokens, fused) {s:10s} {statistics.median(t):7.3f} ms/step "
              f"(min {min(t):.3f}, max {max(t):.3f})", flush=True)
    plugin.uninstall_moe_aux_loss()
    plugin.restore_model(model)
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
