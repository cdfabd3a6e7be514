"""GPU worker: the UNMODIFIED reference MoE models (the copy under oracle/_ref, see oracle/make_ref.py) trained one step
with both auxiliary losses configured (the default ``BalancingLossConfig`` and a ``ZLossConfig``, global averages on
over a one-rank NCCL group), converted by ``xtuner_b200.plugin.convert_model`` per-op and (greedy router) with
``fused=True``, first without and then with ``install_moe_aux_loss``.  The uninstalled step runs twice, which measures
the run-to-run noise of the reference's own GPU kernels.  Prints one JSON line; tests/test_gpu_moe_aux_loss.py asserts
on it."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref")
LOSSES = ("loss", "balancing_loss", "z_loss")


def step(model, cfg):
    import torch
    from xtuner.v1.loss.ce_loss import CELossConfig
    from xtuner.v1.loss.moe_loss import BalancingLossConfig, ZLossConfig
    from xtuner.v1.model.moe.moe import SequenceContext

    g = torch.Generator().manual_seed(7)
    input_ids = torch.randint(0, cfg.vocab_size, (1, 513), dtype=torch.int64, generator=g).cuda()
    seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cuda")
    loss_cfg = CELossConfig()
    lctx = loss_cfg.loss_ctx_cls.build_batches([loss_cfg.build(data={"shifted_labels": input_ids[:, 1:]}, sp_mesh=None)])[0]
    loss_ctx = {"lm": lctx, "balancing": BalancingLossConfig().build(), "z_loss": ZLossConfig(z_loss_alpha=1e-2).build()}
    model.zero_grad(set_to_none=True)
    o = model(seq_ctx=seq_ctx, loss_ctx=loss_ctx)
    fields = {k: getattr(o, k) for k in type(o).model_fields}
    total = sum(v for k, v in fields.items() if "loss" in k and isinstance(v, torch.Tensor) and v.requires_grad)
    total.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}
    return ({k: float(fields[k]) for k in LOSSES}, grads, fields["tokens_per_expert_global"].clone())


def worst(a, b):
    w, name = 0.0, ""
    for k in b:
        d = (a[k] - b[k]).abs().max().item() / max(b[k].abs().max().item(), 1e-12)
        if d > w:
            w, name = d, k
    return w, name


def main():
    import torch

    os.environ["XTUNER_REFERENCE_ROOT"] = REF
    from tests.golden import ref_shim

    ref_shim.REFERENCE_ROOT = REF
    ref_shim.import_reference()
    import torch.distributed as dist

    from tests.workers.router_replay_worker import build_model
    from xtuner_b200 import ops, plugin

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=os.environ.get("MASTER_PORT", "29717"), RANK="0", WORLD_SIZE="1",
                      LOCAL_RANK="0")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    calls = [0]
    stats = ops.moe_aux_stats

    def counting(*a, **kw):
        calls[0] += 1
        return stats(*a, **kw)

    ops.moe_aux_stats = counting
    out = {}
    for kind, mode, kw in (("greedy", "fused", {"fused": True}), ("greedy", "per_op", {}), ("noaux", "per_op", {})):
        model, cfg = build_model(kind)
        plugin.convert_model(model, **kw)
        base_l, base_g, base_tpe = step(model, cfg)
        again_l, again_g, _ = step(model, cfg)
        plugin.install_moe_aux_loss()
        calls[0] = 0
        l, g_, tpe = step(model, cfg)
        n_calls = calls[0]
        plugin.uninstall_moe_aux_loss()
        plugin.restore_model(model)
        w, wn = worst(g_, base_g)
        out[f"{kind}/{mode}"] = {
            "layers": cfg.num_hidden_layers, "aux_calls": n_calls, "tpe_equal": bool(torch.equal(tpe, base_tpe)),
            "losses": l, "loss_rel_diff": {k: abs(l[k] - base_l[k]) / abs(base_l[k]) for k in LOSSES},
            "noise": {k: abs(again_l[k] - base_l[k]) / abs(base_l[k]) for k in LOSSES},
            "same_grad_keys": set(g_) == set(base_g), "worst_grad_rel_to_max": w, "worst_grad": wn,
            "grad_noise": worst(again_g, base_g)[0],
        }
    ops.moe_aux_stats = stats
    print("MOEAUXLOSS " + json.dumps(out), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
