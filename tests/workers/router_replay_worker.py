"""GPU worker: the UNMODIFIED reference MoE models (the copy under oracle/_ref, see oracle/make_ref.py) trained one step
with routing replay — ``seq_ctx.rollout_routed_experts`` set to one int64 [S, L, K] tensor — first on the reference's
own GPU path, then through ``xtuner_b200.plugin.convert_model`` per-op and (greedy router) with ``fused=True``.  Models:
the greedy-router MoE of tests/workers/reference_plugin_worker.py, and a DeepSeek-style one (NoAuxRouter with a group
mask and a correction bias, one shared expert).  For ``fused=True`` the step is also run with the ids in host memory and
``offload_rollout_routed_experts`` set, which the layer moves to the device as the reference's does.  Prints one JSON
line; tests/test_gpu_router_replay_reference.py asserts on it."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref")


def build_model(kind):
    import torch
    from xtuner.v1.model.moe.moe import MoE, MoEConfig
    from xtuner.v1.module.attention import MHAConfig
    from xtuner.v1.module.router import GreedyRouterConfig, NoAuxRouterConfig

    if kind == "greedy":
        router, E, K, shared = GreedyRouterConfig(scoring_func="softmax", router_scaling_factor=1.0, norm_topk_prob=True), 8, 2, 0
    else:
        router = NoAuxRouterConfig(scoring_func="sigmoid", router_scaling_factor=2.5, norm_topk_prob=True, n_group=4, topk_group=2)
        E, K, shared = 32, 4, 1
    cfg = MoEConfig(
        vocab_size=1024, max_position_embeddings=1024, pad_token_id=0, eos_token_id=0, num_hidden_layers=2, hidden_size=256,
        intermediate_size=512, rms_norm_eps=1e-6, rope_theta=1e6, hidden_act="silu",
        attention=MHAConfig(num_attention_heads=4, num_key_value_heads=2, head_dim=64, attn_impl="eager_attention"),
        tie_word_embeddings=False, n_routed_experts=E, n_shared_experts=shared, num_experts_per_tok=K,
        first_k_dense_replace=0, hidden_factor=1.0, moe_intermediate_size=128, router=router, compile_cfg=False,
    )
    torch.manual_seed(0)
    model = MoE(config=cfg)
    model.init_weights()
    with torch.no_grad():
        for m in model.modules():
            if hasattr(m, "e_score_correction_bias"):
                m.e_score_correction_bias.copy_(torch.randn_like(m.e_score_correction_bias) * 0.05)
    return model.to(torch.bfloat16).cuda(), cfg


def compare(kind, out):
    import torch
    from xtuner.v1.loss.ce_loss import CELossConfig
    from xtuner.v1.model.moe.moe import SequenceContext

    from xtuner_b200 import _capi, fused, plugin

    model, cfg = build_model(kind)
    S, L, K, E, V = 512, cfg.num_hidden_layers, cfg.num_experts_per_tok, cfg.n_routed_experts, cfg.vocab_size
    g = torch.Generator().manual_seed(7)
    input_ids = torch.randint(0, V, (1, S + 1), dtype=torch.int64, generator=g).cuda()
    replay = torch.randint(0, E, (S, L, K), dtype=torch.int64, generator=g)
    replay[::3, :, 0] = replay[::3, :, -1]  # duplicates, as the reference's own padding ids may have
    replay_dev = replay.cuda()
    ids_seen = []

    def hook(_m, _inp, res):
        ids_seen.append(res["topk_ids"].detach().clone())

    handles = [m.gate.register_forward_hook(hook) for m in model.modules() if hasattr(m, "dispatcher") and hasattr(m, "gate")]
    block = fused.fused_moe_block

    def block_spy(*a, **kw):  # the fused node does not call the gate module
        o, rr = block(*a, **kw)
        ids_seen.append(rr["topk_ids"].detach().clone())
        return o, rr

    fused.fused_moe_block = block_spy

    def run(ids, offload=False):
        ids_seen.clear()
        seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cuda")
        seq_ctx.rollout_routed_experts = ids
        seq_ctx.offload_rollout_routed_experts = offload
        loss_cfg = CELossConfig()
        lctx = loss_cfg.build(data={"shifted_labels": input_ids[:, 1:]}, sp_mesh=None)
        lctx = loss_cfg.loss_ctx_cls.build_batches([lctx])[0]
        model.zero_grad(set_to_none=True)
        o = model(seq_ctx=seq_ctx, loss_ctx={"lm": lctx})
        fields = {k: getattr(o, k) for k in type(o).model_fields} if hasattr(type(o), "model_fields") else dict(o)
        total = sum(v for k, v in fields.items() if "loss" in k and isinstance(v, torch.Tensor) and v.requires_grad)
        total.backward()
        torch.cuda.synchronize()
        grads = {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}
        return float(total), grads, [t.clone() for t in ids_seen]

    def replayed(ids):
        return [bool(len(ids) == L)] + [bool(torch.equal(ids[l].cpu(), replay[:, l, :])) for l in range(min(len(ids), L))]

    ref_total, ref_g, ref_ids = run(replay_dev)
    ref2_total, _, _ = run(replay_dev)
    res = {"reference": {"total": ref_total, "rerun_total": ref2_total, "ids_replayed": replayed(ref_ids)}}
    lib = _capi.ensure_init()
    modes = (("per_op", {}), ("fused", {"fused": True})) if kind == "greedy" else (("per_op", {}),)
    for mode, kw in modes:
        lib.xtb_reset_launch_count()
        n = plugin.convert_model(model, **kw)
        total, g_, ids = run(replay_dev)
        launches = int(lib.xtb_launch_count())
        m = {"layers_converted": n, "total": total, "loss_rel_diff": abs(total - ref_total) / abs(ref_total),
             "same_grad_keys": set(g_) == set(ref_g), "ids_replayed": replayed(ids), "kernel_launches": launches}
        worst, worst_name = 0.0, ""
        for k in ref_g:
            d = (g_[k] - ref_g[k]).abs().max().item() / max(ref_g[k].abs().max().item(), 1e-12)
            if d > worst:
                worst, worst_name = d, k
        m.update(worst_grad_rel_to_max=worst, worst_grad=worst_name)
        # the ids in host memory with the offload flag: moved to the device by the layer, same result
        off_total, off_g, off_ids = run(replay, offload=True)
        m["offload_same"] = bool(off_total == total and all(torch.equal(off_g[k], g_[k]) for k in g_)
                                 and all(replayed(off_ids)))
        plugin.restore_model(model)
        res[mode] = m
    fused.fused_moe_block = block
    for h in handles:
        h.remove()
    out[kind] = res


def main():
    import torch

    os.environ["XTUNER_REFERENCE_ROOT"] = REF
    os.environ.setdefault("XTUNER_DETERMINISTIC", "true")
    from tests.golden import ref_shim

    ref_shim.REFERENCE_ROOT = REF
    ref_shim.import_reference()
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=os.environ.get("MASTER_PORT", "29697"), RANK="0", WORLD_SIZE="1",
                      LOCAL_RANK="0")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    out = {}
    for kind in ("greedy", "noaux"):
        compare(kind, out)
    print("ROUTERREPLAY " + json.dumps(out), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
