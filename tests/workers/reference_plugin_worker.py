"""GPU worker: the UNMODIFIED reference MoE model (the copy under oracle/_ref, see oracle/make_ref.py) on an
H100 — first on the reference's own GPU path (Triton grouped GEMM, torch-fallback permute/unpermute), then with
``xtuner_b200.plugin.convert_model`` (per-op classes) and ``convert_model(fused=True)`` (one autograd node per MoE half).
The recipe is the reference's ``tests/model/test_moe.py:57-148`` (tiny random-init MoE, same batch through two
dispatcher implementations).  Prints one JSON line; tests/test_gpu_reference_plugin.py asserts on it."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.path.join(ROOT, "oracle", "_ref")


def main():
    import torch

    os.environ["XTUNER_REFERENCE_ROOT"] = REF
    os.environ.setdefault("XTUNER_DETERMINISTIC", "true")  # parity run: pins Triton autotune (xtuner/v1/__init__.py:14-21)
    from tests.golden import ref_shim

    ref_shim.REFERENCE_ROOT = REF
    ref_shim.import_reference()
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=os.environ.get("MASTER_PORT", "29695"), RANK="0", WORLD_SIZE="1",
                      LOCAL_RANK="0")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    from xtuner.v1.loss.ce_loss import CELossConfig
    from xtuner.v1.model.moe.moe import MoE, MoEConfig, SequenceContext
    from xtuner.v1.module.attention import MHAConfig
    from xtuner.v1.module.router import GreedyRouterConfig
    from xtuner.v1.ops import moe as ref_ops

    H, I, E, K, L, S, V = 256, 128, 8, 2, 2, 512, 1024
    cfg = MoEConfig(
        vocab_size=V, max_position_embeddings=1024, pad_token_id=0, eos_token_id=0, num_hidden_layers=L, hidden_size=H,
        intermediate_size=512, rms_norm_eps=1e-6, rope_theta=1e6, hidden_act="silu",
        attention=MHAConfig(num_attention_heads=4, num_key_value_heads=2, head_dim=64, attn_impl="eager_attention"),
        tie_word_embeddings=False, n_routed_experts=E, n_shared_experts=0, num_experts_per_tok=K, first_k_dense_replace=0,
        hidden_factor=1.0, moe_intermediate_size=I,
        router=GreedyRouterConfig(scoring_func="softmax", router_scaling_factor=1.0, norm_topk_prob=True), compile_cfg=False,
    )
    torch.manual_seed(0)
    model = MoE(config=cfg)
    model.init_weights()
    model = model.to(torch.bfloat16).cuda()
    out = {"reference_ops": {n: getattr(getattr(ref_ops, n), "__name__", "?") for n in ("group_gemm", "permute", "unpermute")}}

    torch.manual_seed(123)
    input_ids = torch.randint(0, V, (1, S + 1), dtype=torch.int64, device="cuda")
    ids_seen = []

    def hook(_m, _inp, res):
        ids_seen.append(res["topk_ids"].detach().clone())

    gates = [m.gate for m in model.modules() if hasattr(m, "dispatcher") and hasattr(m, "gate")]
    handles = [g.register_forward_hook(hook) for g in gates]

    def run():
        ids_seen.clear()
        seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cuda")
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
        scal = {k: float(v) for k, v in fields.items() if isinstance(v, torch.Tensor) and v.numel() == 1}
        return scal, grads, [t.clone() for t in ids_seen], float(total)

    ref_scal, ref_g, ref_ids, ref_total = run()
    ref2_scal, _, _, ref2_total = run()  # run-to-run noise of the reference path itself (atomics / autotune)
    out["reference"] = {"losses": ref_scal, "total": ref_total, "rerun_total": ref2_total}

    from xtuner_b200 import _capi, plugin

    lib = _capi.ensure_init()
    for mode, kw in (("per_op", {}), ("fused", {"fused": True})):
        lib.xtb_reset_launch_count()
        n = plugin.convert_model(model, **kw)
        scal, g, ids, total = run()
        plugin.restore_model(model)
        rel = abs(total - ref_total) / abs(ref_total)
        worst = 0.0
        worst_name = ""
        for k in ref_g:
            d = (g[k] - ref_g[k]).abs().max().item() / max(ref_g[k].abs().max().item(), 1e-12)
            if d > worst:
                worst, worst_name = d, k
        ids_equal = [bool(torch.equal(a, b)) for a, b in zip(ids, ref_ids)]
        ids_agree = [float((a == b).float().mean()) for a, b in zip(ids, ref_ids)]
        out[mode] = {"layers_converted": n, "losses": scal, "total": total, "loss_rel_diff": rel, "same_grad_keys": set(g) == set(ref_g),
                     "worst_grad_rel_to_max": worst, "worst_grad": worst_name, "topk_ids_equal": ids_equal,
                     "topk_ids_agreement": ids_agree, "kernel_launches": int(lib.xtb_launch_count())}
    back_scal, _, _, back_total = run()
    out["restored_total"] = back_total
    for h in handles:
        h.remove()

    # ---- the same comparison under the reference's FSDP wrapping (model/moe/moe.py:1144-1313: fp32 master params as
    # DTensors, bf16 MixedPrecisionPolicy, per-layer fully_shard, activation checkpointing at the default ratio) ----------
    try:
        from xtuner.v1.config import FSDPConfig

        torch.manual_seed(0)
        model = MoE(config=cfg)
        model.init_weights()
        model = model.cuda().fully_shard(FSDPConfig(torch_compile=False))
        gates = [m.gate for m in model.modules() if hasattr(m, "dispatcher") and hasattr(m, "gate")]
        handles = [g.register_forward_hook(hook) for g in gates]

        def full(g):
            return (g.full_tensor() if hasattr(g, "full_tensor") else g).detach().float().clone()

        def run_fsdp():
            ids_seen.clear()
            seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cuda")
            loss_cfg = CELossConfig()
            lctx = loss_cfg.build(data={"shifted_labels": input_ids[:, 1:]}, sp_mesh=None)
            lctx = loss_cfg.loss_ctx_cls.build_batches([lctx])[0]
            model.zero_grad(set_to_none=True)
            o = model(seq_ctx=seq_ctx, loss_ctx={"lm": lctx})
            fields = {k: getattr(o, k) for k in type(o).model_fields} if hasattr(type(o), "model_fields") else dict(o)
            total = sum(v for k, v in fields.items() if "loss" in k and isinstance(v, torch.Tensor) and v.requires_grad)
            total.backward()
            torch.cuda.synchronize()
            grads = {n: full(p.grad) for n, p in model.named_parameters() if p.grad is not None}
            return grads, [t.clone() for t in ids_seen[: len(gates)]], float(total)

        fg, fids, ftotal = run_fsdp()
        st = {"reference_total": ftotal}
        lib.xtb_reset_launch_count()
        n = plugin.convert_model(model, fused=True)
        plugin.install_fsdp_comm(model)
        g, ids, total = run_fsdp()
        plugin.restore_model(model)
        worst = max((g[k] - fg[k]).abs().max().item() / max(fg[k].abs().max().item(), 1e-12) for k in fg)
        st.update(layers_converted=n, total=total, loss_rel_diff=abs(total - ftotal) / abs(ftotal), same_grad_keys=set(g) == set(fg),
                  worst_grad_rel_to_max=worst, topk_ids_equal=[bool(torch.equal(a, b)) for a, b in zip(ids, fids)],
                  kernel_launches=int(lib.xtb_launch_count()), ok=True)
        out["fsdp_fused"] = st
    except Exception as e:  # noqa: BLE001 — reported, not fatal: the un-sharded comparison above is the pinned one
        import traceback

        out["fsdp_fused"] = {"ok": False, "error": f"{type(e).__name__}: {e}"[:400], "traceback": traceback.format_exc()[-1500:]}
    print("REFPLUGIN " + json.dumps(out), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
