"""Golden vectors for the MoE auxiliary-loss statistics (``tests/golden/moe_aux_loss.pt``), made on the CPU by the
REFERENCE'S OWN ``AuxLossContext``, ``BalancingLossContext`` and ``ZLossContext`` (loss/aux_loss.py, loss/moe_loss.py),
imported through ``ref_shim``:

    python tests/golden/make_moe_aux_loss_golden.py

Per case, ``L`` layers of ``AuxLossContext.accumulate`` over fp32 router logits ``[N, E]``, their softmax as the router
weights and int64 top-k ids ``[N, K]``, with a list of ``B`` balancing and ``B`` z contexts (``build_batches`` sets their
batch size), then ``finalize``, then the backward of the balancing loss plus a weighted sum of the carrier hidden states
(which brings in every layer's z-loss through ``AuxLossScaler``).  A gloo process group of one rank is up, so the
global-average branches run where the case turns them on.  Stored: the inputs, the per-layer counts, both losses after
``finalize``, the returned global counts and the gradients at the weights and the logits.
"""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ref_shim.apply_cpu_patches()

from make_golden import save  # noqa: E402
from xtuner.v1.loss.aux_loss import AuxLossConfig  # noqa: E402
from xtuner.v1.loss.moe_loss import BalancingLossConfig, BalancingLossContext, ZLossConfig, ZLossContext  # noqa: E402

H = 16  # width of the carrier hidden states
CASES = {  # name: (E, K, N, layers, contexts, z alpha, global average, experts the ids avoid)
    "e8k2": (8, 2, 64, 3, 1, 1e-3, True, ()),
    "e128k8": (128, 8, 48, 2, 1, 1e-3, False, tuple(range(100, 128))),
    "batch2": (8, 2, 40, 2, 2, 1e-2, True, (3,)),
    "zalpha0": (8, 2, 32, 2, 1, 0.0, False, ()),
    "n0": (8, 2, 0, 2, 1, 1e-3, False, ()),
}


def run_case(seed: int, E: int, K: int, N: int, layers: int, B: int, alpha: float, glob: bool, avoid) -> dict:
    g = torch.Generator().manual_seed(seed)
    aux = AuxLossConfig().build(n_routed_experts=E, num_experts_per_tok=K)
    bal = BalancingLossContext.build_batches(
        [BalancingLossConfig(balancing_loss_global_average=glob).build() for _ in range(B)])
    zs = ZLossContext.build_batches([ZLossConfig(z_loss_alpha=alpha, z_loss_global_average=glob).build() for _ in range(B)])
    num_tokens_global = torch.tensor(N, dtype=torch.int64) if glob else None
    hidden = torch.randn(N, H, generator=g).requires_grad_(True)
    h = hidden
    out, leaves = {}, []
    for l in range(layers):
        logits = (torch.randn(N, E, generator=g) * 2).requires_grad_(True)
        masked = logits.detach().clone()
        if avoid:
            masked[:, list(avoid)] = -float("inf")
        ids = masked.topk(K, dim=-1).indices.to(torch.int64)
        rw = torch.softmax(logits, dim=-1)
        rw.retain_grad()
        h = aux.accumulate(selected_router_weights=rw, selected_router_logits=logits, selected_experts=ids, hidden_states=h,
                           balancing_ctx=bal, z_ctx=zs, num_tokens_local=N, num_tokens_global=num_tokens_global,
                           world_size=1)
        out[f"rw{l}"], out[f"logits{l}"], out[f"ids{l}"] = rw.detach().clone(), logits.detach().clone(), ids
        out[f"tpe{l}"] = aux._local_load_logits_list[-1].clone()
        leaves.append((rw, logits))
    bal_loss, z_loss, tpe_global = aux.finalize(balancing_ctx=bal, z_ctx=zs, non_pad_token=N)
    w = torch.randn(N, H, generator=g)
    (bal_loss + (h * w).sum()).backward()
    out.update({"balancing_loss": bal_loss.detach(), "z_loss": z_loss.detach(), "tpe_global": tpe_global,
                "w": w, "hidden": hidden.detach(), "hidden_grad": hidden.grad})
    for l, (rw, logits) in enumerate(leaves):
        out[f"g_rw{l}"] = rw.grad if rw.grad is not None else torch.zeros_like(rw)
        out[f"g_logits{l}"] = logits.grad if logits.grad is not None else torch.zeros_like(logits)
    return out


def main():
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=os.environ.get("MASTER_PORT", "29711"), RANK="0",
                      WORLD_SIZE="1", LOCAL_RANK="0")
    dist.init_process_group("gloo", rank=0, world_size=1)
    out = {"cases": list(CASES)}
    for i, (name, spec) in enumerate(CASES.items()):
        out[f"{name}.spec"] = list(spec[:7])
        for key, v in run_case(2000 + i, *spec).items():
            out[f"{name}.{key}"] = v
    dist.destroy_process_group()
    save("moe_aux_loss", out)


if __name__ == "__main__":
    main()
