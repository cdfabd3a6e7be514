"""Golden vectors for the lm_head cross-entropy (``tests/golden/lm_head_ce*.pt``), made by the REFERENCE'S OWN
``LMHeadLossContext`` (``xtuner/v1/loss/ce_loss.py``, imported through ``ref_shim``) on the CPU:

    python tests/golden/make_lm_head_ce_golden.py

One set of inputs (T = 300 rows of one packed batch of three sequences, H = 256, V = 1024, about 30 % of the labels
ignored, the second sequence entirely ignored, labels 0 and V - 1 present), run through ``build_batches`` and
``forward`` + ``backward`` in modes "eager" and "chunk" (chunk 128: chunks of 128, 128 and 44 rows) with "token" and
"sample" reduction, plus one batch whose every label is ignored.  Stored per case: the loss weight ``build_batches``
made, the loss, and the gradients of the hidden states and of the head weight.
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
from xtuner.v1.loss.ce_loss import CELossConfig, CELossKwargs, LMHeadLossContext  # noqa: E402

T, H, V, IGNORE = 300, 256, 1024, -100
CU_SEQ_LENS = [0, 120, 170, 300]  # sequence 1 (rows 120..169) has no counted label


def inputs():
    g = torch.Generator().manual_seed(4242)
    hidden = torch.randn(1, T, H, generator=g).to(torch.bfloat16)
    weight = (torch.randn(V, H, generator=g) * H ** -0.5).to(torch.bfloat16)
    labels = torch.randint(0, V, (1, T), generator=g)
    labels[torch.rand(1, T, generator=g) < 0.3] = IGNORE
    labels[0, CU_SEQ_LENS[1]:CU_SEQ_LENS[2]] = IGNORE
    labels[0, 5], labels[0, 6], labels[0, T - 1] = 0, V - 1, V - 1
    return hidden, weight, labels


def run_case(hidden, weight, labels, mode, reduction):
    cfg = CELossConfig(mode=mode, chunk_size=128, loss_reduction=reduction, ignore_idx=IGNORE)
    ctx = LMHeadLossContext(cfg, CELossKwargs(shifted_labels=labels.clone()))
    cu = torch.tensor(CU_SEQ_LENS, dtype=torch.int32)
    (ctx,) = LMHeadLossContext.build_batches([ctx], cu_seq_lens_list=[cu])
    h = hidden.clone().requires_grad_(True)
    w = weight.clone().requires_grad_(True)
    loss, _ = ctx.forward(h, w)
    loss.backward()
    return {"loss_weight": ctx.loss_kwargs.loss_weight.clone(), "loss": loss.detach().clone(), "dh": h.grad.clone(),
            "dw": w.grad.clone()}


def main():
    hidden, weight, labels = inputs()
    out = {"hidden": hidden, "weight": weight, "labels": labels, "ignore_index": IGNORE, "chunk_size": 128,
           "cu_seq_lens": torch.tensor(CU_SEQ_LENS)}
    for mode in ("eager", "chunk"):
        for reduction in ("token", "sample"):
            for k, v in run_case(hidden, weight, labels, mode, reduction).items():
                out[f"{mode}.{reduction}.{k}"] = v
        none = torch.full_like(labels, IGNORE)
        r = run_case(hidden, weight, none, mode, "token")
        out[f"{mode}.all_ignored.loss"] = r["loss"]
        out[f"{mode}.all_ignored.grad_nonzero"] = int(r["dh"].count_nonzero() + r["dw"].count_nonzero())
    save("lm_head_ce", out)


if __name__ == "__main__":
    main()
