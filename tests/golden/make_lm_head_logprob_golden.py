"""Golden vectors for the lm_head log-probabilities and the GRPO loss (``tests/golden/lm_head_logprob.pt``), made by the
REFERENCE'S OWN ``LogProbContext`` (``xtuner/v1/loss/rl_loss.py``) and ``GRPOLossContext``
(``xtuner/v1/rl/loss/grpo_loss.py``), imported through ``ref_shim``, on the CPU:

    python tests/golden/make_lm_head_logprob_golden.py

One packed batch of T = 128 rows, H = 128, V = 256, about 30 % of the labels ignored (-100), labels 0 and V - 1 present.

* ``logprob.{eager,chunk}``: ``LogProbContext.forward`` under ``no_grad`` (chunk 48: chunks of 48, 48 and 32 rows).
* ``grpo.{eager,chunk}.{none,k1,low_var_kl}``: ``build_batches`` then ``forward`` + ``backward(grad_output)`` with the
  vanilla policy loss (clip 0.2 / 0.28, clip_ratio_c 3), without KL and with ``kl_loss_type`` k1 and low_var_kl
  (coefficient 0.1).  ``old_logprobs`` are the eager log-probabilities shifted per position so that the ratios fall on
  1 exactly (the tie in ``torch.maximum``), inside the clip range, below 1 - 0.2, above 1 + 0.28 and above
  ``clip_ratio_c``; the advantages are positive, negative and zero.  Stored per case: the loss and every ``extra_info``
  entry; for three cases, among them two with ``grad_output != 1``, also the gradients of the hidden states and weight.
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
from xtuner.v1.loss.rl_loss import LogProbConfig, LogProbContext  # noqa: E402
from xtuner.v1.rl.loss.grpo_loss import GRPOLossConfig, GRPOLossContext, GRPOLossKwargs  # noqa: E402

T, H, V, IGNORE, CHUNK = 128, 128, 256, -100, 48
POLICY = {"loss_type": "vanilla", "cliprange_low": 0.2, "cliprange_high": 0.28, "clip_ratio_c": 3.0}
KL_COEF = 0.1
# (mode, kl type, grad_output, store the gradients)
GRPO_CASES = [("eager", None, 1.0, True), ("eager", "k1", 0.3, True), ("eager", "low_var_kl", 1.0, False),
              ("chunk", None, 1.0, False), ("chunk", "k1", 1.0, False), ("chunk", "low_var_kl", 0.3, True)]
# logp - old_logp per position, cycled: ratio 1 exactly, inside the clip range, below 0.8, above 1.28, above 3
LOG_RATIOS = [0.0, 0.1, -0.05, -0.3, 0.3, 1.5, -1.0, 0.0, 2.5]


def inputs():
    g = torch.Generator().manual_seed(5151)
    hidden = torch.randn(1, T, H, generator=g).to(torch.bfloat16)
    weight = (torch.randn(V, H, generator=g) * H ** -0.5 * 2).to(torch.bfloat16)
    labels = torch.randint(0, V, (1, T), generator=g)
    labels[torch.rand(1, T, generator=g) < 0.3] = IGNORE
    labels[0, 3], labels[0, 4], labels[0, T - 1] = 0, V - 1, V - 1
    advantages = torch.tensor([1.3, -0.7, 0.0, 0.4, -2.0])[torch.randint(0, 5, (1, T), generator=g)]
    ref_noise = torch.randn(1, T, generator=g) * 0.4
    return hidden, weight, labels, advantages, ref_noise


def logprobs_of(hidden, weight, labels, mode):
    ctx = LogProbConfig(mode=mode, chunk_size=CHUNK, ignore_idx=IGNORE).build({"shifted_labels": labels.clone()})
    (ctx,) = LogProbContext.build_batches([ctx])
    with torch.no_grad():
        logprobs, _ = ctx.forward(hidden, weight)
    return logprobs


def grpo_case(hidden, weight, labels, old, ref, advantages, mode, kl, grad_output):
    cfg = GRPOLossConfig(policy_loss_cfg=dict(POLICY), use_kl_loss=kl is not None, kl_loss_coef=KL_COEF,
                         kl_loss_type=kl, mode=mode, chunk_size=CHUNK, ignore_idx=IGNORE)
    kw = GRPOLossKwargs(shifted_labels=labels.clone(), old_logprobs=old.clone(), advantages=advantages.clone(),
                        ref_logprobs=ref.clone())
    (ctx,) = GRPOLossContext.build_batches([GRPOLossContext(cfg, kw)])
    h = hidden.clone().requires_grad_(True)
    w = weight.clone().requires_grad_(True)
    loss, (_, extra) = ctx.forward(h, w)
    loss.backward(torch.tensor(grad_output))
    return loss.detach(), {k: v.detach().clone() for k, v in extra.items()}, h.grad, w.grad


def main():
    hidden, weight, labels, advantages, ref_noise = inputs()
    out = {"hidden": hidden, "weight": weight, "labels": labels, "advantages": advantages, "ignore_index": IGNORE,
           "chunk_size": CHUNK, "policy_loss_cfg": dict(POLICY), "kl_loss_coef": KL_COEF}
    for mode in ("eager", "chunk"):
        out[f"logprob.{mode}"] = logprobs_of(hidden, weight, labels, mode)
    logp = out["logprob.eager"]
    shift = torch.tensor(LOG_RATIOS)[torch.arange(T) % len(LOG_RATIOS)].view(1, T)
    old = logp - shift  # a shift of 0 leaves logp - old == 0 exactly
    out["old_logprobs"], out["ref_logprobs"] = old, logp + ref_noise
    for mode, kl, grad_output, keep_grads in GRPO_CASES:
        key = f"grpo.{mode}.{kl or 'none'}"
        loss, extra, dh, dw = grpo_case(hidden, weight, labels, old, out["ref_logprobs"], advantages, mode, kl,
                                        grad_output)
        out[f"{key}.grad_output"], out[f"{key}.loss"], out[f"{key}.extra_info"] = grad_output, loss, extra
        if keep_grads:
            out[f"{key}.dh"], out[f"{key}.dw"] = dh, dw
    save("lm_head_logprob", out)


if __name__ == "__main__":
    main()
