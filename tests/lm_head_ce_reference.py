"""Plain-torch restatement of the reference's lm_head cross-entropy (test infrastructure only; nothing under
``xtuner_b200/`` imports it), and float64 formulas for the pieces of ``xtb_lm_head_ce``.

:func:`lm_head_ce` follows ``LMHeadLossContext`` of ``xtuner/v1/loss/ce_loss.py``:

* mode "eager" (``chunk_size=None``), ``loss_fn``: ``logits = F.linear(h, W).float()``; ``loss = sum(CE(logits, labels,
  reduction="none", ignore_index) * loss_weight)``, or ``logits.sum() * 0`` when no row counts; autograd gives ``dh`` and
  ``dW`` for a loss gradient ``grad_output``.
* mode "chunk", ``ChunkLoss`` (``loss/chunk_loss.py``): ``loss_fn`` per chunk of ``chunk_size`` rows with its gradients
  taken right away, the chunk losses added into an fp32 zero, the chunk ``dW`` added into a bf16 zero, and both
  gradients multiplied by ``grad_output`` when it is not 1.

On the CPU it reproduces the reference bit for bit (``tests/test_lm_head_ce_cpu.py`` checks it against fixtures made by the
reference's own classes); on a GPU it is the reference's arithmetic on cuBLAS and torch's CUDA kernels.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _loss_fn(h, w, labels, loss_weight, ignore_index):
    logits = F.linear(h, w).float()
    if int((labels != ignore_index).sum()) == 0:
        return logits.sum() * 0
    return (F.cross_entropy(logits, labels, reduction="none", ignore_index=ignore_index) * loss_weight).sum()


def lm_head_ce(hidden, weight, labels, loss_weight, ignore_index=-100, chunk_size=None, grad_output=1.0):
    """-> (loss fp32 scalar, dh [rows, H] bf16, dW [V, H] bf16) for ``hidden`` [..., H] and one label / weight per row."""
    h = hidden.detach().reshape(-1, hidden.shape[-1])
    w = weight.detach()
    lab = labels.reshape(-1)
    lw = loss_weight.reshape(-1)
    g = torch.as_tensor(grad_output, dtype=torch.float32, device=h.device)
    if chunk_size is None:
        hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
        with torch.enable_grad():
            loss = _loss_fn(hh, ww, lab, lw, ignore_index)
            dh, dw = torch.autograd.grad(loss, (hh, ww), g)
        return loss.detach(), dh, dw
    loss = torch.tensor(0.0, device=h.device)
    dh = torch.empty_like(h)
    dw = torch.zeros_like(w)
    ww = w.clone().requires_grad_(True)
    for s in range(0, h.shape[0], chunk_size):
        hc = h[s:s + chunk_size].clone().requires_grad_(True)
        with torch.enable_grad():
            lc = _loss_fn(hc, ww, lab[s:s + chunk_size], lw[s:s + chunk_size], ignore_index)
            dhc, dwc = torch.autograd.grad(lc, (hc, ww))
        loss.add_(lc.detach())
        dh[s:s + chunk_size].copy_(dhc)
        dw.add_(dwc)
    if float(g) != 1.0:
        dh, dw = dh * g, dw * g
    return loss, dh, dw


# ---- float64 formulas of the kernel's pieces ---------------------------------------------------------------------------


def logsumexp64(z: torch.Tensor) -> torch.Tensor:
    """per-row log(sum(exp(z))) of bf16 logits, in float64"""
    return torch.logsumexp(z.double(), dim=-1)


def row_ce64(z: torch.Tensor, labels: torch.Tensor, ignore_index: int) -> torch.Tensor:
    """ce_t = logsumexp(z_t) - z_t[label_t] in float64; 0 for ignored rows"""
    keep = labels != ignore_index
    safe = torch.where(keep, labels, torch.zeros_like(labels))
    ce = logsumexp64(z) - z.double().gather(1, safe[:, None])[:, 0]
    return torch.where(keep, ce, torch.zeros_like(ce))


def grad64(z: torch.Tensor, labels: torch.Tensor, loss_weight: torch.Tensor, ignore_index: int) -> torch.Tensor:
    """G = (softmax(z) - onehot(label)) * w in float64; 0 for ignored rows"""
    keep = labels != ignore_index
    p = torch.softmax(z.double(), dim=-1)
    safe = torch.where(keep, labels, torch.zeros_like(labels))
    p.scatter_add_(1, safe[:, None], -torch.ones_like(p[:, :1]))
    g = p * loss_weight.double()[:, None]
    return torch.where(keep[:, None], g, torch.zeros_like(g))
