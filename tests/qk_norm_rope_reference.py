"""Exact restatements, float64 references and bounds for ``xtb_qk_norm_rope`` / ``xtb_qk_norm_rope_bwd``
(``csrc/qk_norm_rope.cu``): q_norm / k_norm (``F.rms_norm``) followed by ``apply_rotary_pos_emb_cuda``, as
``MultiHeadAttention.forward`` runs them.  Test infrastructure only; nothing under ``xtuner_b200/`` imports it.  Plain
torch on whatever device the operands are on.  Operands are [T, H, D] (any strides), cos / sin [T, D], weights [D].

Exact restatements (a correct kernel, and the reference's autograd, match them bit for bit):

  :func:`forward`   n = bf16((x rstd) w) given an fp32 rstd (n = x without a weight), then
                    out = bf16(bf16(n cos) + bf16(rotate_half(n) sin)).
  :func:`grad_n`    gn_i = bf16(bf16(g_i cos_i) + bf16(g_{i+D/2} sin_{i+D/2})) for i < D/2 and
                    gn_i = bf16(bf16(g_i cos_i) - bf16(g_{i-D/2} sin_{i-D/2})) otherwise: autograd through the two products,
                    the ``cat`` and the negation of ``rotate_half``, and the sum of the two branches.

float64 references and bounds (u = 2^-24; ``gamma``, ``rstd_rel``, ``g_h_ref`` and the checkers come from
``tests/norm_combine_reference.py``; the depths are counted from the kernels, where a row of D values is held by L = D/8
lanes, 8 values each):

  ``rstd``  each lane chains 8 fmaf, then a log2(L)-level butterfly (3, 4, 5 levels for D = 64, 128, 256): at most 13
            roundings of a sum of positive terms, /D exact, + eps one more.  ``rstd_rel(D)`` covers a depth of
            D/32 + 14 >= 16, so it holds here.
  ``dx``    (w gn - x c) rstd with c = (sum w gn x) rstd^2 / D: w gn rounds once, the dot is 8 fmaf and a butterfly of
            at most 5 levels, c three more roundings, x c, the difference and the product one each: at most 20 roundings,
            inside the 32 of ``g_h_ref``'s bound.  Checked with the near-tie checker against that fp64 value, computed from
            the exact ``gn`` and the kernel's own rstd.
  ``dw``    sum over (t, h) of fl(gn rstd) x: a thread fmaf-chains the rows it owns (one per 8 L-lane slots of a CTA
            per pass: ceil(4 H / (256 / L)) per token group, 4 tokens a group, over ceil(n_groups / n_cta) groups), a CTA
            adds its 256/L slots in order, and the partial rows of the n_cta CTAs are added by 32 warps in order
            (ceil(n_cta / 32) each) and the 32 warp sums in order: :func:`dw_depth` roundings of a sum bounded by
            sum |gn x rstd|.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from tests.norm_combine_reference import g_h_ref, gamma, rstd_ref

TOKENS_PER_CTA = 4


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def _b(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).float()


def norm(x: torch.Tensor, rstd: Optional[torch.Tensor], w: Optional[torch.Tensor]) -> torch.Tensor:
    """bf16 [T, H, D]: bf16((x rstd) w), or x without a weight"""
    if w is None:
        return x
    return ((x.float() * rstd[..., None]) * w.float()).to(torch.bfloat16)


def rope(n: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """bf16 [T, H, D]: bf16(bf16(n cos) + bf16(rotate_half(n) sin))"""
    c, s = cos.float()[:, None, :], sin.float()[:, None, :]
    return (_b(n.float() * c) + _b(rotate_half(n.float()) * s)).to(torch.bfloat16)


def forward(x: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, rstd: Optional[torch.Tensor] = None,
            w: Optional[torch.Tensor] = None) -> torch.Tensor:
    return rope(norm(x, rstd, w), cos, sin)


def grad_n(g: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor) -> torch.Tensor:
    """bf16 [T, H, D]: the gradient at the norm output (the input gradient without the norm)"""
    h = g.shape[-1] // 2
    gf = g.float()
    a = _b(gf * cos.float()[:, None, :])
    s = _b(gf * sin.float()[:, None, :])
    partner = torch.cat((s[..., h:], -s[..., :h]), dim=-1)
    return (a + partner).to(torch.bfloat16)


def rstd_torch(x: torch.Tensor, eps: float) -> torch.Tensor:
    """fp32 [T, H]: the rstd torch's composite ``F.rms_norm`` computes (fp32 mean of squares, then rsqrt)"""
    return torch.rsqrt(x.float().pow(2).mean(-1) + eps)


def rstd_fp64(x: torch.Tensor, eps: float) -> torch.Tensor:
    return rstd_ref(x.reshape(-1, x.shape[-1]), eps).view(x.shape[:-1])


def dx_ref(gn: torch.Tensor, x: torch.Tensor, rstd: torch.Tensor, w: torch.Tensor
           ) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(dx, bound)`` in float64 [T, H, D] from the exact gn and the kernel's rstd"""
    T, H, D = x.shape
    ref, bound = g_h_ref(gn.reshape(-1, D), x.reshape(-1, D), rstd.reshape(-1), w.float())
    return ref.view(T, H, D), bound.view(T, H, D)


def dw_depth(T: int, H: int, D: int, n_cta: int) -> int:
    L = D // 8
    n_groups = -(-T // TOKENS_PER_CTA)
    rows = -(-n_groups // n_cta) * -(-TOKENS_PER_CTA * H // (256 // L))
    return rows + 1 + 256 // L + -(-n_cta // 32) + 32


def bwd_ctas(T: int, sm_count: int) -> int:
    """the backward's persistent grid: 2 CTAs per SM, at most one per token group"""
    return max(1, min(2 * sm_count, -(-T // TOKENS_PER_CTA)))


def dw_ref(gn: torch.Tensor, x: torch.Tensor, rstd: torch.Tensor, n_cta: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(dw, bound)`` in float64 [D]"""
    T, H, D = x.shape
    terms = (gn.double() * x.double() * rstd.double()[..., None]).reshape(-1, D)
    return terms.sum(0), gamma(dw_depth(T, H, D, n_cta)) * terms.abs().sum(0)
