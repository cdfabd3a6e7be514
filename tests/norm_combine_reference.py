"""Exact restatements, float64 references, checkers and input generators for the memory-bound kernels around the
grouped GEMMs in ``FusedMoEBlock``: ``xtb_rmsnorm_gate`` and ``xtb_moe_dispatch_bwd_rmsnorm`` (``csrc/norm.cu``),
``xtb_moe_combine`` / ``xtb_moe_unpermute`` and ``xtb_moe_unpermute_bwd`` (``csrc/permute.cu``).  Test infrastructure
only; nothing under ``xtuner_b200/`` imports it.  Plain torch on whatever device the operands are on.

Exact restatements (fp32 torch, the kernels' documented rounding points; a correct kernel matches them bit for bit):

  :func:`combine`      acc = p_0 y_0 (+ p_1 y_1) (+ ...), each product rounded to fp32 and added in k order starting
                       from the k = 0 product (a row mapped to -1 adds nothing); then bf16(acc), then bf16(. * hf) when
                       hf != 1, then bf16(. + residual) when a residual is given.
  :func:`act_grad`     unpermute backward: act_grad[row(t, k)] = bf16(fp32(g[t]) * p[t, k]).
  :func:`dispatch_gx`  dispatch backward: g_x = bf16(bf16(sum_k g_xp[row(t, k)]) + g_x_gate), fp32 sum in k order.
  :func:`rmsnorm_x`    x = bf16((h * rstd) * w) given the kernel's own fp32 rstd.
  The residual of the dispatch backward is a composition: g_h(res) = bf16(bf16(g_h(no res)) + g_res).

float64 references and their bounds (u = 2^-24, fp32 round-to-nearest; gamma(n) = n u / (1 - n u), the classic bound
on n successive roundings of a sum whose partial sums are at most S = sum |terms|; every reduction below is a fixed
tree of fp32 adds or fmas whose depth is counted from the kernel):

  ``rstd``      1/sqrt(mean(h^2) + eps).  Both norm kernels sum h^2 with fmaf: the column kernel 8 per thread, a 5-level
                warp butterfly and 8 warp partials in order (20 roundings); the gate kernel H/32 per lane and the
                butterfly.  n = H/32 + 13 covers both.  The terms are positive, so the sum is off by gamma(n) relative;
                /H is exact (H is a power of two), + eps rounds once, and rsqrtf is within 2 ulp (4u relative).  A
                square root halves a relative error: |err| <= ((n + 1) / 2 gamma-ish + 4u) rstd, :func:`rstd_rel`.
  ``x``         h rstd w before the bf16 round is off by rstd_rel + 2u relative (two fp32 products).
  ``logits``    sum_h x w of the kernel's own bf16 x: fmaf chains of H/32 per lane and a 5-level butterfly,
                |err| <= gamma(H/32 + 6) sum |x w|.
  ``prob_grad`` sum_h g y: each lane chains 8 fmaf per 16-byte vector over ceil(H/256) vectors, then the butterfly,
                |err| <= gamma(8 ceil(H/256) + 6) sum |g y|.
  ``g_h``       before the residual, (w g - h c) rstd with c = (sum_h w g h) rstd^2 / H.  The dot is one fmaf per
                column per thread (8), the butterfly (5) and 8 warp partials (8), after w g rounds once: 22; c adds three
                roundings, h c, the difference and the final product one each: 28 in all, taken as 32.  Each rounding
                is relative to a quantity no larger than S = rstd (|w g| + |h| rstd^2 sum_h |w g h| / H), so
                |err| <= gamma(32) S (:func:`g_h_ref`).
  ``g_norm_w``  sum_t g_x h rstd: fl(g_x rstd) then one fmaf per token into a per-CTA register (a CTA walks at most
                ceil(T / n_cta) + 8 tokens), then the partial rows are added by 32 warps in order (ceil(n_cta / 32)
                each) and the 32 warp sums in order: |err| <= gamma(depth) sum_t |g_x h rstd| (:func:`gnw_depth`).

For a bf16 output the check (:func:`check_near_tie`) is: correctly rounded, or one ulp away only where the float64
value lies within the bound of the midpoint between the two bf16 neighbours.  Every mismatch must be explained by such
a near tie; no fraction of mismatches is tolerated.  fp32 outputs are checked as |got - ref| <= bound
(:func:`check_bound`).  Both return the largest |err| / bound (for bf16: the distance past the midpoint over the
bound, 0 when everything is correctly rounded).

Inputs: exact mode draws integers in [-4, 4] times a power of two per token and probabilities that are multiples of
1/64, so every product and every K-sum is exact in fp32 and the rounding points above are the only roundings; random
mode draws N(0, 1) times the same per-token powers of two and uniform probabilities.  :func:`norm_rows` gives rows at
magnitudes from 2^-60 to 2^40, all-zero rows and rows where eps dominates mean(h^2).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

U32 = 2.0 ** -24
BF16_U = 2.0 ** -8
G_H_ROUNDINGS = 32
MAG_EXP = (0, -60, 40, -8, 20, -40, 8, -20)  # per-row exponents of norm_rows; rows t % 13 == 5 are all zero
EPS = 1e-6


def gamma(n: int) -> float:
    return n * U32 / (1.0 - n * U32)


# ---- inputs ----------------------------------------------------------------------------------------------------------


def _gen(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def token_scales(T: int, seed: int, device="cpu", exp_range: Tuple[int, int] = (-8, 8)) -> torch.Tensor:
    """fp32 [T]: a power of two per token in [2^lo, 2^hi]."""
    lo, hi = exp_range
    e = torch.randint(lo, hi + 1, (T,), generator=_gen(seed, device), device=device)
    return torch.pow(2.0, e.float())


def values(shape, mode: str, seed: int, device="cpu") -> torch.Tensor:
    g = _gen(seed, device)
    if mode == "exact":
        return torch.randint(-4, 5, shape, generator=g, device=device).float()
    if mode == "random":
        return torch.randn(shape, generator=g, device=device)
    raise ValueError(mode)


def row_map(T: int, K: int, seed: int, neg_frac: float = 0.1, device="cpu") -> Tuple[torch.Tensor, torch.Tensor]:
    """``(row_id_map int32 [T*K], owner int64 [T*K])``: a random permutation of the T*K permuted rows, with about
    ``neg_frac`` of the entries replaced by -1.  ``owner[r]`` is the token whose entry points at row r, -1 for a row
    no entry references."""
    g = _gen(seed, device)
    M = T * K
    rmap = torch.randperm(M, generator=g, device=device)
    if neg_frac > 0:
        rmap[torch.rand(M, generator=g, device=device) < neg_frac] = -1
    owner = torch.full((M,), -1, dtype=torch.int64, device=device)
    ok = rmap >= 0
    owner[rmap[ok]] = torch.arange(M, device=device)[ok] // K
    return rmap.to(torch.int32), owner


def permuted_rows(owner: torch.Tensor, H: int, scales: torch.Tensor, mode: str, seed: int,
                  orphan=float("nan")) -> torch.Tensor:
    """bf16 [M, H]: row r carries the scale of its owner token; rows no entry references hold ``orphan``."""
    v = values((owner.numel(), H), mode, seed, owner.device)
    s = torch.where(owner >= 0, scales[owner.clamp_min(0)], torch.full_like(owner, 0, dtype=torch.float32))
    out = (v * s[:, None]).to(torch.bfloat16)
    out[owner < 0] = orphan
    return out


def token_rows(scales: torch.Tensor, H: int, mode: str, seed: int) -> torch.Tensor:
    """bf16 [T, H], row t times scales[t]."""
    return (values((scales.numel(), H), mode, seed, scales.device) * scales[:, None]).to(torch.bfloat16)


def probs(T: int, K: int, mode: str, seed: int, device="cpu") -> torch.Tensor:
    """fp32 [T, K]: multiples of 1/64 in (0, 1] (exact mode) or uniform in (0, 1)."""
    g = _gen(seed, device)
    if mode == "exact":
        return torch.randint(1, 65, (T, K), generator=g, device=device).float() / 64
    return torch.rand((T, K), generator=g, device=device)


def norm_rows(T: int, H: int, seed: int, device="cpu") -> torch.Tensor:
    """bf16 [T, H]: N(0, 1) rows times 2^MAG_EXP[t % 8] (rows at 2^-20 and below have mean(h^2) far under eps), and
    all-zero rows at t % 13 == 5."""
    e = torch.tensor([MAG_EXP[t % len(MAG_EXP)] for t in range(T)], dtype=torch.float64, device=device)
    s = torch.pow(2.0, e)
    s[torch.arange(T, device=device) % 13 == 5] = 0
    return (torch.randn((T, H), generator=_gen(seed, device), device=device, dtype=torch.float64) * s[:, None]).to(
        torch.bfloat16)


def norm_weight(H: int, seed: int, device="cpu") -> torch.Tensor:
    """fp32 [H] around 1, not representable in bf16."""
    return 1.0 + 0.5 * torch.randn(H, generator=_gen(seed, device), device=device)


# ---- exact restatements ----------------------------------------------------------------------------------------------


def _gather(rows: torch.Tensor, rmap_k: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    ok = rmap_k >= 0
    return rows[rmap_k.long().clamp_min(0)].float(), ok[:, None]


def combine(y: torch.Tensor, rmap: torch.Tensor, p: Optional[torch.Tensor], residual: Optional[torch.Tensor],
            hf: float, K: int) -> torch.Tensor:
    """bf16 [T, H] of xtb_moe_combine (``p``, ``residual`` may be None)."""
    T = rmap.numel() // K
    m = rmap.view(T, K)
    acc = None
    for k in range(K):
        yk, ok = _gather(y, m[:, k])
        prod = yk * p[:, k : k + 1] if p is not None else yk
        prod = torch.where(ok, prod, torch.zeros_like(prod))
        acc = prod if acc is None else acc + prod
    out = acc.to(torch.bfloat16)
    if hf != 1.0:
        out = (out.float() * torch.tensor(hf, dtype=torch.float32, device=out.device)).to(torch.bfloat16)
    if residual is not None:
        out = (out.float() + residual.float()).to(torch.bfloat16)
    return out


def act_grad(g: torch.Tensor, rmap: torch.Tensor, p: Optional[torch.Tensor], K: int, M: int
             ) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(rows bf16 [M, H], written bool [M])`` of xtb_moe_unpermute_bwd's act_grad; unwritten rows are zero."""
    T, H = g.shape
    out = torch.zeros((M, H), dtype=torch.bfloat16, device=g.device)
    written = torch.zeros(M, dtype=torch.bool, device=g.device)
    flat = rmap.long()
    ok = flat >= 0
    tok = torch.arange(T * K, device=g.device) // K
    pk = p.reshape(-1)[ok][:, None] if p is not None else 1.0
    out[flat[ok]] = (g[tok[ok]].float() * pk).to(torch.bfloat16)
    written[flat[ok]] = True
    return out, written


def dispatch_gx(g_xp: torch.Tensor, rmap: torch.Tensor, g_x_gate: Optional[torch.Tensor], K: int) -> torch.Tensor:
    """bf16 [T, H]: bf16(bf16(0 + g_xp[row_0] + g_xp[row_1] + ...) + g_x_gate), -1 rows skipped."""
    T = rmap.numel() // K
    m = rmap.view(T, K)
    acc = torch.zeros((T, g_xp.shape[1]), dtype=torch.float32, device=g_xp.device)
    for k in range(K):
        yk, ok = _gather(g_xp, m[:, k])
        acc = torch.where(ok, acc + yk, acc)
    out = acc.to(torch.bfloat16)
    if g_x_gate is not None:
        out = (out.float() + g_x_gate.float()).to(torch.bfloat16)
    return out


def rmsnorm_x(h: torch.Tensor, rstd: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """bf16 [T, H]: bf16((fp32(h) * rstd) * w), given the kernel's fp32 rstd."""
    return ((h.float() * rstd[:, None]) * w).to(torch.bfloat16)


# ---- float64 references ----------------------------------------------------------------------------------------------


def rstd_rel(H: int) -> float:
    """Relative bound on the kernels' fp32 rstd (module docstring)."""
    return (gamma(H // 32 + 14) / 2 + 4 * U32) * 1.01


def rstd_ref(h: torch.Tensor, eps: float) -> torch.Tensor:
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    return torch.rsqrt(h.double().square().mean(-1) + eps32)


def x_ref(h: torch.Tensor, eps: float, w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(x, bound)`` in float64: h rstd w before the bf16 round, and the bound on the kernel's fp32 value."""
    x = h.double() * rstd_ref(h, eps)[:, None] * w.double()
    return x, (rstd_rel(h.shape[1]) + 3 * U32) * x.abs()


def logits_ref(x: torch.Tensor, gate_w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(logits, bound)`` in float64 from the kernel's own bf16 x."""
    xd, wd = x.double(), gate_w.double()
    return xd @ wd.T, gamma(x.shape[1] // 32 + 6) * (xd.abs() @ wd.abs().T)


def prob_grad_ref(g: torch.Tensor, y: torch.Tensor, rmap: torch.Tensor, K: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(prob_grad, bound)`` in float64 [T, K]; an entry mapped to -1 must be exactly 0."""
    T, H = g.shape
    m = rmap.view(T, K)
    ref = torch.zeros((T, K), dtype=torch.float64, device=g.device)
    S = torch.zeros_like(ref)
    gd = g.double()
    for k in range(K):
        ok = m[:, k] >= 0
        yk = y[m[:, k].long().clamp_min(0)].double()
        yk = torch.where(ok[:, None], yk, torch.zeros_like(yk))
        ref[:, k] = (gd * yk).sum(-1)
        S[:, k] = (gd * yk).abs().sum(-1)
    return ref, gamma(8 * ((H + 255) // 256) + 6) * S


def g_h_ref(g_x: torch.Tensor, h: torch.Tensor, rstd: torch.Tensor, w: torch.Tensor
            ) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(g_h, bound)`` in float64: the RMSNorm backward before the residual, from the restated bf16 g_x."""
    H = h.shape[1]
    wg = g_x.double() * w.double()
    hd = h.double()
    r = rstd.double()[:, None]
    c = (wg * hd).sum(-1, keepdim=True) * r * r / H
    D = (wg * hd).abs().sum(-1, keepdim=True)
    return (wg - hd * c) * r, gamma(G_H_ROUNDINGS) * r * (wg.abs() + hd.abs() * r * r * D / H)


def gnw_depth(T: int, n_cta: int) -> int:
    return -(-T // n_cta) + 9 + -(-n_cta // 32) + 32


def g_norm_w_ref(g_x: torch.Tensor, h: torch.Tensor, rstd: torch.Tensor, n_cta: int = 264
                 ) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(g_norm_w, bound)`` in float64 [H]."""
    terms = g_x.double() * h.double() * rstd.double()[:, None]
    return terms.sum(0), gamma(gnw_depth(h.shape[0], n_cta)) * terms.abs().sum(0)


def combine_ref(y: torch.Tensor, rmap: torch.Tensor, p: Optional[torch.Tensor], residual: Optional[torch.Tensor],
                hf: float, K: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(out, bound)`` in float64: (sum_k p y) hf + residual, and how far three bf16 roundings after an fp32 sum of
    2K roundings may take it: 2^-8 (3.125 |hf| P + 1.0625 |residual|) + gamma(2K) |hf| P, P = sum_k |p y|."""
    T = rmap.numel() // K
    m = rmap.view(T, K)
    acc = torch.zeros((T, y.shape[1]), dtype=torch.float64, device=y.device)
    P = torch.zeros_like(acc)
    for k in range(K):
        ok = (m[:, k] >= 0)[:, None]
        yk = y[m[:, k].long().clamp_min(0)].double()
        t = yk * p[:, k : k + 1].double() if p is not None else yk
        t = torch.where(ok, t, torch.zeros_like(t))
        acc += t
        P += t.abs()
    hf32 = float(torch.tensor(hf, dtype=torch.float32))
    out = acc * hf32
    R = torch.zeros_like(acc)
    if residual is not None:
        out = out + residual.double()
        R = residual.double().abs()
    return out, BF16_U * (3.125 * abs(hf32) * P + 1.0625 * R) + gamma(2 * K) * abs(hf32) * P


# ---- checks ----------------------------------------------------------------------------------------------------------


def _first(mask: torch.Tensor) -> Tuple[int, ...]:
    return tuple(int(i) for i in mask.nonzero()[0])


def assert_bits_equal(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """bf16 tensors equal bit for bit as int16 views; +0 and -0 count as one value."""
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} != {tuple(want.shape)}"
    a = got.contiguous().view(torch.int16)
    b = want.contiguous().view(torch.int16)
    zero = ((a & 0x7FFF) == 0) & ((b & 0x7FFF) == 0)
    bad = (a != b) & ~zero
    if bool(bad.any()):
        i = _first(bad)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at {i}: "
                             f"got {got[i].item()!r}, want {want[i].item()!r}")


def _ratio(err: torch.Tensor, bound: torch.Tensor) -> torch.Tensor:
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return torch.where(torch.isnan(err), math.inf, r)


def check_bound(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = "") -> float:
    """|got - ref| <= bound everywhere (NaN fails); returns the largest |got - ref| / bound."""
    err = (got.double() - ref).abs()
    ratio = _ratio(err, bound)
    r = float(ratio.max()) if ratio.numel() else 0.0
    if r > 1.0:
        i = _first(ratio > 1.0)
        raise AssertionError(f"{what}: {int((ratio > 1).sum())} elements outside the bound; first at {i}: "
                             f"got {got[i].item()!r}, fp64 {ref[i].item()!r}, bound {bound[i].item()!r}")
    return r


def _half_step_toward(g: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """Half the distance from bf16 value g to its bf16 neighbour on the side of ref (float64)."""
    m, e = torch.frexp(g)  # g = m 2^e, 0.5 <= |m| < 1
    step = torch.pow(2.0, (e - 8).double())
    step = torch.where((m.abs() == 0.5) & (ref.abs() < g.abs()), step / 2, step)
    return torch.where(g == 0, torch.full_like(g, 2.0 ** -133), step.clamp_min(2.0 ** -133)) / 2


def check_near_tie(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = "") -> Tuple[float, int]:
    """A bf16 output is correctly rounded from the float64 ``ref``, or off by one ulp where ``ref`` lies within
    ``bound`` of the midpoint between the two candidates.  Returns ``(largest distance past the midpoint / bound,
    number of elements that are not correctly rounded)``."""
    g = got.double()
    d = (g - ref).abs()
    half = _half_step_toward(g, ref)
    past = (d - half).clamp_min(0)
    ratio = _ratio(past, bound)
    ratio = torch.where(torch.isfinite(g), ratio, math.inf)
    r = float(ratio.max()) if ratio.numel() else 0.0
    if r > 1.0:
        i = _first(ratio > 1.0)
        raise AssertionError(f"{what}: {int((ratio > 1).sum())} of {ratio.numel()} elements are neither correctly "
                             f"rounded nor a near tie; first at {i}: got {got[i].item()!r}, fp64 {ref[i].item()!r}, "
                             f"bound {bound[i].item()!r}")
    return r, int((past > 0).sum())
