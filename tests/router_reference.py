"""float64 references, exact restatements, bounds and input generators for the gate and router kernels
(``csrc/route.cu``, ``csrc/gate_mma.cu``).  Test infrastructure only; nothing under ``xtuner_b200/`` imports it.  Plain
torch on whatever device the operands are on.

Gate logits, logits = x w^T + b with bf16 x and fp32 w.  The reference is float64 with S = |x| |w|^T.  u = 2^-24 and
gamma(n) = n u / (1 - n u) bound n successive fp32 roundings of a sum whose partial sums are at most S.

  ``small``    gate_logits_small_kernel: each lane chains H/32 fmaf (8 per 256-column chunk), a 5-level warp tree adds
               the 32 lane sums, the bias adds once: gamma(H/32 + 6) (S + |b|).
  ``strided``  sgemm_strided_kernel: one chain of H fmaf per output, then the bias: gamma(H + 1) (S + |b|).
  ``mma``      the tensor-core gate of xtb_gate_route_dispatch: w = hi + mid + lo exactly (three bf16 planes, 24
               bits), every bf16 product is exact in fp32, and each K quarter runs 6 H/128 m16n8k16 steps into one fp32
               accumulator; the four quarters are added in order, then the bias.  The tensor core's internal
               accumulation is not assumed to round to nearest: each step is allowed 2u (truncation) relative to the
               partial sums, so 2 gamma(6 H/128) + gamma(4) on S, + |b| gamma(1).

Input modes for the gate (:func:`gate_inputs`):

  ``exact``    x = integers in [-4, 4] times 2^s, w = integers in [-8, 8] times 2^-m: every partial sum is an integer
               multiple of 2^(s - m) below 2^24 of them, so every kernel equals float64 bit for bit (with an exact bias).
  ``onehot``   row t of x is a single +-2^j at column h(t) = t mod H (every column is visited), w is random fp32 with a
               full 24-bit mantissa over exponents -100 .. 100, with columns whose hi or mid bf16 rounding is a tie.
               The logits must be exactly 2^j w[:, h(t)]: this pins the hi/mid/lo split, the column permutation of the
               K ordering and which warp owns which K quarter.
  ``random``   N(0, 1) x and w.

Greedy router (softmax or sigmoid, then K rounds of arg-max).  expf is within 2 ulp.  Softmax: p = exp(x - m) / sum;
x - m rounds once (relative u |x - m| in the exponent's argument), expf adds 4u, the fp32 sum of E terms gamma(E), the
division u: |p - p64| <= (u |x - m| + 6u + gamma(E)) p + 2^-149.  Sigmoid: 1 / (1 + expf(-x)) is within 6u relative.
The exact checks (:func:`check_greedy_exact`) do not depend on expf: the ids are K rounds of (value desc, index asc)
over the kernel's own router_weights, topk_weights is an fp32 sum of the selected weights in k order, then / sum when
normalising, then * scaling only when scaling != 1, and tokens_per_expert is the bincount of the ids.

No-aux router: :func:`noaux_ref` restates it in float64 with the kernels' tie rules (groups and experts tied on the
value are taken lowest index first).

Backward references are float64 autograd through ``oracle.greedy_router`` / ``oracle.noaux_router`` on float64 logits
(:func:`greedy_bwd_ref`).  The bound on an fp32 grad_logits entry is gamma(4K + 16) times the sum of the magnitudes of
the terms that make it (:func:`greedy_bwd_bound`), plus 8u of p's own error times |g|.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

U32 = 2.0 ** -24


def gamma(n: float) -> float:
    return n * U32 / (1.0 - n * U32)


def _gen(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


# ---- gate inputs -----------------------------------------------------------------------------------------------------


def _ties(w: torch.Tensor, g: torch.Generator) -> torch.Tensor:
    """Replace some entries by values whose bf16 rounding (of w, or of w - hi) is a tie: 9 significant bits ending in 1,
    or 17 ending in 1."""
    n = w.numel()
    flat = w.reshape(-1).clone()
    sel = torch.randperm(n, generator=g, device=w.device)[: max(1, n // 8)]
    m9 = (torch.randint(0, 256, (sel.numel(),), generator=g, device=w.device) * 2 + 257).double()  # 9 bits, odd
    m17 = (torch.randint(0, 65536, (sel.numel(),), generator=g, device=w.device) * 2 + 65537).double()  # 17 bits, odd
    e = torch.randint(-40, 40, (sel.numel(),), generator=g, device=w.device).double()
    v = torch.where(torch.arange(sel.numel(), device=w.device) % 2 == 0, m9 * 2.0 ** (e - 8), m17 * 2.0 ** (e - 16))
    sign = torch.where(torch.rand(sel.numel(), generator=g, device=w.device) < 0.5, -1.0, 1.0)
    flat[sel] = (v * sign).float()
    return flat.view_as(w)


def gate_inputs(T: int, H: int, E: int, mode: str, seed: int, device="cpu", with_bias: bool = True
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """``(x bf16 [T, H], w fp32 [E, H], bias fp32 [E] or None)`` for ``mode`` in exact / onehot / random."""
    g = _gen(seed, device)
    if mode == "exact":
        s = 2.0 ** torch.randint(-4, 5, (T, 1), generator=g, device=device).float()
        x = (torch.randint(-4, 5, (T, H), generator=g, device=device).float() * s).to(torch.bfloat16)
        w = torch.randint(-8, 9, (E, H), generator=g, device=device).float() * 2.0 ** -6
        b = torch.randint(-8, 9, (E,), generator=g, device=device).float() * 2.0 ** -3
    elif mode == "onehot":
        j = torch.randint(-20, 21, (T,), generator=g, device=device).float()
        sign = torch.where(torch.rand(T, generator=g, device=device) < 0.5, -1.0, 1.0)
        x = torch.zeros(T, H, device=device)
        x[torch.arange(T, device=device), torch.arange(T, device=device) % H] = sign * 2.0 ** j
        x = x.to(torch.bfloat16)
        mant = 1.0 + torch.rand(E, H, generator=g, device=device, dtype=torch.float64)
        ex = torch.randint(-100, 101, (E, H), generator=g, device=device).double()
        sg = torch.where(torch.rand(E, H, generator=g, device=device) < 0.5, -1.0, 1.0).double()
        w = _ties((mant * 2.0 ** ex * sg).float(), g)
        b = None
    elif mode == "random":
        x = torch.randn(T, H, generator=g, device=device).to(torch.bfloat16)
        w = torch.randn(E, H, generator=g, device=device)
        b = torch.randn(E, generator=g, device=device)
    else:
        raise ValueError(mode)
    return x, w, (b if with_bias else None)


def gate_ref(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(logits, S)`` in float64; S = |x| |w|^T + |b|."""
    xd, wd = x.double(), w.double()
    ref = xd @ wd.T
    S = xd.abs() @ wd.abs().T
    if bias is not None:
        ref = ref + bias.double()
        S = S + bias.double().abs()
    return ref, S


def gate_bound(kernel: str, H: int, S: torch.Tensor) -> torch.Tensor:
    """Bound on |logits - float64| for the kernel's accumulation (module docstring)."""
    if kernel == "small":
        return gamma(H // 32 + 6) * S
    if kernel == "strided":
        return gamma(H + 1) * S
    if kernel == "mma":
        return (2 * gamma(6 * H // 128) + gamma(5)) * S
    raise ValueError(kernel)


def gate_kernel(T: int, H: int, E: int) -> str:
    """Which kernel xtb_gate_logits runs (the fused entry always runs ``mma``)."""
    return "small" if (E <= 16 and H % 256 == 0 and E * H * 4 <= 200 * 1024) else "strided"


# ---- gate emulations (the CPU test plants mistakes in these) ---------------------------------------------------------


def split3(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The three bf16 planes of the fused gate, as fp32: hi = bf16(w), mid = bf16(w - hi), lo = bf16(w - hi - mid)."""
    hi = w.to(torch.bfloat16).float()
    mid = (w - hi).to(torch.bfloat16).float()
    lo = (w - hi - mid).to(torch.bfloat16).float()
    return hi, mid, lo


def emulate_gate_mma(x: torch.Tensor, w: torch.Tensor, planes: int = 3, order=None) -> torch.Tensor:
    """fp32 emulation of the plane-split gate: per plane x @ plane^T in fp32 (whatever summation order torch uses),
    added smallest plane first.  ``planes`` < 3 drops the smallest planes."""
    xf = x.float()
    hi, mid, lo = split3(w)
    parts = [hi, mid, lo][:planes]
    acc = torch.zeros(x.shape[0], w.shape[0], dtype=torch.float32, device=x.device)
    for p in reversed(parts):
        acc = acc + xf @ p.T
    return acc


# ---- greedy router ---------------------------------------------------------------------------------------------------


def greedy_ref(logits: torch.Tensor, scoring: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(router_weights, bound)`` in float64 from fp32 logits."""
    ld = logits.double()
    E = logits.shape[1]
    if scoring == "softmax":
        m = ld.max(-1, keepdim=True).values
        p = torch.softmax(ld, -1)
        rel = U32 * (ld - m).abs() + 6 * U32 + gamma(E)
    else:
        p = torch.sigmoid(ld)
        rel = torch.full_like(p, 6 * U32)
    return p, rel * p + 2.0 ** -149


def topk_rounds(v: torch.Tensor, K: int) -> torch.Tensor:
    """int64 [T, K]: K rounds of arg-max over each row by (value desc, index asc); rows must be NaN-free."""
    idx = torch.arange(v.shape[1], device=v.device).expand_as(v)
    # sort by index asc, then stable by value desc
    order = torch.sort(v, dim=-1, descending=True, stable=True)[1]
    return idx.gather(1, order)[:, :K]


def topk_weights_restated(rw: torch.Tensor, ids: torch.Tensor, norm: bool, scaling: float) -> torch.Tensor:
    """fp32 restatement of the kernels' topk_weights from their own router_weights."""
    sel = rw.gather(1, ids)
    s = torch.zeros_like(sel[:, 0])
    for k in range(ids.shape[1]):
        s = s + sel[:, k]
    out = sel / s[:, None] if norm else sel.clone()
    if scaling != 1.0:
        out = out * torch.tensor(scaling, dtype=torch.float32, device=out.device)
    return out


def check_greedy_exact(rw, tw, ids, tpe, K: int, norm: bool, scaling: float, what: str = "") -> None:
    """ids, topk_weights and tokens_per_expert against the kernel's own router_weights, bit for bit (NaN-free rows)."""
    want_ids = topk_rounds(rw, K)
    bad = (ids != want_ids).any(-1)
    if bool(bad.any()):
        t = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} rows with other ids; row {t}: got {ids[t].tolist()}, "
                             f"want {want_ids[t].tolist()}")
    want_tw = topk_weights_restated(rw, ids, norm, scaling)
    d = (tw.view(torch.int32) != want_tw.view(torch.int32)) & ~((tw == 0) & (want_tw == 0))
    if bool(d.any()):
        t, k = (int(i) for i in d.nonzero()[0])
        raise AssertionError(f"{what}: topk_weights differ in {int(d.sum())} places; first [{t}, {k}]: "
                             f"{tw[t, k].item()!r} != {want_tw[t, k].item()!r}")
    E = rw.shape[1]
    want_tpe = torch.bincount(ids.reshape(-1), minlength=E)
    assert torch.equal(tpe.to(torch.int64), want_tpe), f"{what}: tokens_per_expert != bincount(ids)"


def decided_rows(p64: torch.Tensor, bound: torch.Tensor, K: int) -> torch.Tensor:
    """bool [T]: rows whose K-th and (K+1)-th float64 values (and every pair among the top K + 1 values) are more
    than twice the bound apart, or exactly equal in the inputs, so the fp32 kernel must choose the float64 ids."""
    E = p64.shape[1]
    if K >= E:
        return torch.ones(p64.shape[0], dtype=torch.bool, device=p64.device)
    v, i = torch.sort(p64, dim=-1, descending=True, stable=True)
    b = bound.gather(1, i)
    gap = v[:, : K] - v[:, 1 : K + 1]
    ok = (gap > 2 * (b[:, : K] + b[:, 1 : K + 1])) | (gap == 0)
    return ok.all(-1)


# ---- no-aux router ---------------------------------------------------------------------------------------------------


def noaux_ref(logits: torch.Tensor, bias: torch.Tensor, K: int, n_group: int, topk_group: int
              ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``(ids, kept, choice)`` in float64: group score = top-2 sum, groups and experts by (value desc, index asc)."""
    from oracle import moe_oracle as O

    s = torch.sigmoid(logits.double())
    ch = s + bias.double()
    kept = O.noaux_kept_experts(ch, n_group, topk_group)
    masked = torch.where(kept, ch, torch.zeros_like(ch))
    ids = topk_rounds(masked, K)
    return ids, kept, masked


# ---- backward --------------------------------------------------------------------------------------------------------


def greedy_bwd_ref(logits, K, scoring, norm, scaling, g_tw, g_rw, g_direct):
    """float64 grad_logits by autograd through oracle.greedy_router (its own ids are replaced by ``ids`` via the
    caller's choice of decided rows), plus the magnitude sum the bound scales with."""
    from oracle import moe_oracle as O

    ld = logits.double().clone().requires_grad_(True)
    r = O.greedy_router(ld, K, norm, scaling, scoring)
    outs, grads = [], []
    if g_tw is not None:
        outs.append(r["topk_weights"])
        grads.append(g_tw.double())
    if g_rw is not None:
        outs.append(r["router_weights"])
        grads.append(g_rw.double())
    gl = torch.zeros_like(ld)
    if outs:
        (gl,) = torch.autograd.grad(outs, ld, grads)
    if g_direct is not None:
        gl = gl + g_direct.double()
    return gl.detach(), r["topk_ids"]


def greedy_bwd_bound(p64, K, g_tw, g_rw, g_direct, scaling, norm) -> torch.Tensor:
    """|err| <= gamma(4K + 16) (|p| (|gp| + D) + |g_direct|) with gp the gradient reaching router_weights, D = sum |gp p|."""
    T, E = p64.shape
    gp = torch.zeros_like(p64)
    if g_rw is not None:
        gp = gp + g_rw.double().abs()
    if g_tw is not None:
        topv = torch.sort(p64, -1, descending=True).values[:, :K]
        s = topv.sum(-1, keepdim=True)
        gt = g_tw.double().abs()
        c = abs(scaling) * (gt + (gt * topv / s).sum(-1, keepdim=True)) / (s if norm else 1.0)
        gp = gp + c.max(-1, keepdim=True).values
    D = (gp * p64).sum(-1, keepdim=True)
    mag = p64 * (gp + D) + (g_direct.double().abs() if g_direct is not None else 0.0)
    return gamma(4 * K + 16) * mag + 8 * U32 * p64 * (gp + D) + 2.0 ** -140


def check_bound(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = "") -> float:
    """|got - ref| <= bound everywhere (NaN fails); returns the largest |got - ref| / bound."""
    err = (got.double() - ref).abs()
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    ratio = torch.where(torch.isnan(err), math.inf, ratio)
    r = float(ratio.max()) if ratio.numel() else 0.0
    if r > 1.0:
        i = tuple(int(v) for v in (ratio > 1).nonzero()[0])
        raise AssertionError(f"{what}: {int((ratio > 1).sum())} elements outside the bound; first at {i}: "
                             f"got {got[i].item()!r}, fp64 {ref[i].item()!r}, bound {bound[i].item()!r}")
    return r
