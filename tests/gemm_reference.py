"""float64 references, input generators and a scale-aware checker for the grouped expert GEMMs of
``xtuner_b200/csrc/group_gemm.cu`` (test infrastructure only; nothing under ``xtuner_b200/`` imports it).

References, one expert at a time (``counts`` = rows per expert, the host copy of ``tokens_per_expert``):

  ``nt``  out[rows_e] = x[rows_e] . w[e]^T           (xtb_group_gemm_nt, and ``h`` of xtb_group_gemm_nt_swiglu)
  ``nn``  out[rows_e] = dy[rows_e] . w[e]            (xtb_group_gemm_nn)
  ``tn``  dw[e]       = dy[rows_e]^T . x[rows_e]     (xtb_group_gemm_tn / _tn_pair; an expert without rows: zeros)
  :func:`swiglu_act`  a = bf16(bf16(silu(h_gate)) * h_up) of a bf16 ``h``

They run in float64 with plain torch on whatever device the operands are on (on a GPU that is cuBLAS DGEMM, which shares
no code with this library), and convert one expert at a time, so a 128-expert weight is never held in float64 at once.
Each expert's reference comes with ``S = |A|.|B|^T``, the sum of ``|a_k| |b_k|`` behind every output element.

Inputs (:func:`rows_operand`, :func:`weight_operand`):

* exact mode: integers in [-4, 4] times a power of two in [2^-8, 2^8] that depends on the expert (consecutive experts
  never share one), so data used for the wrong expert shows.  Every product is exact in fp32, and a partial sum over
  at most 16384 terms is an integer below 16 * 16384 = 2^18 in units of its expert's scale product, far inside fp32's
  24 bits: an fp32 accumulator gives the exact sum in any order, and the only rounding left is the final fp32 -> bf16
  round-to-nearest-even.  The kernel's output must then equal ``bf16_rn(reference)`` bit for bit (:func:`assert_exact`).
* random mode: N(0, 1) times the same per-expert powers of two.

The bound (:func:`check_bound`), per element:  ``|out - ref| <= 2^-8 |ref| + tau * S``.

``2^-8 |ref|`` is the final round-to-nearest to bf16 (unit roundoff 2^-8).  ``tau * S`` covers the fp32 accumulation:
the kernel multiplies bf16 operands exactly and adds them into an fp32 accumulator in k order, one 16-deep wgmma step at
a time, so an element of a K-long reduction takes at most K/16 fp32 roundings.  Each is below 2^-23 of the running
partial sum (2^-23 also covers an adder that truncates instead of rounding), and a partial sum is at most S, so the
worst case is ``K/16 * 2^-23 * S = K * 2^-27 * S``: ``tau = 2^-16`` covers it outright for K <= 2048, which is every NT
and NN reduction used here.  TN reduces over the rows of one expert, up to 16384 here, where the worst case is 8x tau;
but the partial sums of zero-mean data grow like sqrt(k) while S grows like k, which puts the expected error more than
an order of magnitude under tau at that length.

tau is small next to every error the suite must catch (``tests/test_gemm_reference_cpu.py`` shows each rejected): a
dropped 64-deep k-block moves an element by a 64-term sum, about 8 rms(a b), while ``tau * S`` stays below
16384 * 2^-16 mean|a b| = mean|a b| / 4 at the longest reduction; truncating to bf16 instead of rounding errs by up to
one ulp (2^-7 relative), and the bound allows half of one.
"""
from __future__ import annotations

import math
import random
from typing import Iterator, List, Sequence, Tuple

import torch

ROW_COUNTS = (0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 129, 255, 256, 257)  # 16-row store box, 64-row TN k-block, 128-row tile
BLOCK_M = 128
TAU = 2.0 ** -16
BF16_U = 2.0 ** -8
SCALE_EXP = (-8, 8)


# ---- count patterns ------------------------------------------------------------------------------------------------


def offsets(counts: Sequence[int]) -> List[int]:
    o = [0]
    for c in counts:
        o.append(o[-1] + int(c))
    return o


def m_tiles(counts: Sequence[int]) -> int:
    """128-row tiles of the NT / NN tile list (times the output-column tiles, the number of persistent-kernel tiles)."""
    return sum((int(c) + BLOCK_M - 1) // BLOCK_M for c in counts)


def counts_pattern(E: int, kind: str, seed: int = 0, total: int = 0) -> List[int]:
    """Rows per expert.
    ``ragged``:  drawn from ROW_COUNTS without 0; first and last expert empty and (E >= 8) two consecutive empty experts in
                 the middle
    ``single``:  one expert (the middle one) owns all ``total`` rows
    ``zipf``:    ``total`` rows over a Zipf(1.2) law on a shuffled rank order; first, last and every 16th expert empty
    ``sparse``:  mostly empty (E = 1024): every 37th expert draws from ROW_COUNTS, first and last empty
    ``balanced``: ``total`` rows evenly, the remainder to expert 0"""
    rng = random.Random(seed * 7919 + E)
    if kind == "ragged":
        c = [rng.choice(ROW_COUNTS[1:]) for _ in range(E)]
        if E >= 8:
            c[E // 2 : E // 2 + 2] = [0, 0]
        c[0] = c[-1] = 0 if E > 1 else max(c[0], 1)
    elif kind == "single":
        c = [0] * E
        c[E // 2] = total
    elif kind == "zipf":
        ranks = list(range(1, E + 1))
        rng.shuffle(ranks)
        wgt = [0.0 if (e == 0 or e == E - 1 or e % 16 == 8) else ranks[e] ** -1.2 for e in range(E)]
        s = sum(wgt)
        c = [int(math.floor(w / s * total)) for w in wgt]
        c[max(range(E), key=lambda e: wgt[e])] += total - sum(c)
    elif kind == "sparse":
        c = [rng.choice(ROW_COUNTS[1:]) if e % 37 == 5 else 0 for e in range(E)]
        c[0] = c[-1] = 0
    elif kind == "balanced":
        c = [total // E] * E
        c[0] += total - sum(c)
    else:
        raise ValueError(kind)
    assert len(c) == E and min(c) >= 0
    return c


# ---- inputs ----------------------------------------------------------------------------------------------------------


def expert_scales(E: int, seed: int, exp_range: Tuple[int, int] = SCALE_EXP) -> List[float]:
    """A power of two per expert in [2^lo, 2^hi]; consecutive experts get different ones."""
    lo, hi = exp_range
    n = hi - lo + 1
    step = 7 if n % 7 else 5
    return [2.0 ** (lo + (e * step + seed) % n) for e in range(E)] if n > 1 else [2.0 ** lo] * E


def _values(shape, mode: str, g: torch.Generator, device) -> torch.Tensor:
    if mode == "exact":
        return torch.randint(-4, 5, shape, generator=g, device=device, dtype=torch.float32)
    if mode == "random":
        return torch.randn(shape, generator=g, device=device)
    raise ValueError(mode)


def _gen(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def rows_operand(counts: Sequence[int], cols: int, mode: str, seed: int, device="cpu",
                 exp_range: Tuple[int, int] = SCALE_EXP) -> torch.Tensor:
    """bf16 [sum(counts), cols]: the rows of expert e carry expert e's scale."""
    sc = expert_scales(len(counts), seed, exp_range)
    per_row = torch.repeat_interleave(torch.tensor(sc, dtype=torch.float32), torch.tensor(list(counts), dtype=torch.int64))
    v = _values((sum(counts), cols), mode, _gen(seed, device), device)
    return (v * per_row.to(device)[:, None]).to(torch.bfloat16)


def weight_operand(E: int, rows: int, cols: int, mode: str, seed: int, device="cpu",
                   exp_range: Tuple[int, int] = SCALE_EXP) -> torch.Tensor:
    """bf16 [E, rows, cols], expert e scaled by its own power of two (generated one expert at a time)."""
    sc = expert_scales(E, seed + 1, exp_range)
    g = _gen(seed, device)
    w = torch.empty((E, rows, cols), dtype=torch.bfloat16, device=device)
    for e in range(E):
        w[e] = (_values((rows, cols), mode, g, device) * sc[e]).to(torch.bfloat16)
    return w


# ---- references ------------------------------------------------------------------------------------------------------


def products(kind: str, a: torch.Tensor, b: torch.Tensor, counts: Sequence[int], bound: bool = True
             ) -> Iterator[Tuple[int, object, torch.Tensor, torch.Tensor]]:
    """Per expert: ``(e, sel, ref, S)`` in float64, where ``out[sel]`` is expert e's block of the output.
    nt: a = x [M, Kd], b = w [E, N, Kd];  nn: a = dy [M, N], b = w [E, N, Kd];  tn: a = dy [M, N], b = x [M, Kd].
    NT / NN skip experts without rows (they own no output); TN yields zeros for them (S = 0 demands exact zeros)."""
    o = offsets(counts)
    for e in range(len(counts)):
        s, t = o[e], o[e + 1]
        if kind == "tn":
            A = a[s:t].double().T
            B = b[s:t].double()
            ref = A @ B
            yield e, e, ref, ((A.abs() @ B.abs()) if bound else None)
            continue
        if s == t:
            continue
        A = a[s:t].double()
        B = b[e].double()
        if kind == "nt":
            B = B.T
        elif kind != "nn":
            raise ValueError(kind)
        yield e, slice(s, t), A @ B, ((A.abs() @ B.abs()) if bound else None)


def reference(kind: str, a: torch.Tensor, b: torch.Tensor, counts: Sequence[int]) -> torch.Tensor:
    """The whole float64 reference (small shapes only: it holds the output in float64)."""
    E = len(counts)
    if kind == "nt":
        out = torch.zeros((a.shape[0], b.shape[1]), dtype=torch.float64, device=a.device)
    elif kind == "nn":
        out = torch.zeros((a.shape[0], b.shape[2]), dtype=torch.float64, device=a.device)
    else:
        out = torch.zeros((E, a.shape[1], b.shape[1]), dtype=torch.float64, device=a.device)
    for _, sel, ref, _ in products(kind, a, b, counts, bound=False):
        out[sel] = ref
    return out


def bf16_rn(t: torch.Tensor) -> torch.Tensor:
    """float64 -> bf16, round to nearest even.  Goes through fp32, which is exact for exact-mode sums (below 2^24 units)."""
    return t.float().to(torch.bfloat16)


def swiglu_act(h: torch.Tensor) -> torch.Tensor:
    """a = bf16(bf16(silu(h_gate)) * h_up) for a bf16 h [M, 2I] (silu in float64; the product of two bf16 is exact)."""
    I = h.shape[1] // 2
    g, u = h[:, :I].double(), h[:, I:].double()
    s = bf16_rn(g * torch.sigmoid(g)).double()
    return bf16_rn(s * u)


def ulp_distance(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Distance in bf16 steps between two bf16 tensors (+0 and -0 are one value)."""

    def ordered(t):
        i = t.contiguous().view(torch.int16).to(torch.int32)
        mag = i & 0x7FFF
        return torch.where(i < 0, -mag, mag)

    return (ordered(a) - ordered(b)).abs()


# ---- checks ----------------------------------------------------------------------------------------------------------


def _where(e, sel, idx) -> str:
    if isinstance(sel, slice):
        return f"expert {e}, row {sel.start + int(idx[0])} (local row {int(idx[0])}), column {int(idx[1])}"
    return f"expert {e}, dW element {tuple(int(i) for i in idx)}"


def assert_exact(out: torch.Tensor, kind: str, a: torch.Tensor, b: torch.Tensor, counts: Sequence[int], what: str = "") -> None:
    """Every element of ``out`` equals ``bf16_rn(reference)`` (+0 and -0 count as equal)."""
    for e, sel, ref, _ in products(kind, a, b, counts, bound=False):
        want = bf16_rn(ref)
        got = out[sel]
        bad = got != want
        if bool(bad.any()):
            idx = bad.nonzero()[0]
            raise AssertionError(
                f"{what} {kind}: {int(bad.sum())} elements differ from bf16(fp64 reference); first at {_where(e, sel, idx)}: "
                f"got {got[tuple(idx)].item()!r}, want {want[tuple(idx)].item()!r} (fp64 {ref[tuple(idx)].item()!r})")


def check_bound(out: torch.Tensor, kind: str, a: torch.Tensor, b: torch.Tensor, counts: Sequence[int], tau: float = TAU,
                what: str = "") -> float:
    """Asserts ``|out - ref| <= 2^-8 |ref| + tau S`` everywhere; returns the largest ``|out - ref| / bound``."""
    worst = 0.0
    for e, sel, ref, S in products(kind, a, b, counts):
        got = out[sel].double()
        err = (got - ref).abs()
        bnd = BF16_U * ref.abs() + tau * S
        ratio = torch.where(bnd > 0, err / bnd.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        ratio = torch.where(torch.isnan(got), math.inf, ratio)
        r = float(ratio.max()) if ratio.numel() else 0.0
        if r > 1.0:
            idx = (ratio > 1.0).nonzero()[0]
            i = tuple(idx)
            raise AssertionError(
                f"{what} {kind}: {int((ratio > 1).sum())} elements outside the bound; first at {_where(e, sel, idx)}: "
                f"got {got[i].item()!r}, fp64 {ref[i].item()!r}, bound {bnd[i].item()!r} (S = {S[i].item()!r})")
        worst = max(worst, r)
    return worst
