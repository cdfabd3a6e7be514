"""Independent references, checkers and input generators for the peer-exchange kernels (``csrc/comm.cu``) and the
expert-parallel pulls (``csrc/ep.cu``), run on ONE device.  Test infrastructure only; nothing under ``xtuner_b200/``
imports it.  Plain torch on whatever device the operands are on.

Simulated world.  Every exchange kernel takes a device array of per-rank base pointers and dereferences it with ordinary
global loads and stores, so W allocations on one device stand in for W ranks.  :class:`SimWorld` places the W buffers
inside one arena filled with :data:`FILL32` (a bit pattern that is an fp32 NaN and, in each half, a bf16 NaN no kernel
produces), with guard bytes before, between and after them, and builds the int64 device pointer table.

References (restated from the operations' definitions, not from the kernels' offset tables):

  :func:`a2a`              Ulysses all-to-all: rank r receives cat([in_s.tensor_split(W, scatter_dim)[r] for s], gather_dim).
  :func:`allgather`        out[r n : (r + 1) n] = bf16_rne(shard_r) on every rank (bf16 shards are copied as they are).
  :func:`reduce_scatter`   exact restatement: fp32 acc = +0, acc = acc + float(in_r[me n + i]) for r = 0 .. W-1 (separate
                           adds, no fma), then acc * scale in fp32, then bf16_rne for a bf16 output.
  :func:`allreduce`        the same over fp32 inputs without the rank offset.
  :func:`ep_to_experts`    for owner d: the rows every source s sends to d, concatenated in rank order (the variable-split
                           all-to-all by owner rank), then stably re-sorted by local expert.  Returned as (source, row) pairs.
  :func:`ep_to_sources`    its exact inverse: for each row p of rank s, the (owner, position) that holds (s, p).

float64 bounds (u = 2^-24; gamma(n) = n u / (1 - n u) bounds n successive fp32 roundings of a sum whose partial sums are
at most S = sum_r |x_r|).  The first add is 0 + x_0 and is exact, so the rank sum rounds W - 1 times:
|fl(sum) - sum| <= gamma(W - 1) S.  Multiplying by the fp32 scale s carries that error times |s| and rounds once more,
at most u |fl(sum) s| <= u (|ref64| + |s| gamma(W - 1) S).  Hence, for an fp32 output,

    |out - ref64| <= (1 + u) gamma(W - 1) |s| S + u |ref64|                                     (:func:`rs_bound`)

and a bf16 output rounds the fp32 value y once more.  bf16 keeps 8 significant bits, so half an ulp is up to 2^-8 |y|
(at |y| just above a power of two; 2^-9 would only hold just below one): |bf16(y) - y| <= 2^-8 (|ref64| + bound_f32),
which is added.  (Inputs are bf16 or fp32 values, exact in float64; no result here is subnormal.)

Inputs: exact mode draws integers in [-4, 4] times a power of two 2^k per rank with k in [0, 16], so every partial sum
of up to 16 ranks is an integer below 2^23 and exact in fp32; random mode draws N(0, 1) times a per-rank scale from 2^-40
to 2^40, so the rank order changes the fp32 bits; cancel mode puts 2^20 x and -2^20 x on the first and last rank, so the
order changes the result by more than a bf16 ulp.  :func:`labels` fills a buffer with 32-bit words that name their source
rank and position; :func:`ep_rows` gives row r of rank s the words (s, r, ...), so a misplaced row is identified by name.
:func:`f32_specials` lists the fp32 classes the bf16 cast must round right.

NaN: the CUDA cast ``__float2bfloat16_rn`` returns 0x7FFF for every NaN, torch returns 0x7FC0 (with the sign); the bits of
a NaN are therefore compared by position only (:func:`assert_bits_equal`).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np
import torch

U32 = 2.0 ** -24
BF16_U = 2.0 ** -8  # unit roundoff of bf16 (8 significant bits): half an ulp relative to the value
FILL32 = 0x7FA57FA5  # fp32 NaN; each 16-bit half is the bf16 NaN 0x7FA5
GUARD_BYTES = 256


def gamma(n: int) -> float:
    return n * U32 / (1.0 - n * U32)


def ep_hdr_bytes(E: int) -> int:
    """Header size the expert-parallel dispatcher gives a staging buffer: int32 cnt[E], padded to 256 bytes."""
    return (E * 4 + 255) // 256 * 256


# ---- simulated world -------------------------------------------------------------------------------------------------


class SimWorld:
    """W buffers of ``nbytes`` each (16-byte aligned) inside one FILL32 arena, ``guard`` bytes before, between and after
    them.  ``table`` is the int64 device array of their addresses, what the exchange kernels take as peer pointers."""

    def __init__(self, W: int, nbytes: int, device="cuda", guard: int = GUARD_BYTES):
        assert guard % 16 == 0
        self.W, self.nbytes, self.guard = W, nbytes, guard
        self.slot = (nbytes + 15) // 16 * 16 + guard
        total = guard + W * self.slot
        self.arena = torch.full((total // 4,), FILL32, dtype=torch.int32, device=device)
        self.offsets = [guard + r * self.slot for r in range(W)]
        base = self.arena.data_ptr()
        self.table = torch.tensor([base + o for o in self.offsets], dtype=torch.int64, device=device)

    def bytes(self, r: int) -> torch.Tensor:
        o = self.offsets[r]
        return self.arena.view(torch.uint8)[o : o + self.nbytes]

    def buf(self, r: int, dtype=torch.uint8, shape=None) -> torch.Tensor:
        t = self.bytes(r).view(dtype)
        return t if shape is None else t.view(shape)

    def ptr(self, r: int, byte_offset: int = 0) -> int:
        return self.arena.data_ptr() + self.offsets[r] + byte_offset

    def guards_intact(self) -> bool:
        keep = torch.ones(self.arena.numel(), dtype=torch.bool, device=self.arena.device)
        for o in self.offsets:
            keep[o // 4 : (o + (self.nbytes + 3) // 4 * 4) // 4] = False
        return bool((self.arena[keep] == FILL32).all())


def guarded(nbytes: int, device="cuda", guard: int = GUARD_BYTES) -> SimWorld:
    """One NaN-guarded output buffer (a world of one)."""
    return SimWorld(1, nbytes, device, guard)


# ---- bit comparison --------------------------------------------------------------------------------------------------


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def assert_bits_equal(got: torch.Tensor, want: torch.Tensor, what: str) -> None:
    """Bit for bit; a NaN only has to sit where a NaN is expected (payloads differ between CUDA and torch)."""
    assert got.shape == want.shape and got.dtype == want.dtype, f"{what}: {got.shape}/{got.dtype} vs {want.shape}/{want.dtype}"
    gb, wb = _bits(got), _bits(want)
    same = gb == wb
    if got.is_floating_point():
        same |= torch.isnan(got) & torch.isnan(want)
    if not bool(same.all()):
        bad = (~same).nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int((~same).sum())} elements differ; first at {bad}: got bits "
                             f"{int(gb[tuple(bad)]):#x}, want {int(wb[tuple(bad)]):#x}")


def assert_within(got: torch.Tensor, ref64: torch.Tensor, bound: torch.Tensor, what: str) -> float:
    """|got - ref64| <= bound everywhere; returns the largest |err| / bound (0 / 0 counts as 0)."""
    err = (got.double() - ref64).abs()
    if not bool((err <= bound).all()):
        i = int((err - bound).argmax())
        raise AssertionError(f"{what}: |err| {float(err.view(-1)[i]):.3e} > bound {float(bound.view(-1)[i]):.3e} at {i}")
    ratio = torch.where(bound > 0, err / bound, torch.zeros_like(err))
    return float(ratio.max()) if ratio.numel() else 0.0


# ---- casts -----------------------------------------------------------------------------------------------------------


def bf16_rne(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16, round to nearest even, from the bits (NaN -> 0x7FFF, as the CUDA intrinsic)."""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    r = torch.where(torch.isnan(x), torch.full_like(r, 0x7FFF), r)
    return (r & 0xFFFF).to(torch.int32).to(torch.int16).view(torch.bfloat16).view(x.shape)


def bf16_trunc(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> bf16 by dropping the low half (a wrong cast, for the checkers' tests)."""
    b = x.contiguous().view(torch.int32) >> 16
    return b.to(torch.int16).view(torch.bfloat16).view(x.shape)


# ---- references ------------------------------------------------------------------------------------------------------


def a2a(inputs: Sequence[torch.Tensor], scatter_dim: int, gather_dim: int, r: int) -> torch.Tensor:
    W = len(inputs)
    return torch.cat([x.tensor_split(W, scatter_dim)[r] for x in inputs], gather_dim)


def allgather(shards: Sequence[torch.Tensor]) -> torch.Tensor:
    return torch.cat([s.view(-1) if s.dtype == torch.bfloat16 else bf16_rne(s.view(-1)) for s in shards])


def reduce_scatter(inputs: Sequence[torch.Tensor], me: int, scale: float, out_f32: bool, start: int = 0,
                   reverse: bool = False, scale_each: bool = False) -> torch.Tensor:
    """Exact restatement.  ``start`` / ``reverse`` / ``scale_each`` plant the mistakes the CPU tests reject."""
    W = len(inputs)
    n = inputs[0].numel() // W
    s = torch.tensor(scale, dtype=torch.float32, device=inputs[0].device)
    order = [(start + k) % W for k in range(W)]
    if reverse:
        order = order[::-1]
    acc = torch.zeros(n, dtype=torch.float32, device=inputs[0].device)
    for r in order:
        term = inputs[r].view(-1)[me * n : (me + 1) * n].float()
        acc = acc + (term * s if scale_each else term)
    if not scale_each:
        acc = acc * s
    return acc if out_f32 else bf16_rne(acc)


def allreduce(inputs: Sequence[torch.Tensor], scale: float) -> torch.Tensor:
    """Exact restatement of the fp32 all-reduce: the same rank-order sum as :func:`reduce_scatter`, no rank offset."""
    s = torch.tensor(scale, dtype=torch.float32, device=inputs[0].device)
    acc = torch.zeros_like(inputs[0].view(-1), dtype=torch.float32)
    for x in inputs:
        acc = acc + x.view(-1).float()
    return acc * s


def sum_ref64(inputs: Sequence[torch.Tensor], me: int, scale: float, shard: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
    """(float64 reference, S = sum_r |x_r|) of the reduction ``rank me`` computes."""
    W = len(inputs)
    n = inputs[0].numel() // W if shard else inputs[0].numel()
    lo = me * n if shard else 0
    terms = torch.stack([x.view(-1)[lo : lo + n].double() for x in inputs])
    return terms.sum(0) * float(np.float32(scale)), terms.abs().sum(0)


def rs_bound(ref64: torch.Tensor, S: torch.Tensor, W: int, scale: float, out_f32: bool) -> torch.Tensor:
    b = (1 + U32) * gamma(W - 1) * abs(float(np.float32(scale))) * S + U32 * ref64.abs()
    return b if out_f32 else b + BF16_U * (ref64.abs() + b)


# ---- expert-parallel exchange ----------------------------------------------------------------------------------------


def ep_to_experts(cnt: np.ndarray, d: int) -> np.ndarray:
    """[rows, 2] int64 (source rank, row in its source-major buffer), in owner d's expert-major order."""
    W, E = cnt.shape
    E_loc = E // W
    src, row, loc = [], [], []
    for s in range(W):  # the variable-split all-to-all: sources in rank order, each one's rows for d in its order
        expert = np.repeat(np.arange(E), cnt[s])  # source rows are sorted by global expert
        sel = np.nonzero(expert // E_loc == d)[0]
        src.append(np.full(len(sel), s, dtype=np.int64))
        row.append(sel.astype(np.int64))
        loc.append(expert[sel] % E_loc)
    src, row, loc = np.concatenate(src), np.concatenate(row), np.concatenate(loc)
    order = np.argsort(loc, kind="stable")  # the re-sort by local expert
    return np.stack([src[order], row[order]], 1).reshape(-1, 2)


def ep_to_sources(cnt: np.ndarray, s: int, te_all=None) -> np.ndarray:
    """[rows of s, 2] int64 (owner rank, position in its expert-major buffer) holding row p of rank s: the inverse of
    :func:`ep_to_experts` (``te_all``: its result for every owner, when already computed)."""
    W = cnt.shape[0]
    te_all = te_all if te_all is not None else [ep_to_experts(cnt, d) for d in range(W)]
    back = np.full((int(cnt[s].sum()), 2), -1, dtype=np.int64)
    for d, te in enumerate(te_all):
        pos = np.nonzero(te[:, 0] == s)[0]
        back[te[pos, 1], 0] = d
        back[te[pos, 1], 1] = pos
    assert (back >= 0).all()
    return back


def ep_rows(cnt: np.ndarray, row_bytes: int, device="cuda") -> List[torch.Tensor]:
    """Labelled source-major rows of every rank: int32 words (s, r, s * 2^20 + r, then r * 4099 + w + s * 7919 for word w)."""
    W = cnt.shape[0]
    words = row_bytes // 4
    out = []
    for s in range(W):
        M = int(cnt[s].sum())
        r = torch.arange(M, dtype=torch.int64, device=device)[:, None]
        w = torch.arange(words, dtype=torch.int64, device=device)[None, :]
        t = (r * 4099 + w + s * 7919) & 0x7FFFFFFF
        t[:, 0:1] = s
        if words > 1:
            t[:, 1:2] = r
        if words > 2:
            t[:, 2:3] = (s << 20) + r
        out.append(t.to(torch.int32))
    return out


def gather_rows(rows: Sequence[torch.Tensor], pairs: np.ndarray) -> torch.Tensor:
    """rows[pairs[i, 0]][pairs[i, 1]] for every i."""
    if len(pairs) == 0:
        return rows[0][:0]
    dev = rows[0].device
    flat = torch.cat(list(rows))
    base = np.cumsum([0] + [len(r) for r in rows])[:-1]
    idx = torch.as_tensor(base[pairs[:, 0]] + pairs[:, 1], device=dev)
    return flat[idx]


def assert_rows_equal(got: torch.Tensor, want: torch.Tensor, what: str) -> None:
    """int32 row tables equal; a misplaced row is reported by its label (source rank, row)."""
    assert got.shape == want.shape, f"{what}: shape {tuple(got.shape)} vs {tuple(want.shape)}"
    bad = (got != want).any(1)
    if bool(bad.any()):
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} rows differ; row {i} holds label {got[i, :2].tolist()}, "
                             f"want {want[i, :2].tolist()}")


def check_to_experts(out: torch.Tensor, rows: Sequence[torch.Tensor], cnt: np.ndarray, d: int, cap: int, what: str) -> int:
    """``out`` ([>= cap, words] int32, FILL32 where never written) against owner d's reference order: the first
    min(total, cap) rows are the reference's, every later row is untouched.  Returns the total received."""
    want = gather_rows(rows, ep_to_experts(cnt, d))
    n = min(len(want), cap)
    assert_rows_equal(out[:n], want[:n], what)
    assert bool((out[n:] == FILL32).all()), f"{what}: a row at or past min(total={len(want)}, cap={cap}) was written"
    return len(want)


def check_to_sources(out: torch.Tensor, owner_rows: Sequence[torch.Tensor], cnt: np.ndarray, s: int, cap: int, m_rows: int,
                     what: str, te_all=None) -> None:
    """``out`` ([>= rows of s, words] int32) on the way back: row p < m_rows holds owner_rows[d][pos] for the
    (d, pos) of :func:`ep_to_sources` when pos < cap; every other row is untouched."""
    back = ep_to_sources(cnt, s, te_all)
    keep = np.zeros(len(out), dtype=bool)
    keep[: min(m_rows, len(back))] = True
    keep[: len(back)] &= back[:, 1] < cap
    p = np.nonzero(keep)[0]
    if len(p):
        assert_rows_equal(out[torch.as_tensor(p, device=out.device)], gather_rows(owner_rows, back[p]), what)
    rest = torch.as_tensor(np.nonzero(~keep)[0], device=out.device)
    assert bool((out[rest] == FILL32).all()), f"{what}: a row with no fetch (past m_rows or capacity) was written"


def staging(cnt_row: np.ndarray, rows: torch.Tensor, hdr_bytes: int) -> torch.Tensor:
    """Bytes of a source-major staging buffer: int32 cnt[E], zero-padded to hdr_bytes, then the rows."""
    hdr = torch.zeros(hdr_bytes // 4, dtype=torch.int32, device=rows.device)
    hdr[: len(cnt_row)] = torch.as_tensor(np.asarray(cnt_row, dtype=np.int32), device=rows.device)
    return torch.cat([hdr.view(torch.uint8), rows.contiguous().view(torch.uint8).view(-1)])


def ep_counts(W: int, E: int, load: str, seed: int, rows_per_rank: int = 256) -> np.ndarray:
    """cnt[W, E] int64.  uniform, zipf, holes (most experts empty), empty_rank (rank 1 sends nothing) or one_owner
    (every row goes to experts of rank W - 1)."""
    rng = np.random.default_rng(seed)
    mean = max(1, rows_per_rank // E)
    if load == "uniform":
        cnt = rng.integers(0, 2 * mean + 1, size=(W, E))
    elif load == "zipf":
        cnt = np.minimum(rng.zipf(1.6, size=(W, E)) - 1, 8 * mean)
    elif load == "holes":
        cnt = rng.integers(1, 4 * mean + 1, size=(W, E)) * (rng.random((W, E)) < 0.25)
    elif load == "empty_rank":
        cnt = rng.integers(0, 2 * mean + 1, size=(W, E))
        cnt[min(1, W - 1)] = 0
    elif load == "one_owner":
        cnt = np.zeros((W, E), dtype=np.int64)
        E_loc = E // W
        cnt[:, (W - 1) * E_loc :] = rng.integers(0, 2 * mean * W + 1, size=(W, E_loc))
    else:
        raise ValueError(load)
    return cnt.astype(np.int64)


# ---- inputs ----------------------------------------------------------------------------------------------------------


def _gen(seed: int, device) -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def rank_values(W: int, n: int, mode: str, seed: int, dtype=torch.bfloat16, device="cuda") -> List[torch.Tensor]:
    """W flat tensors.  exact: integers in [-4, 4] times 2^k, k in [0, 16] per rank; random: N(0, 1) times 2^k, k in
    [-40, 40] per rank; cancel: N(0, 1) on every rank except 2^20 x on rank 0 and -2^20 x on rank W - 1 (W >= 2)."""
    g = _gen(seed, device)
    if mode == "cancel":
        out = [torch.randn(n, generator=g, device=device).to(dtype) for _ in range(W)]
        out[0] = (torch.randn(n, generator=g, device=device) * 2.0 ** 20).to(dtype)
        out[-1] = -out[0]
        return out
    lo, hi = (0, 16) if mode == "exact" else (-40, 40)
    ks = torch.randint(lo, hi + 1, (W,), generator=g, device=device)
    out = []
    for r in range(W):
        if mode == "exact":
            v = torch.randint(-4, 5, (n,), generator=g, device=device).float()
        else:
            v = torch.randn(n, generator=g, device=device)
        out.append((v * torch.pow(2.0, ks[r].float())).to(dtype))
    return out


def labels(nbytes: int, rank: int, device="cuda") -> torch.Tensor:
    """nbytes (multiple of 4) of 32-bit words rank * 2^27 + word index (mod 2^31): names its source and position."""
    i = torch.arange(nbytes // 4, dtype=torch.int64, device=device)
    return ((i + rank * (1 << 27)) & 0x7FFFFFFF).to(torch.int32).view(torch.uint8)


F32_SPECIAL_BITS = [
    0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,  # RNE ties: even stays, odd rounds up (both signs)
    0x3F80FFFF, 0x3F808001, 0x3F807FFF,              # just above / below a tie
    0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000,              # round to +-inf
    0x7F7F7FFF,                                      # largest that stays finite
    0x00000001, 0x80000001, 0x00008000, 0x00018000, 0x007FFFFF, 0x807FFFFF,  # subnormals (incl. ties)
    0x00000000, 0x80000000, 0x7F800000, 0xFF800000,  # +-0, +-inf
    0x7FC00000, 0xFFC00001, 0x7F800001, 0x7FBFFFFF,  # NaN (quiet, negative, signalling)
]


def f32_specials(n: int, device="cuda", seed: int = 0) -> torch.Tensor:
    """n fp32 values: every special class above, repeated, mixed with N(0, 1)."""
    sp = torch.tensor(np.array(F32_SPECIAL_BITS, dtype=np.uint32).view(np.int32), device=device).view(torch.float32)
    x = torch.randn(n, generator=_gen(seed, device), device=device)
    k = min(n, 4 * len(sp))
    x[:k] = sp.repeat(4)[:k]
    return x
