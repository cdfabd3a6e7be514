"""The references and checkers of tests/exchange_reference.py on CPU: they accept correct emulations of the exchange
kernels (written the way the kernels compute: the a2a byte gather from its plan, the 4-wide rank batches of the
reductions, the expert-parallel offset tables) and reject each planted mistake on inputs where it shows."""
import dataclasses

import numpy as np
import pytest
import torch

from tests import exchange_reference as R
from xtuner_b200.comm import a2a_plan, apply_plan_reference

CPU = "cpu"


# ---- emulations of the kernels (the same loops, in Python) -----------------------------------------------------------


def _rs_kernel(inputs, me, scale, out_f32):
    """reduce_scatter_pull_kernel: ranks in batches of 4, each batch added in order into one fp32 accumulator."""
    W = len(inputs)
    n = inputs[0].numel() // W
    acc = torch.zeros(n, dtype=torch.float32)
    for r0 in range(0, W, 4):
        for j in range(4):
            if r0 + j < W:
                acc = acc + inputs[r0 + j][me * n : (me + 1) * n].float()
    acc = acc * torch.tensor(scale, dtype=torch.float32)
    return acc if out_f32 else acc.to(torch.bfloat16)


def _a2a_kernel(inputs, plan):
    """a2a_pull_kernel: every (source, o, x, m) row copied from its plan offsets; writes that fall outside the output
    are dropped (a wrong plan must fail the comparison, not the emulation)."""
    n_out = int(np.prod(plan.out_shape)) * inputs[0].element_size()
    ob = torch.zeros(n_out, dtype=torch.uint8)
    for src, t in enumerate(inputs):
        ib = t.contiguous().view(-1).view(torch.uint8)
        for o in range(plan.n_o):
            for x in range(plan.n_x):
                for m in range(plan.n_m):
                    so = plan.src_base + o * plan.src_stride_o + x * plan.src_stride_x + m * plan.src_stride_m
                    do = src * plan.dst_peer_stride + o * plan.dst_stride_o + x * plan.dst_stride_x + m * plan.dst_stride_m
                    k = max(0, min(plan.row_bytes, n_out - do))
                    ob[do : do + k] = ib[so : so + k]
    return ob.view(inputs[0].dtype).view(plan.out_shape)


def _ep_tables(cnt, me, rem0_le=False):
    W, E = cnt.shape
    El = E // W
    src0 = np.zeros(El * W, dtype=np.int64)
    for s in range(W):
        run = int(cnt[s, : me * El].sum())
        for j in range(El):
            src0[j * W + s] = run
            run += cnt[s, me * El + j]
    rem0 = np.zeros(E, dtype=np.int64)
    for d in range(W):
        run = 0
        for j in range(El):
            e = d * El + j
            before = int(cnt[: me + (1 if rem0_le else 0), e].sum())
            rem0[e] = run + before
            run += int(cnt[:, e].sum())
    return src0, rem0


def _to_experts_kernel(cnt, me, rows, cap, order="es", clamp=True):
    """ep_pull_to_experts_kernel on CPU: segments (j, s) in that order ("se": the planted (source, expert) order)."""
    W, E = cnt.shape
    El = E // W
    src0, _ = _ep_tables(cnt, me)
    segs = [(j, s) for j in range(El) for s in range(W)] if order == "es" else [(j, s) for s in range(W) for j in range(El)]
    out = torch.full((max(cap, 1) + 8, rows[0].shape[1]), R.FILL32, dtype=torch.int32)
    row = 0
    for j, s in segs:
        for i in range(int(cnt[s, me * El + j])):
            if row < cap or not clamp:
                if row < len(out):
                    out[row] = rows[s][src0[j * W + s] + i]
            row += 1
    return out


def _to_sources_kernel(cnt, me, owner_rows, cap, m_rows, rem0_le=False):
    W, E = cnt.shape
    El = E // W
    _, rem0 = _ep_tables(cnt, me, rem0_le)
    M = int(cnt[me].sum())
    out = torch.full((M + 4, owner_rows[0].shape[1]), R.FILL32, dtype=torch.int32)
    row = 0
    for e in range(E):
        for i in range(int(cnt[me, e])):
            src = rem0[e] + i
            if row < m_rows and src < cap and src < len(owner_rows[e // El]):  # a wrong table may point past the owner's rows
                out[row] = owner_rows[e // El][src]
            row += 1
    return out


# ---- casts -----------------------------------------------------------------------------------------------------------


def test_bf16_rne_matches_torch_and_specials():
    x = R.f32_specials(4096, device=CPU)
    got, want = R.bf16_rne(x), x.to(torch.bfloat16)
    R.assert_bits_equal(got, want, "bf16_rne vs torch")
    bits = got.view(torch.int16).to(torch.int32) & 0xFFFF
    assert bool((bits[torch.isnan(x)] == 0x7FFF).all())
    # ties: 0x3F808000 -> 0x3F80 (even stays), 0x3F818000 -> 0x3F82 (odd rounds up); the max float rounds to inf
    assert bits[:4].tolist() == [0x3F80, 0x3F82, 0xBF80, 0xBF82]
    assert bits[7].item() == 0x7F80 and bits[8].item() == 0xFF80
    with pytest.raises(AssertionError):
        R.assert_bits_equal(R.bf16_trunc(x), want, "truncation")


# ---- a2a -------------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("shape,s,g", [((1, 8, 6, 16), 1, 2), ((1, 8, 6, 16), 2, 1), ((2, 4, 3, 8, 4), 3, 1)])
def test_a2a_reference_accepts_plan_emulation_and_rejects_swapped_strides(shape, s, g):
    W = 2 if shape[s] % 4 else 4
    inputs = [R.labels(int(np.prod(shape)) * 4, r, CPU).view(torch.float32).view(shape) for r in range(W)]
    for r in range(W):
        plan = a2a_plan(shape, s, g, W, r, 4)
        R.assert_bits_equal(apply_plan_reference(inputs, plan), R.a2a(inputs, s, g, r), "a2a plan emulation")
        R.assert_bits_equal(_a2a_kernel(inputs, plan), R.a2a(inputs, s, g, r), "a2a kernel emulation")
        # the peer stride and the chunk stride swapped
        chunk = "dst_stride_x" if s < g else "dst_stride_m"
        bad = dataclasses.replace(plan, dst_peer_stride=getattr(plan, chunk), **{chunk: plan.dst_peer_stride})
        with pytest.raises(AssertionError):
            R.assert_bits_equal(_a2a_kernel(inputs, bad), R.a2a(inputs, s, g, r), "swapped strides")


# ---- all-gather ------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_allgather_reference_rejects_offset_zero(dtype):
    W, n = 3, 256
    shards = [R.f32_specials(n, CPU, seed=r).to(dtype) if dtype == torch.bfloat16 else R.f32_specials(n, CPU, seed=r)
              for r in range(W)]
    emu = torch.empty(W * n, dtype=torch.bfloat16)
    for r in range(W):
        emu[r * n : (r + 1) * n] = shards[r].to(torch.bfloat16)
    R.assert_bits_equal(emu, R.allgather(shards), "all-gather emulation")
    bad = emu.clone()
    for r in range(W):
        bad[:n] = shards[r].to(torch.bfloat16)  # every rank writes at offset 0
    with pytest.raises(AssertionError):
        R.assert_bits_equal(bad, R.allgather(shards), "offset 0")


# ---- reductions ------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("W", [2, 3, 5, 8])
@pytest.mark.parametrize("out_f32", [True, False])
def test_reduce_scatter_checkers(W, out_f32):
    n = 4096
    me = W - 1
    scale = 1.0 / 3.0
    # a bf16 output hides most one-ulp fp32 differences; ranks 0 and W - 1 cancel exactly (2^20 x and -2^20 x) so that
    # where the small ranks' bits are lost depends on the order and the scale, by far more than a bf16 ulp
    mode = "random" if out_f32 or W == 2 else "cancel"
    rnd = R.rank_values(W, W * n, mode, seed=W, device=CPU)
    want = R.reduce_scatter(rnd, me, scale, out_f32)
    R.assert_bits_equal(_rs_kernel(rnd, me, scale, out_f32), want, "4-wide batched emulation")
    ref64, S = R.sum_ref64(rnd, me, scale)
    r = R.assert_within(_rs_kernel(rnd, me, scale, out_f32), ref64, R.rs_bound(ref64, S, W, scale, out_f32), "fp64")
    assert 0 < r <= 1
    wrong = {}
    if mode != "random" or out_f32:
        wrong["scale per term"] = R.reduce_scatter(rnd, me, scale, out_f32, scale_each=True)
    if W > 2:  # fp32 addition of two terms commutes: the order only shows from three ranks on
        wrong["reverse rank order"] = R.reduce_scatter(rnd, me, scale, out_f32, reverse=True)
        wrong["sum started at rank me"] = R.reduce_scatter(rnd, me, scale, out_f32, start=me)
    if not out_f32:
        wrong["truncating cast"] = R.bf16_trunc(R.reduce_scatter(rnd, me, scale, True))
    for what, bad in wrong.items():
        with pytest.raises(AssertionError):
            R.assert_bits_equal(bad, want, what)
    # exact mode: every order gives the same bits, and they equal the exactly rounded sum
    ex = R.rank_values(W, W * n, "exact", seed=W, device=CPU)
    ref64, _ = R.sum_ref64(ex, me, 1.0)
    R.assert_bits_equal(R.reduce_scatter(ex, me, 1.0, True, reverse=True), ref64.float(), "exact sum")


def test_allreduce_reference_matches_reduce_scatter_of_replicated_rows():
    W, n = 5, 1024
    x = R.rank_values(W, n, "random", seed=1, dtype=torch.float32, device=CPU)
    want = R.allreduce(x, 0.25)
    rep = [t.repeat(W) for t in x]
    for me in range(W):
        R.assert_bits_equal(R.reduce_scatter(rep, me, 0.25, True), want, f"rank {me}")
    ref64, S = R.sum_ref64(x, 0, 0.25, shard=False)
    R.assert_within(want, ref64, R.rs_bound(ref64, S, W, 0.25, True), "all-reduce fp64")


# ---- expert-parallel pulls -------------------------------------------------------------------------------------------


@pytest.mark.parametrize("W,E,load", [(2, 8, "uniform"), (4, 16, "zipf"), (4, 8, "holes"), (3, 6, "empty_rank"),
                                      (4, 8, "one_owner"), (1, 4, "uniform")])
def test_ep_checkers_accept_kernel_tables(W, E, load):
    cnt = R.ep_counts(W, E, load, seed=W + E, rows_per_rank=64)
    rows = R.ep_rows(cnt, 32, CPU)
    owner = []
    for d in range(W):
        cap = int(cnt.sum())
        out = _to_experts_kernel(cnt, d, rows, cap)
        R.check_to_experts(out, rows, cnt, d, cap, f"owner {d}")
        owner.append(out)
    for s in range(W):
        M = int(cnt[s].sum())
        R.check_to_sources(_to_sources_kernel(cnt, s, owner, int(cnt.sum()), M), owner, cnt, s, int(cnt.sum()), M, f"src {s}")
        R.assert_rows_equal(_to_sources_kernel(cnt, s, owner, int(cnt.sum()), M)[:M], rows[s], f"round trip {s}")


def test_ep_checkers_reject_planted_mistakes():
    W, E = 3, 6
    cnt = R.ep_counts(W, E, "uniform", seed=7, rows_per_rank=60)
    assert (cnt > 0).sum() > 12
    rows = R.ep_rows(cnt, 16, CPU)
    total = [len(R.ep_to_experts(cnt, d)) for d in range(W)]
    # to-experts segments in (source, expert) order
    with pytest.raises(AssertionError, match="label"):
        R.check_to_experts(_to_experts_kernel(cnt, 1, rows, total[1], order="se"), rows, cnt, 1, total[1], "order")
    # capacity clamp ignored
    cap = total[0] - 3
    R.check_to_experts(_to_experts_kernel(cnt, 0, rows, cap), rows, cnt, 0, cap, "clamped")
    with pytest.raises(AssertionError, match="written"):
        R.check_to_experts(_to_experts_kernel(cnt, 0, rows, cap, clamp=False), rows, cnt, 0, cap, "no clamp")
    # rem0 counting ranks <= me
    owner = [_to_experts_kernel(cnt, d, rows, total[d]) for d in range(W)]
    big = int(cnt.sum())
    for s in (0, 2):
        M = int(cnt[s].sum())
        R.check_to_sources(_to_sources_kernel(cnt, s, owner, big, M), owner, cnt, s, big, M, "rem0")
        with pytest.raises(AssertionError):
            R.check_to_sources(_to_sources_kernel(cnt, s, owner, big, M, rem0_le=True), owner, cnt, s, big, M, "rem0 <=")
    # on the way back, a fetch past the owner's capacity must leave the row untouched
    M = int(cnt[2].sum())
    R.check_to_sources(_to_sources_kernel(cnt, 2, owner, 5, M), owner, cnt, 2, 5, M, "cap")
    with pytest.raises(AssertionError, match="written"):
        R.check_to_sources(_to_sources_kernel(cnt, 2, owner, big, M), owner, cnt, 2, 5, M, "cap ignored")


def test_staging_layout():
    cnt = np.array([[2, 0, 3]])
    rows = R.ep_rows(cnt, 16, CPU)[0]
    b = R.staging(cnt[0], rows, R.ep_hdr_bytes(3))
    assert R.ep_hdr_bytes(3) == 256 and R.ep_hdr_bytes(64) == 256 and R.ep_hdr_bytes(65) == 512
    assert b[:12].view(torch.int32).tolist() == [2, 0, 3] and bool((b[12:256] == 0).all())
    assert torch.equal(b[256:].view(torch.int32).view(5, 4), rows)
    assert rows[:, 0].tolist() == [0] * 5 and rows[:, 1].tolist() == list(range(5))
