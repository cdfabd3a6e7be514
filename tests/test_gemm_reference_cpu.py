"""The checker of tests/gemm_reference.py against itself, on the CPU: it accepts what a correct kernel computes (fp32
accumulation, round-to-nearest to bf16) and rejects each of the ways a grouped GEMM has been seen to go subtly wrong —
a dropped 64-deep k-block, a row on the wrong side of an expert boundary, two experts' weights swapped, the gate and up
column tiles of the SwiGLU GEMM swapped, truncation instead of rounding.  Exact-mode inputs are judged by the bit-exact
check the exact GPU tests use, random-mode inputs by the scale-aware bound."""
import pytest
import torch

from tests import gemm_reference as R

COUNTS = [17, 64, 0, 129, 64, 65]  # experts 1 and 4 have equal sizes; expert 2 is empty
E = len(COUNTS)
M = sum(COUNTS)
N, KD, I = 256, 1024, 256  # I = 256: the SwiGLU GEMM's 256-wide tiles, so n_blk = 1 exists


def _fp32(kind, a, b, counts, rn=True):
    """What a correct kernel computes: fp32 accumulation, then bf16 by round-to-nearest-even (or, rn=False, truncation)."""
    o = R.offsets(counts)
    if kind == "tn":
        out = torch.zeros((len(counts), a.shape[1], b.shape[1]), dtype=torch.float32)
        for e in range(len(counts)):
            out[e] = a[o[e] : o[e + 1]].float().T @ b[o[e] : o[e + 1]].float()
    else:
        out = torch.zeros((a.shape[0], b.shape[1] if kind == "nt" else b.shape[2]), dtype=torch.float32)
        for e in range(len(counts)):
            bw = b[e].float()
            out[o[e] : o[e + 1]] = a[o[e] : o[e + 1]].float() @ (bw.T if kind == "nt" else bw)
    if rn:
        return out.to(torch.bfloat16)
    return (out.view(torch.int32) >> 16).to(torch.int16).view(torch.bfloat16)  # drop the low 16 bits


def _operands(kind, mode):
    if kind == "nt":
        return R.rows_operand(COUNTS, KD, mode, 1), R.weight_operand(E, N, KD, mode, 2)
    if kind == "nn":
        return R.rows_operand(COUNTS, N, mode, 3), R.weight_operand(E, N, KD, mode, 4)
    return R.rows_operand(COUNTS, N, mode, 5), R.rows_operand(COUNTS, KD, mode, 6)


def _check(mode, out, kind, a, b, counts=COUNTS):
    if mode == "exact":
        R.assert_exact(out, kind, a, b, counts)
    else:
        R.check_bound(out, kind, a, b, counts)


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("kind", ["nt", "nn", "tn"])
def test_checker_accepts_fp32_accumulation_rounded_to_nearest(kind, mode):
    a, b = _operands(kind, mode)
    out = _fp32(kind, a, b, COUNTS)
    _check(mode, out, kind, a, b)
    assert R.check_bound(out, kind, a, b, COUNTS) <= 1.0
    if kind == "tn":
        assert not out[2].any()


def test_exact_mode_sums_are_exact_in_fp32():
    """The premise of exact mode: fp32 accumulation in any order lands on the fp64 sum, at a 16384-term reduction too."""
    counts = [16384, 0, 300]
    dy, x = R.rows_operand(counts, 128, "exact", 7), R.rows_operand(counts, 128, "exact", 8)
    ref = R.reference("tn", dy, x, counts)
    fwd = _fp32("tn", dy, x, counts)
    rev = _fp32("tn", dy.flip(0), x.flip(0), counts[::-1]).flip(0)  # the reversed row order sums in the other direction
    assert torch.equal(fwd, R.bf16_rn(ref)) and torch.equal(rev, R.bf16_rn(ref))
    assert float(ref.abs().max() / 2.0 ** (2 * R.SCALE_EXP[1])) < 2 ** 24


def test_per_expert_scales_differ_between_neighbours():
    s = R.expert_scales(1024, 3)
    assert all(a != b for a, b in zip(s, s[1:]))
    assert min(s) == 2.0 ** -8 and max(s) == 2.0 ** 8


def test_count_patterns():
    for E_ in (8, 33, 128):
        c = R.counts_pattern(E_, "ragged", 1)
        assert c[0] == 0 and c[-1] == 0 and set(c) <= set(R.ROW_COUNTS)
        assert c[E_ // 2 : E_ // 2 + 2] == [0, 0] and c.count(0) == 4
    z = R.counts_pattern(128, "zipf", 1, 32768)
    assert sum(z) == 32768 and z[0] == z[-1] == 0 and z.count(0) >= 8 and max(z) > 8 * 32768 // 128
    s = R.counts_pattern(1024, "sparse", 1)
    assert s.count(0) > 990 and sum(s) > 0


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("kind", ["nt", "tn"])
def test_checker_rejects_a_dropped_k_block(kind, mode):
    a, b = _operands(kind, mode)
    a2 = a.clone()
    o = R.offsets(COUNTS)
    if kind == "nt":
        a2[o[3] : o[4], 64:128] = 0  # expert 3 skips reduction columns [64, 128)
    else:
        a2[o[3] + 64 : o[3] + 128] = 0  # expert 3's dW skips its token rows [64, 128)
    with pytest.raises(AssertionError):
        _check(mode, _fp32(kind, a2, b, COUNTS), kind, a, b)


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("kind", ["nt", "tn"])
@pytest.mark.parametrize("shift", [-1, 1])
def test_checker_rejects_a_row_across_an_expert_boundary(kind, mode, shift):
    """shift -1: expert 3 misses its last row (it goes to expert 4); +1: expert 3 takes expert 4's first row."""
    a, b = _operands(kind, mode)
    wrong = list(COUNTS)
    wrong[3] += shift
    wrong[4] -= shift
    with pytest.raises(AssertionError):
        _check(mode, _fp32(kind, a, b, wrong), kind, a, b)


@pytest.mark.parametrize("mode", ["exact", "random"])
def test_checker_rejects_swapped_expert_weights(mode):
    x, w = _operands("nt", mode)
    assert COUNTS[1] == COUNTS[4]
    w2 = w.clone()
    w2[[1, 4]] = w[[4, 1]]
    with pytest.raises(AssertionError):
        _check(mode, _fp32("nt", x, w2, COUNTS), "nt", x, w)


@pytest.mark.parametrize("mode", ["exact", "random"])
def test_checker_rejects_swapped_gate_and_up_tiles(mode):
    """The SwiGLU GEMM's tile n_blk = 1 (256 wide) holds gate columns [128, 256) and up columns [I + 128, I + 256)."""
    x, w13 = R.rows_operand(COUNTS, KD, mode, 9), R.weight_operand(E, 2 * I, KD, mode, 10)
    h = _fp32("nt", x, w13, COUNTS)
    _check(mode, h, "nt", x, w13)
    bad = h.clone()
    bad[:, 128:256], bad[:, I + 128 : I + 256] = h[:, I + 128 : I + 256], h[:, 128:256]
    with pytest.raises(AssertionError):
        _check(mode, bad, "nt", x, w13)


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("kind", ["nt", "nn", "tn"])
def test_checker_rejects_truncation_to_bf16(kind, mode):
    a, b = _operands(kind, mode)
    with pytest.raises(AssertionError):
        _check(mode, _fp32(kind, a, b, COUNTS, rn=False), kind, a, b)


def test_bound_rejects_a_dropped_k_block_at_the_benchmark_reduction():
    """H = 2048, the longest NT reduction of the benchmark, with unit scales: a dropped k-block still shows."""
    counts = [300]
    x, w = R.rows_operand(counts, 2048, "random", 11, exp_range=(0, 0)), R.weight_operand(1, 128, 2048, "random", 12, exp_range=(0, 0))
    out = _fp32("nt", x, w, counts)
    assert R.check_bound(out, "nt", x, w, counts) <= 1.0
    x2 = x.clone()
    x2[:, :64] = 0
    with pytest.raises(AssertionError):
        R.check_bound(_fp32("nt", x2, w, counts), "nt", x, w, counts)


def test_swiglu_act_and_ulp_distance():
    h = (torch.randn(64, 256, generator=torch.Generator().manual_seed(0)) * 2).to(torch.bfloat16)
    a = R.swiglu_act(h)
    from oracle import moe_oracle as O

    d = R.ulp_distance(a, O.swiglu(h))
    assert int(d.max()) <= 1 and float((d > 0).float().mean()) < 1e-2
    z = torch.tensor([0.0, -0.0, 1.0], dtype=torch.bfloat16)
    assert R.ulp_distance(z, torch.tensor([-0.0, 0.0, 1.0078125], dtype=torch.bfloat16)).tolist() == [0, 0, 1]
