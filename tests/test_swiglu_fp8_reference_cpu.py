"""CPU self-tests of ``tests/swiglu_fp8_reference.py``: the SwiGLU checks accept torch's own autograd of
``silu(g) * u`` (bf16, as the reference runs it) and reject fp32 restatements that drop one of its bf16 roundings; the
fp8 model equals the oracle's restatements of the reference, NaN, inf and all-zero blocks included; and a numpy model
of the SwiGLU backward's row split shows its 32-bit reciprocal exact up to the widest accepted row."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import moe_oracle as O
from tests import swiglu_fp8_reference as R

pytestmark = pytest.mark.filterwarnings("ignore")


def _torch_swiglu(h, d):
    """(a, grad_h) of torch's bf16 autograd: the reference's native_swiglu (silu output a bf16 tensor, then the mul)."""
    h = h.clone().requires_grad_(True)
    I = h.shape[1] // 2
    a = F.silu(h[:, :I]) * h[:, I:]
    a.backward(d)
    return a.detach(), h.grad


def _inputs(seed=0, M=64, I=1024):
    """bf16 h [M, 2I] whose gate half spans magnitudes 2^-6 to 2^6 times N(0, 1), with the zero of 1 + g (1 - sigmoid(g))
    and bf16 subnormals in it, and d [M, I]."""
    gen = torch.Generator().manual_seed(seed)
    g = torch.randn(M, I, generator=gen, dtype=torch.float64) * torch.pow(4.0, torch.randint(-3, 4, (M, 1), generator=gen))
    g[0, :64] = -1.2785 + torch.arange(64, dtype=torch.float64) * 2.0 ** -10
    g[1, :64] = torch.arange(64, dtype=torch.float64) * 2.0 ** -133
    u = torch.randn(M, I, generator=gen, dtype=torch.float64) * 3
    d = torch.randn(M, I, generator=gen, dtype=torch.float64)
    return torch.cat([g, u], 1).to(torch.bfloat16), d.to(torch.bfloat16)


def test_torch_autograd_passes_the_swiglu_checks():
    h, d = _inputs()
    a, gh = _torch_swiglu(h, d)
    R.check_swiglu_fwd(h, a, "torch swiglu")
    R.check_swiglu_bwd(h, d, gh, "torch swiglu backward")


def test_bf16_round_and_neighbour():
    x = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -40, 2.0 ** -134, 2.0 ** -134 * 3,
                      -2.0 ** -135, R.BF16_MAX, R.BF16_OVERFLOW, R.BF16_OVERFLOW * (1 - 2.0 ** -30)], dtype=torch.float64)
    want = torch.tensor([1.0, 1.0 + 2 * 2.0 ** -7, 1.0 + 2.0 ** -7, 0.0, 2.0 ** -132, -0.0, R.BF16_MAX, float("inf"),
                         R.BF16_MAX], dtype=torch.float64)
    got = R.bf16_round(x)
    assert torch.equal(got.double(), want), got
    # one rounding: fp32 first would turn 1 + 2^-8 + 2^-40 into the tie 1 + 2^-8 and then round to 1
    assert got[2].item() != x[2:3].float().to(torch.bfloat16).item()
    nb = R.bf16_neighbour(got, x)
    assert nb[2].item() == 1.0 and nb[4].item() == 2.0 ** -133 and nb[5].item() == -(2.0 ** -133)


def test_swiglu_checks_reject_a_missing_rounding_of_s():
    h, d = _inputs(1)
    I = h.shape[1] // 2
    g, u = h[:, :I].float(), h[:, I:].float()
    s32 = g * torch.sigmoid(g)  # fp32 silu, never rounded to bf16
    a = (s32 * u).to(torch.bfloat16)
    with pytest.raises(AssertionError):
        R.check_swiglu_fwd(h, a, "s not rounded")
    _, gh = _torch_swiglu(h, d)
    gh = gh.clone()
    gh[:, I:] = (d.float() * s32).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="grad_u"):
        R.check_swiglu_bwd(h, d, gh, "s not rounded")


def test_swiglu_checks_reject_a_missing_rounding_of_ds():
    h, d = _inputs(2)
    I = h.shape[1] // 2
    g, u = h[:, :I].float(), h[:, I:].float()
    sig = torch.sigmoid(g)
    _, gh = _torch_swiglu(h, d)
    gh = gh.clone()
    gh[:, :I] = ((d.float() * u) * sig * (1 + g * (1 - sig))).to(torch.bfloat16)  # ds kept in fp32
    with pytest.raises(AssertionError, match="grad_g"):
        R.check_swiglu_bwd(h, d, gh, "ds not rounded")


def test_swiglu_model_of_the_fp32_overflow_band():
    """From g = -88.72 on, 1 + exp(-g) is inf in fp32 and both the kernel's and torch's sigmoid are 0, although g e^g
    is still a normal bf16 value down to g = -92: the references model that band as computed, so torch passes there and
    the float64 value (what an e^g branch would give) does not."""
    g = torch.tensor([[-88.5, -89.0, -90.0, -91.0, -92.0, -100.0, -1e30]], dtype=torch.bfloat16)
    h = torch.cat([g, torch.full_like(g, 3.0)], 1)
    d = torch.ones_like(g)
    a, gh = _torch_swiglu(h, d)
    R.check_swiglu_fwd(h, a, "torch in the overflow band")
    R.check_swiglu_bwd(h, d, gh, "torch in the overflow band")
    assert a[0, 0].item() != 0 and bool((a[0, 1:] == 0).all())
    x = g.double()
    exact = (x * torch.exp(x) * 3).to(torch.bfloat16)
    assert exact[0, 1].item() != 0
    with pytest.raises(AssertionError):
        R.check_swiglu_fwd(h, exact, "float64 silu in the overflow band")


def test_swiglu_bound_is_absolute_at_the_zero_of_the_derivative():
    """Around g = -1.2785, 1 + g (1 - sigmoid(g)) is 0 and grad_g is tiny: a bound relative to grad_g would be 0 there."""
    g = (-1.2785 + torch.arange(-256, 256, dtype=torch.float64) * 2.0 ** -14).to(torch.bfloat16).unique()
    ds = torch.ones_like(g)
    ref, bound = R.grad_g_ref(g, ds)
    i = int(ref.abs().argmin())
    assert abs(ref[i].item()) < 1e-2 and bound[i].item() > 1e-7


def test_e4m3_model_equals_the_oracle_cast():
    v = R.cast_sweep_values().double()
    extra = torch.tensor([float("inf"), -float("inf"), 449.0, 463.99, 464.0, 465.0, -1e30, 2.0 ** -10, 3 * 2.0 ** -11,
                          2.0 ** -10 + 2.0 ** -30, -(2.0 ** -11)], dtype=torch.float64)
    for x in (v, extra):
        want = O.to_fp8_saturated(x.float()).view(torch.uint8)
        R.assert_fp8_equal(R.e4m3_bits(x.float().double()), want, "e4m3 model")
    n = R.e4m3_bits(torch.tensor([float("nan"), -float("nan")], dtype=torch.float64))
    assert [int(b) & 0x7F for b in n] == [0x7F, 0x7F]


def _special_weights(dtype):
    gen = torch.Generator().manual_seed(3)
    w = (torch.randn(3, 256, 384, generator=gen) * 2).to(dtype)
    w[0, :128, :128] = 0  # all-zero block
    w[0, 128:, 128:256] *= 1e-14  # amax under 1e-12
    w[1, 5, 300] = float("nan")
    w[2, 130, 7] = float("inf")
    w[2, 200, 200] = -float("inf")
    return w


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fp8_block_model_equals_the_oracle(dtype):
    w = _special_weights(dtype)
    s = R.block_scales(w)
    R.assert_scales_equal(s, O.per_block_fp8_scales(w), "block scales")
    assert torch.isnan(s[1, 0, 2]) and torch.isinf(s[2, 1, 0]) and torch.isinf(s[2, 1, 1])
    assert s[0, 0, 0].item() == torch.tensor(1e-12 / 448, dtype=torch.float64).float().item()
    for i in range(3):
        q = R.block_cast(w[i], s[i])
        R.assert_fp8_equal(q, O.cast_to_per_block_fp8(w[i], s[i]), f"block cast {i}")
    q = R.block_cast(w[1], s[1]).view(2, 128, 3, 128)[0, :, 2]
    assert bool(((q & 0x7F) == 0x7F).all())  # the NaN block is NaN throughout
    q = R.block_cast(w[2], s[2])
    assert (int(q[130, 7]) & 0x7F) == 0x7F and int(q[130, 8]) in (0, 0x80)


def test_fp8_tile_model_equals_the_oracle():
    gen = torch.Generator().manual_seed(4)
    x = (torch.randn(16, 512, generator=gen) * 4).to(torch.bfloat16)
    x[0, :128] = 0
    x[1, 128:256] *= 1e-14
    x[2, 300] = float("nan")
    x[3, 5] = float("inf")
    q, s = R.tile_quant(x)
    rq, rs = O.per_tile_quant(x)
    R.assert_scales_equal(s, rs, "tile scales")
    R.assert_fp8_equal(q, rq, "tile cast")
    assert torch.isnan(s[2, 2]) and torch.isinf(s[3, 0])


def test_amax_one_tiles_hold_the_sweep_at_scale_one():
    v = R.cast_sweep_values()
    t = R.amax_one_tiles(v)
    assert t.shape[1] == 128 and bool((t.float().abs().amax(1) == 448).all())
    assert torch.equal(t[:, 1:].reshape(-1)[: v.numel()].view(torch.int16), v.view(torch.int16))
    _, s = R.tile_quant(t)
    assert bool((s == 1).all())


def test_row_split_reciprocal_exhaustive_to_2048():
    """umulhi(i, ceil(2^32 / I8)) == i // I8 for every i a block of kSwRows rows can hold, I8 = 2..2048 (I8 = 1 is
    special-cased in the kernel: 2^32 does not fit 32 bits)."""
    for I8 in range(2, 2049):
        i = np.arange(R.SW_ROWS * I8, dtype=np.uint64)
        r = R.umulhi(i, np.uint64(R.row_split_inverse(I8)))
        assert np.array_equal(r, i // np.uint64(I8)), I8


def test_row_split_reciprocal_at_the_widest_rows():
    """The error of the reciprocal grows with i and peaks at the last column of the last row, i = kSwRows I8 - 1; the
    host check accepts I8 up to 23170 (kSwRows I8^2 < 2^32)."""
    assert R.SW_ROWS * R.SW_I8_MAX ** 2 < 2 ** 32 <= R.SW_ROWS * (R.SW_I8_MAX + 1) ** 2
    for I8 in range(23100, R.SW_I8_MAX + 1):
        inv = R.row_split_inverse(I8)
        for i in (R.SW_ROWS * I8 - 1, R.SW_ROWS * I8 - I8, (R.SW_ROWS - 1) * I8 - 1):
            assert R.umulhi(i, inv) == i // I8, (I8, i)
    # floor instead of ceil is wrong at the first column of row 1 for any I8 that is not a power of two
    assert R.umulhi(3, ((1 << 32) // 3)) != 1
