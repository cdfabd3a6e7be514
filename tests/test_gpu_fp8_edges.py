"""fp8 quantisation kernels (``csrc/fp8.cu``) on an H100 against the float64 model of
``tests/swiglu_fp8_reference.py``, the oracle and the reference's own functions, at the edges ``tests/test_gpu_fp8.py``
does not reach:

* every bf16 value in [-448, 448] through the e4m3 cast at scale exactly 1 (tiles and blocks whose amax is 448):
  subnormals, round-to-nearest-even ties, signed zero, values under half the smallest subnormal;
* all-zero tiles and blocks (scale 1e-12 / 448, bytes 0), amax under 1e-12, amax near the fp32 maximum;
* random blocks at the Qwen3-30B-A3B expert shapes and at non-square block grids, one and three matrices, fp32 and
  bf16 weights;
* NaN and inf: the scale follows torch's amax (a NaN makes its whole tile or block NaN, an inf gives an inf scale,
  0 for the finite elements and NaN for the inf one), the other tiles and blocks stay as they are;
* more than 2^31 elements for the tile path and for a bf16 block tensor;
* ``plugin.install_fp8_cast()`` against the reference's own ``cast_to_per_block_fp8_with_scales`` and
  ``tensor_to_per_block_fp8_scales`` on CUDA tensors (where ``oracle/_ref`` holds the reference package).

Scales are compared with ``torch.equal``, bytes as uint8; NaN is matched as NaN (the sign of a NaN byte is not
pinned)."""
import importlib
import os

import pytest
import torch

from oracle import moe_oracle as O
from tests import swiglu_fp8_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "xtuner", "v1"))


def _lib():
    from xtuner_b200 import _capi

    return _capi.ensure_init()


def _ok(rc, what):
    from xtuner_b200._capi import check

    check(rc, what)


def _st():
    from xtuner_b200._capi import current_stream

    return current_stream()


def tile_quant(x):
    M, K = x.shape
    q = torch.empty(M, K, dtype=torch.uint8, device="cuda")
    s = torch.empty(M, K // 128, dtype=torch.float32, device="cuda")
    _ok(_lib().xtb_fp8_per_tile_quant(x.data_ptr(), q.data_ptr(), s.data_ptr(), M, K, _st()), "xtb_fp8_per_tile_quant")
    return q, s


def block_scales(w):
    nw, dout, din = w.shape
    s = torch.empty(nw, dout // 128, din // 128, dtype=torch.float32, device="cuda")
    _ok(_lib().xtb_fp8_block_scales(w.data_ptr(), int(w.dtype == torch.float32), nw, dout, din, s.data_ptr(), _st()),
        "xtb_fp8_block_scales")
    return s


def block_cast(w, s):
    nw, dout, din = w.shape
    q = torch.empty(nw, dout, din, dtype=torch.uint8, device="cuda")
    _ok(_lib().xtb_fp8_block_cast(w.data_ptr(), int(w.dtype == torch.float32), nw, dout, din, s.data_ptr(),
                                  q.data_ptr(), _st()), "xtb_fp8_block_cast")
    return q


def _check_blocks(w, what):
    """Kernels on w [nw, dout, din] (cuda) against the float64 model and the oracle (cpu)."""
    s = block_scales(w)
    q = block_cast(w, s)
    torch.cuda.synchronize()
    wc = w.cpu()
    want_s = R.block_scales(wc)
    R.assert_scales_equal(s.cpu(), want_s, f"{what} scales")
    R.assert_scales_equal(s.cpu(), O.per_block_fp8_scales(wc), f"{what} scales vs oracle")
    for i in range(w.shape[0]):
        R.assert_fp8_equal(q[i].cpu(), R.block_cast(wc[i], want_s[i]), f"{what} cast [{i}]")
        R.assert_fp8_equal(q[i].cpu(), O.cast_to_per_block_fp8(wc[i], want_s[i]), f"{what} cast [{i}] vs oracle")
    return s.cpu(), q.cpu()


def test_e4m3_cast_of_every_bf16_in_range():
    t = R.amax_one_tiles(R.cast_sweep_values())  # [n, 128], amax 448 per row
    q, s = tile_quant(t.cuda())
    torch.cuda.synchronize()
    assert bool((s == 1).all())
    want = R.e4m3_bits(t.double())
    R.assert_fp8_equal(q.cpu(), want, "tile cast of every bf16 in [-448, 448]")
    assert torch.equal(q.cpu(), O.per_tile_quant(t)[0].view(torch.uint8))
    # the same values through the block path: rows of a 128-row block, with (0, 0) = 448 in every block
    n = t.shape[0]
    rows = -(-n // 128) * 128
    body = torch.full((rows, 128), R.E4M3_MAX, dtype=torch.bfloat16)
    body[:n] = t
    body[::128, 0] = R.E4M3_MAX
    for dtype in (torch.bfloat16, torch.float32):
        w = body.to(dtype).view(1, rows, 128)
        s, q = _check_blocks(w.cuda(), f"block cast of every bf16 in [-448, 448], {dtype}")
        assert bool((s == 1).all())
        R.assert_fp8_equal(q[0, :n], want, f"block cast equals tile cast, {dtype}")


def test_zero_tiny_and_huge_scales():
    eps_scale = torch.tensor(1e-12 / 448, dtype=torch.float64).float()
    x = torch.randn(6, 512).to(torch.bfloat16)
    x[0] = 0
    x[1, :128] = -0.0
    x[2, 128:256] *= 1e-14  # amax under 1e-12: scale 1e-12 / 448, bytes from that scale
    x[3, 256:384] = torch.tensor(1e-30).to(torch.bfloat16)
    q, s = tile_quant(x.cuda())
    torch.cuda.synchronize()
    rq, rs = O.per_tile_quant(x)
    R.assert_scales_equal(s.cpu(), rs, "tile scales")
    R.assert_fp8_equal(q.cpu(), rq, "tile bytes")
    assert bool((s[0].cpu() == eps_scale).all()) and bool((q[0] == 0).all())
    assert s[1, 0].item() == eps_scale.item() and bool(((q[1, :128] & 0x7F) == 0).all())
    for dtype in (torch.float32, torch.bfloat16):
        w = (torch.randn(2, 256, 384) * 2).to(dtype)
        w[0, :128, :128] = 0
        w[0, 128:, :128] *= 1e-14
        w[1, :128, 256:] = torch.tensor(1e-30).to(dtype)
        if dtype == torch.float32:
            w[1, 128:, :128] *= 3.4e38 / 8  # amax near the fp32 maximum
            w[1, 200, 100] = torch.finfo(torch.float32).max
        s, q = _check_blocks(w.cuda(), f"zero / tiny / huge blocks, {dtype}")
        assert s[0, 0, 0].item() == eps_scale.item() and bool((q[0, :128, :128] == 0).all())


@pytest.mark.parametrize("nw", [1, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("dout,din", [(1536, 2048), (2048, 768), (128, 384), (640, 256)])
def test_random_blocks(nw, dtype, dout, din):
    gen = torch.Generator().manual_seed(dout * 31 + din + nw)
    w = (torch.randn(nw, dout, din, generator=gen) * torch.pow(4.0, torch.randint(-6, 7, (nw, 1, 1), generator=gen))
         ).to(dtype)
    _check_blocks(w.cuda(), f"random [{nw}, {dout}, {din}] {dtype}")


def _nan_bytes(q):
    return (q.int() & 0x7F) == 0x7F


def test_nan_and_inf_follow_the_reference_amax():
    """A NaN makes its block's (tile's) scale and bytes NaN and leaves the others alone; an inf gives an inf scale,
    0 for the finite elements and NaN for the inf one.  Before the NaN-keeping amax, the kernels dropped the NaN
    (finite scale, byte 0xFE = -448 for the NaN)."""
    for dtype in (torch.float32, torch.bfloat16):
        w = (torch.randn(2, 256, 384) * 2).to(dtype)
        w[0, 5, 300] = float("nan")
        w[1, 130, 7] = float("inf")
        w[1, 131, 8] = -3.0
        s, q = _check_blocks(w.cuda(), f"NaN / inf blocks, {dtype}")
        assert torch.isnan(s[0, 0, 2]) and int(torch.isnan(s).sum()) == 1, s
        assert bool(_nan_bytes(q[0, :128, 256:]).all())
        assert not bool(_nan_bytes(q[0, 128:]).any()) and not bool(_nan_bytes(q[0, :128, :256]).any())
        assert torch.isinf(s[1, 1, 0]) and int(torch.isinf(s).sum()) == 1
        assert bool(_nan_bytes(q[1, 130, 7:8]).all()) and int(q[1, 131, 8]) == 0x80
        blk = q[1, 128:, :128].clone()
        blk[2, 7] = 0
        assert bool(((blk.int() & 0x7F) == 0).all())
    x = torch.randn(4, 512).to(torch.bfloat16)
    x[1, 200] = float("nan")
    x[2, 10] = -float("inf")
    q, s = tile_quant(x.cuda())
    torch.cuda.synchronize()
    rq, rs = O.per_tile_quant(x)
    R.assert_scales_equal(s.cpu(), rs, "NaN / inf tiles")
    R.assert_fp8_equal(q.cpu(), rq, "NaN / inf tiles")
    q = q.cpu()
    assert torch.isnan(s[1, 1]) and bool(_nan_bytes(q[1, 128:256]).all()) and not bool(_nan_bytes(q[1, :128]).any())
    assert torch.isinf(s[2, 0]) and bool(_nan_bytes(q[2, 10:11]).all()) and int(_nan_bytes(q[2]).sum()) == 1


def test_past_2_31_elements():
    M, K = 2 ** 20 + 8, 2048
    gen = torch.Generator("cuda").manual_seed(23)
    x = torch.randn(M, K, generator=gen, device="cuda", dtype=torch.bfloat16)
    x[-1, -128:] = float("nan")
    q, s = tile_quant(x)
    torch.cuda.synchronize()
    for rows in (slice(0, 4), slice(M - 4, M)):
        rq, rs = O.per_tile_quant(x[rows].cpu())
        R.assert_scales_equal(s[rows].cpu(), rs, f"tile scales rows {rows}")
        R.assert_fp8_equal(q[rows].cpu(), rq, f"tile bytes rows {rows}")
    assert torch.isnan(s[-1, -1])
    del x, q, s
    nw, dout, din = 1366, 2048, 768  # 2^31 + 2 Mi elements
    assert nw * dout * din > 2 ** 31
    w = torch.randn(nw, dout, din, generator=gen, device="cuda", dtype=torch.bfloat16)
    w[-1, -1, -1] = float("inf")
    s = block_scales(w)
    q = block_cast(w, s)
    torch.cuda.synchronize()
    for i in (0, nw - 1):
        wi = w[i : i + 1].cpu()
        want_s = O.per_block_fp8_scales(wi)
        R.assert_scales_equal(s[i : i + 1].cpu(), want_s, f"block scales [{i}]")
        R.assert_fp8_equal(q[i].cpu(), O.cast_to_per_block_fp8(wi[0], want_s[0]), f"block bytes [{i}]")
    assert torch.isinf(s[-1, -1, -1])


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref absent (oracle/make_ref.py places the reference package there)")
def test_install_fp8_cast_on_the_reference_functions():
    from tests.golden import ref_shim
    from xtuner_b200 import plugin

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    ref_shim.import_reference()
    fu = importlib.import_module("xtuner.v1.float8.fsdp_utils")
    ref_cast, ref_scales = fu.cast_to_per_block_fp8_with_scales, fu.tensor_to_per_block_fp8_scales
    cases = []
    for dtype in (torch.float32, torch.bfloat16):
        w = (torch.randn(3, 256, 384) * 2).to(dtype)
        w[0, :128, :128] = 0
        w[1, 5, 300] = float("nan")
        w[2, 130, 7] = float("inf")
        w[2, 200, 200] = -float("inf")
        cases.append(w.cuda())
    want = []
    for w in cases:
        s = ref_scales(w)
        want.append((s, [ref_cast(w[i], s[i]) for i in range(w.shape[0])]))
    _lib()
    plugin.install_fp8_cast()
    try:
        assert fu.cast_to_per_block_fp8_with_scales is not ref_cast
        for w, (want_s, want_q) in zip(cases, want):
            got_s = fu.tensor_to_per_block_fp8_scales(w)
            R.assert_scales_equal(got_s, want_s, f"scales {w.dtype}")
            for i in range(w.shape[0]):
                got = fu.cast_to_per_block_fp8_with_scales(w[i], want_s[i])
                assert got.dtype == torch.float8_e4m3fn
                R.assert_fp8_equal(got.view(torch.uint8), want_q[i].view(torch.uint8), f"cast {w.dtype} [{i}]")
        assert torch.isnan(want[0][0][1, 0, 2]) and torch.isinf(want[0][0][2, 1, 0])
    finally:
        plugin.uninstall_fp8_cast()
    assert fu.cast_to_per_block_fp8_with_scales is ref_cast
