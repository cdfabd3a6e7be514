"""``xtb_swiglu`` and ``xtb_swiglu_bwd`` (``csrc/permute.cu``) on an H100 against the float64 references and exact
restatements of ``tests/swiglu_fp8_reference.py``:

* every one of the 65,536 bf16 gate values (±0, subnormals, ±inf, NaNs, the band g = -87.3 .. -88.7 where
  1 + exp(-g) nears the fp32 maximum and its reciprocal goes subnormal, and beyond, where it overflows and the
  sigmoid is 0 as in the reference's fp32 silu) with
  u in {1, -1, 3, 2^-100, the largest bf16, 0, NaN}: with u = 1 the output is the kernel's s itself, checked against
  the float64 silu; every other u must then give bf16(s u) bit for bit;
* widths I = 8 (one vector per row, the special-cased row split), non-power-of-two I / 8 (the reciprocal row split)
  up to the widest row the host accepts, and row counts that are not a multiple of the backward's 8-row block, with
  every output inside NaN guard rows;
* the backward launched right behind the grouped GEMM that produces its input, as the fused layer runs it;
* more than 2^31 elements, repeat runs, CUDA-graph replay and the torch custom-op checks."""
import pytest
import torch

from tests import swiglu_fp8_reference as R
from tests.gpu_harness import Guarded
from xtuner_b200._capi import check, current_stream, ensure_init

pytestmark = pytest.mark.gpu


def fwd(h, out):
    M, twoI = h.shape
    check(ensure_init().xtb_swiglu(h.data_ptr(), out.data_ptr(), M, twoI // 2, current_stream()), "xtb_swiglu")


def bwd(d, h, gh):
    M, twoI = h.shape
    check(ensure_init().xtb_swiglu_bwd(d.data_ptr(), h.data_ptr(), gh.data_ptr(), M, twoI // 2, current_stream()),
          "xtb_swiglu_bwd")


def _run(h, d):
    M, twoI = h.shape
    a, gh = Guarded(M, twoI // 2, torch.bfloat16), Guarded(M, twoI, torch.bfloat16)
    fwd(h, a.v)
    bwd(d, h, gh.v)
    torch.cuda.synchronize()
    return a.check("swiglu"), gh.check("swiglu_bwd")


def test_swiglu_every_bf16_gate_value():
    g = R.all_bf16().cuda()
    u = torch.tensor(R.SWEEP_U, dtype=torch.float64).to(torch.bfloat16).cuda()
    n_u = u.numel()
    h = torch.cat([g.expand(n_u, -1), u[:, None].expand(-1, g.numel())], 1).contiguous()
    d = (torch.rand(n_u, g.numel(), generator=torch.Generator("cuda").manual_seed(7), device="cuda") * 2 - 1).to(
        torch.bfloat16)
    a, gh = _run(h, d)
    # u = 1: a is s itself
    s = a[0]
    ref, bound = R.silu_ref(g)
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isnan(s), torch.isnan(ref)), "silu NaN positions"
    ratio, ties = R.check_near_tie(s[fin], ref[fin], bound[fin], "silu over every bf16")
    inf = torch.isinf(ref)
    assert torch.equal(s[inf].double(), ref[inf]), "silu(+inf)"
    band = fin & (g.double() <= -87.0) & (g.double() >= -104.0)
    r_band, t_band = R.check_near_tie(s[band], ref[band], bound[band], "silu, g in [-104, -87]")
    # every u: a = bf16(s u) exactly, with the kernel's own s
    R.assert_bits_equal_nan(a, R.swiglu_a(s.expand(n_u, -1), h[:, g.numel():]), "a = bf16(s u)")
    fwd_ties = R.check_swiglu_fwd(h, a, "swiglu over every bf16")
    # backward: grad_u = bf16(d s) with the same s, grad_g against float64
    R.assert_bits_equal_nan(gh[:, g.numel():], R._mul_bf16(d, s.expand(n_u, -1)), "grad_u = bf16(d s)")
    s_ties, g_ratio, g_ties = R.check_swiglu_bwd(h, d, gh, "swiglu_bwd over every bf16")
    print(f"\nsilu over 65536 g: {ties} near ties of s, worst |err|/bound {ratio:.3g}; g in [-104, -87]: {t_band} near "
          f"ties, worst {r_band:.3g}; a over {a.numel()}: {fwd_ties} candidate pairs; grad_g over {gh.numel() // 2}: "
          f"{g_ties} near ties, worst |err|/bound {g_ratio:.3g}")


SHAPES = [(M, I) for I in (8, 24, 776, 768, 1536) for M in (1, 7, 9, 8 * 37 + 3, 16384)] + [
    (M, 185360) for M in (1, 7, 9, 8 * 2 + 3)]


@pytest.mark.parametrize("M,I", SHAPES)
def test_swiglu_shapes_in_guard_bands(M, I):
    gen = torch.Generator("cuda").manual_seed(M * 7919 + I)
    scale = torch.pow(4.0, torch.randint(-3, 4, (M, 1), generator=gen, device="cuda").double())
    g = torch.randn(M, I, generator=gen, device="cuda", dtype=torch.float64) * scale
    u = torch.randn(M, I, generator=gen, device="cuda", dtype=torch.float64) * 2
    h = torch.cat([g, u], 1).to(torch.bfloat16)
    d = torch.randn(M, I, generator=gen, device="cuda").to(torch.bfloat16)
    a, gh = _run(h, d)
    R.check_swiglu_fwd(h, a, f"swiglu M={M} I={I}")
    R.check_swiglu_bwd(h, d, gh, f"swiglu_bwd M={M} I={I}")


def test_swiglu_bwd_right_behind_the_grouped_gemm():
    """g_a from xtb_group_gemm_nn with xtb_swiglu_bwd launched straight after it on the same stream (fused.py), as a
    programmatic dependent launch: the result equals the same backward on a synchronised copy of g_a."""
    lib = ensure_init()
    gen = torch.Generator("cuda").manual_seed(11)
    E, H = 8, 512
    for I in (768, 1536):
        tpe = torch.tensor([1000, 0, 37, 2048, 501, 129, 3, 378], dtype=torch.int64, device="cuda")
        M = int(tpe.sum())
        g_y = (torch.randn(M, H, generator=gen, device="cuda") * 0.5).to(torch.bfloat16)
        w2 = (torch.randn(E, H, I, generator=gen, device="cuda") * H ** -0.5).to(torch.bfloat16)
        h = (torch.randn(M, 2 * I, generator=gen, device="cuda") * 2).to(torch.bfloat16)
        g_a = torch.empty(M, I, dtype=torch.bfloat16, device="cuda")
        g_h = torch.empty(M, 2 * I, dtype=torch.bfloat16, device="cuda")
        st = current_stream()
        check(lib.xtb_group_gemm_nn(g_y.data_ptr(), w2.data_ptr(), tpe.data_ptr(), M, H, I, E, g_a.data_ptr(), st),
              "xtb_group_gemm_nn")
        check(lib.xtb_swiglu_bwd(g_a.data_ptr(), h.data_ptr(), g_h.data_ptr(), M, I, st), "xtb_swiglu_bwd")
        torch.cuda.synchronize()
        g_a2 = g_a.clone()
        torch.cuda.synchronize()
        g_h2 = torch.empty_like(g_h)
        bwd(g_a2, h, g_h2)
        torch.cuda.synchronize()
        assert torch.equal(g_h.view(torch.int16), g_h2.view(torch.int16)), f"I={I}: backward behind the GEMM differs"
        R.check_swiglu_bwd(h, g_a2, g_h, f"swiglu_bwd behind the GEMM, I={I}")


def test_swiglu_past_2_31_elements():
    M, I = 131073, 8192  # h holds M * 2I = 2^31 + 16384 elements
    assert M * 2 * I > 2 ** 31
    gen = torch.Generator("cuda").manual_seed(13)
    h = torch.randn(M, 2 * I, generator=gen, device="cuda", dtype=torch.bfloat16)
    d = torch.randn(M, I, generator=gen, device="cuda", dtype=torch.bfloat16)
    a = torch.empty(M, I, dtype=torch.bfloat16, device="cuda")
    fwd(h, a)
    gh = torch.empty(M, 2 * I, dtype=torch.bfloat16, device="cuda")
    bwd(d, h, gh)
    torch.cuda.synchronize()
    for rows in (slice(0, 8), slice(M - 9, M)):
        R.check_swiglu_fwd(h[rows], a[rows], f"swiglu rows {rows}")
        R.check_swiglu_bwd(h[rows], d[rows], gh[rows], f"swiglu_bwd rows {rows}")


def test_swiglu_repeat_graph_and_opcheck():
    from xtuner_b200 import ops

    gen = torch.Generator("cuda").manual_seed(17)
    M, I = 4099, 1536
    h = (torch.randn(M, 2 * I, generator=gen, device="cuda") * 3).to(torch.bfloat16)
    d = torch.randn(M, I, generator=gen, device="cuda").to(torch.bfloat16)
    a1, a2 = ops._swiglu_op(h), ops._swiglu_op(h)
    g1, g2 = ops._swiglu_bwd_op(d, h), ops._swiglu_bwd_op(d, h)
    torch.cuda.synchronize()
    assert torch.equal(a1.view(torch.int16), a2.view(torch.int16)) and torch.equal(g1.view(torch.int16), g2.view(torch.int16))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside the capture
        ops._swiglu_op(h), ops._swiglu_bwd_op(d, h)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ag = ops._swiglu_op(h)
        gg = ops._swiglu_bwd_op(d, h)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(ag.view(torch.int16), a1.view(torch.int16)), "graph replay of xtb_swiglu differs"
    assert torch.equal(gg.view(torch.int16), g1.view(torch.int16)), "graph replay of xtb_swiglu_bwd differs"
    torch.library.opcheck(ops._swiglu_op, (h[:64].contiguous(),))
    torch.library.opcheck(ops._swiglu_bwd_op, (d[:64].contiguous(), h[:64].contiguous()))
