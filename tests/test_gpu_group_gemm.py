"""GPU parity of the wgmma grouped GEMMs (forward NT, dX NN, dW TN) against the oracle's per-expert
loop (tests/ops/test_grouped_gemm_triton.py:6-23 semantics) — small ragged cases on the CPU oracle, full
config sizes against a per-expert cuBLAS loop on the same GPU (fp32-accumulate yardstick).
Tolerance: the reference's own (rtol=atol=1e-2, tests/ops/test_grouped_gemm_triton.py:62-64) or tighter."""
import pytest
import torch

from oracle import moe_oracle as O

pytestmark = pytest.mark.gpu


def _ragged_counts(E, total, seed, empty=()):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(E, generator=g) + 0.05
    for e in empty:
        w[e] = 0
    c = torch.floor(w / w.sum() * total).long()
    c[int(torch.argmax(w))] += total - int(c.sum())
    assert int(c.sum()) == total and (c >= 0).all()
    return c


def _loop(x, w, counts):
    outs, s = [], 0
    for i, n in enumerate(counts.tolist()):
        outs.append(x[s : s + n] @ w[i].T)
        s += n
    return torch.cat(outs)


@pytest.mark.parametrize(
    "E,M,N,Kd,empty",
    [(4, 300, 128, 128, ()), (8, 1000, 256, 128, (2,)), (8, 77, 128, 256, (0, 7)), (3, 129, 384, 192 + 64, ()), (1, 128, 128, 128, ()),
     # shapes that take the 256-column tiles
     (4, 700, 256, 256, ()), (8, 1000, 512, 256, (2,)), (3, 100, 256, 512, (1,)), (2, 513, 768, 256, ())],
)
def test_group_gemm_small_vs_cpu_oracle(E, M, N, Kd, empty):
    from xtuner_b200 import ops

    g = torch.Generator().manual_seed(M + N)
    counts = _ragged_counts(E, M, M, empty)
    x = torch.randn(M, Kd, generator=g).to(torch.bfloat16)
    w = (torch.randn(E, N, Kd, generator=g) * Kd**-0.5).to(torch.bfloat16)
    dy = torch.randn(M, N, generator=g).to(torch.bfloat16)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ref = O.group_gemm_fp32acc(xr, wr, counts)
    # autograd of the oracle runs in bf16 matmuls; build fp32 references for the grads explicitly
    dx_ref = torch.cat([dy[s:e].float() @ w[i].float() for i, (s, e) in enumerate(zip((counts.cumsum(0) - counts).tolist(), counts.cumsum(0).tolist()))]).to(torch.bfloat16)
    dw_ref = torch.stack([dy[s:e].float().T @ x[s:e].float() for s, e in zip((counts.cumsum(0) - counts).tolist(), counts.cumsum(0).tolist())]).to(torch.bfloat16)

    xd, wd = x.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    out = ops.group_gemm(xd, wd, counts.cuda())
    torch.testing.assert_close(out.float().cpu(), ref.detach().float(), rtol=1e-2, atol=1e-2)
    dx, dw = torch.autograd.grad(out, (xd, wd), dy.cuda())
    torch.testing.assert_close(dx.float().cpu(), dx_ref.float(), rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(dw.float().cpu(), dw_ref.float(), rtol=1e-2, atol=2e-2)
    for e in empty:
        assert (dw[e] == 0).all(), "empty expert must get a zero dW"


@pytest.mark.parametrize("N,Kd", [(1536, 2048), (2048, 768)])
@pytest.mark.parametrize("skew", [False, True])
def test_group_gemm_config2_vs_cublas_loop(N, Kd, skew):
    """Config 2 sizes (T*K = 16384 rows, 8 experts; SURVEY.md §8) — balanced and Zipf-skewed loads."""
    from xtuner_b200 import ops

    E, M = 8, 16384
    g = torch.Generator().manual_seed(N + skew)
    if skew:
        wgt = 1.0 / torch.arange(1, E + 1).float()
        counts = torch.floor(wgt / wgt.sum() * M).long()
        counts[0] += M - int(counts.sum())
    else:
        counts = _ragged_counts(E, M, 11)
    x = torch.randn(M, Kd, generator=g).to(torch.bfloat16).cuda().requires_grad_(True)
    w = (torch.randn(E, N, Kd, generator=g) * Kd**-0.5).to(torch.bfloat16).cuda().requires_grad_(True)
    dy = torch.randn(M, N, generator=g).to(torch.bfloat16).cuda()
    out = ops.group_gemm(x, w, counts.cuda())
    dx, dw = torch.autograd.grad(out, (x, w), dy)
    xr, wr = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True)
    ref = _loop(xr, wr, counts)
    dxr, dwr = torch.autograd.grad(ref, (xr, wr), dy)
    torch.testing.assert_close(out.float(), ref.float(), rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(dx.float(), dxr.float(), rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(dw.float(), dwr.float(), rtol=1e-2, atol=5e-2)
    # linearity property (size independent): gemm(2x) == 2*gemm(x) exactly in bf16
    out2 = ops.group_gemm((x.detach() * 2), w.detach(), counts.cuda())
    assert torch.equal(out2, out.detach() * 2)


def test_group_gemm_zero_rows_joins_graph():
    from xtuner_b200 import ops

    x = torch.empty(0, 256, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    w = torch.randn(4, 128, 256, device="cuda").to(torch.bfloat16).requires_grad_(True)
    out = ops.group_gemm(x, w, torch.zeros(4, dtype=torch.int64, device="cuda"))
    assert out.shape == (0, 128)
    out.sum().backward()
    assert w.grad is not None


@pytest.mark.parametrize("dims", [(256, 512, 512, 256), (128, 256, 384, 128)])
def test_tn_pair_with_empty_experts_and_fallback_shapes(dims):
    """xtb_group_gemm_tn_pair == two xtb_group_gemm_tn calls: experts without rows get zero matrices from the pair kernel
    too, and shapes that are not multiples of 256 take the two separate launches inside the entry."""
    from xtuner_b200 import _capi
    from xtuner_b200._capi import check, current_stream, ptr

    lib = _capi.ensure_init()
    st = current_stream()
    Na, Ka, Nb, Kb = dims
    counts = [0, 300, 0, 212, 77]
    E, M = len(counts), sum(counts)
    g = torch.Generator().manual_seed(Na + Kb)
    tpe = torch.tensor(counts, dtype=torch.int64).cuda()
    mk = lambda r, c: torch.randn(r, c, generator=g).to(torch.bfloat16).cuda()  # noqa: E731
    dya, xa, dyb, xb = mk(M, Na), mk(M, Ka), mk(M, Nb), mk(M, Kb)
    ref_a = torch.empty(E, Na, Ka, dtype=torch.bfloat16, device="cuda")
    ref_b = torch.empty(E, Nb, Kb, dtype=torch.bfloat16, device="cuda")
    check(lib.xtb_group_gemm_tn(ptr(dya), ptr(xa), ptr(tpe), M, Na, Ka, E, ptr(ref_a), st), "tn a")
    check(lib.xtb_group_gemm_tn(ptr(dyb), ptr(xb), ptr(tpe), M, Nb, Kb, E, ptr(ref_b), st), "tn b")
    out_a = torch.full_like(ref_a, float("nan"))
    out_b = torch.full_like(ref_b, float("nan"))
    check(lib.xtb_group_gemm_tn_pair(ptr(dya), ptr(xa), Na, Ka, ptr(out_a), ptr(dyb), ptr(xb), Nb, Kb, ptr(out_b), ptr(tpe), M, E, st),
          "tn pair")
    torch.cuda.synchronize()
    assert torch.equal(out_a, ref_a) and torch.equal(out_b, ref_b)
    assert not out_a[0].any() and not out_b[2].any()  # empty experts: zero gradients
    s = 300
    want = (dya[:s].float().t() @ xa[:s].float())
    torch.testing.assert_close(out_a[1].float(), want, rtol=2e-2, atol=2e-1)
