"""xtb_lm_head_ce on an H100, each layer against its own reference:

* logits: the EPI_CE instantiation of the NT GEMM with exact-mode integer inputs (``tests/gemm_reference.py``) equals
  bf16(fp64) bit for bit, and rows outside the buffer stay untouched;
* loss and G from the kernel's own logits against float64 formulas;
* dh and dW from the kernel's own G against the scale-aware bound of ``tests/gemm_reference.py``;
* ``ops.lm_head_cross_entropy`` end to end against the reference's arithmetic on the GPU (``tests/lm_head_ce_reference.py``)
  at the Qwen3-MoE head shape, in eager and chunk mode;
* 64-bit addressing (T * V > 2^31), all rows ignored, run-to-run determinism, CUDA-graph capture, and the plugin on the
  reference's own ``LMHead``."""
import os

import pytest
import torch

from tests import gemm_reference as R
from tests.lm_head_ce_reference import grad64, lm_head_ce, row_ce64

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "xtuner", "v1"))
DEV = "cuda"
IGN = -100


def _raw(h, w, labels, lw, need_grad, z, ignore=IGN):
    """one xtb_lm_head_ce call -> (row_ce, loss, dh, dw); z receives z (need_grad=0) or G"""
    from xtuner_b200 import _capi

    lib = _capi.ensure_init()
    T, H = h.shape
    V = w.shape[0]
    ws = torch.empty(max(int(lib.xtb_lm_head_ce_workspace_bytes(T, V)), 16), dtype=torch.uint8, device=DEV)
    row_ce = torch.empty(T, dtype=torch.float32, device=DEV)
    loss = torch.empty((), dtype=torch.float32, device=DEV)
    dh = torch.empty_like(h) if need_grad else None
    dw = torch.empty_like(w) if need_grad else None
    p = _capi.ptr
    _capi.check(lib.xtb_lm_head_ce(p(h), p(w), p(labels), p(lw), T, H, V, ignore, int(need_grad), p(z), p(ws), p(row_ce),
                                   p(loss), p(dh), p(dw), _capi.current_stream()), "xtb_lm_head_ce")
    return row_ce, loss, dh, dw


def _labels(T, V, seed, ignored=0.3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lab = torch.randint(0, V, (T,), generator=g, device=DEV)
    lab[torch.rand(T, generator=g, device=DEV) < ignored] = IGN
    if T > 3:
        lab[1], lab[2] = 0, V - 1
    return lab


def _random(T, H, V, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h = (torch.randn(T, H, generator=g, device=DEV) * scale).to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device=DEV) * H ** -0.5).to(torch.bfloat16)
    return h, w


# 256-column tiles; 128-column tiles (V % 256 == 128); one tile of each width
@pytest.mark.parametrize("V", [512, 384, 1152, 128, 256])
# 16-row store boxes: full, and ragged in their first or second 8-row half; 128-row tiles: one short, full, one over
@pytest.mark.parametrize("T", [1, 100, 128, 1000, 8, 9, 16, 17, 63, 64, 65, 127, 129])
def test_logits_are_exact_and_stay_inside_the_buffer(T, V):
    H = 256
    h = R.rows_operand([T], H, "exact", seed=T, device=DEV)
    w = R.weight_operand(1, V, H, "exact", seed=V, device=DEV)
    buf = torch.full((T + 32, V), float("nan"), dtype=torch.bfloat16, device=DEV)
    z = buf[16:16 + T]
    lw = torch.ones(T, device=DEV)
    _raw(h, w[0], _labels(T, V, 1), lw, False, z)
    R.assert_exact(z, "nt", h, w, [T], what=f"lm_head logits T={T} V={V}")
    assert torch.isnan(buf[:16]).all() and torch.isnan(buf[16 + T:]).all(), "write outside the logits buffer"


def _loss_and_grad(h, w, lab, lw):
    T, V = h.shape[0], w.shape[0]
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    ce0, loss0, _, _ = _raw(h, w, lab, lw, False, z)
    zk = z.clone()
    ce, loss, dh, dw = _raw(h, w, lab, lw, True, z)
    assert torch.equal(ce, ce0) and (torch.equal(loss, loss0) or (loss.isnan() and loss0.isnan()))
    return zk, z, ce, loss, dh, dw


@pytest.mark.parametrize("V,scale", [(1152, 1.0), (2048, 1.0), (1152, 2500.0)])  # 2500: logits of magnitude ~1e4
def test_loss_and_grad_from_the_kernels_logits(V, scale):
    T, H = 1000, 256
    h, w = _random(T, H, V, seed=V, scale=scale)
    lab = _labels(T, V, seed=7)
    lw = torch.rand(T, device=DEV) + 0.5
    zk, G, ce, loss, dh, dw = _loss_and_grad(h, w, lab, lw)
    if scale > 1:
        assert zk.float().abs().max() > 5e3
    ign = lab == IGN
    ce64 = row_ce64(zk, lab, IGN)
    assert torch.isfinite(ce).all() and (ce[ign] == 0).all()
    # relative to the row's CE, floored at 1 for the rows a large-logit input makes almost certain (CE ~ 0)
    rel = ((ce.double() - ce64).abs() / ce64.abs().clamp_min(1.0 if scale > 1 else 0.0))[~ign]
    print(f"V={V} scale={scale}: max rel CE error {rel.max().item():.2e}")
    assert rel.max() <= 1e-6
    want = (ce64 * lw.double()).sum()
    assert abs(loss.item() - want.item()) <= 1e-6 * abs(want.item())
    g64 = R.bf16_rn(grad64(zk, lab, lw, IGN))
    assert (G[ign] == 0).all() and torch.isfinite(G.float()).all()
    d = R.ulp_distance(G, g64)
    print(f"V={V} scale={scale}: G max ulp {d.max().item()}, exact share {(d == 0).double().mean().item():.6f}")
    assert d.max() <= 1 and (d == 0).double().mean() >= 0.999
    # dh and dW are the NN / TN products of the kernel's own G
    r1 = R.check_bound(dh, "nn", G, w[None], [T], what="dh")
    r2 = R.check_bound(dw[None], "tn", G, h, [T], what="dW")
    print(f"dh worst |err|/bound {r1:.3f}, dW {r2:.3f}")


def test_label_out_of_range_gives_nan_for_that_row_only():
    T, H, V = 300, 256, 1024
    h, w = _random(T, H, V, seed=3)
    lab = _labels(T, V, seed=3)
    lab[10], lab[11] = V, 12  # row 10: label V (invalid, not ignored)
    lw = torch.ones(T, device=DEV)
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    ce, loss, dh, dw = _raw(h, w, lab, lw, True, z)
    torch.cuda.synchronize()
    assert torch.isnan(ce[10]) and torch.isfinite(torch.cat([ce[:10], ce[11:]])).all() and torch.isnan(loss)
    assert torch.isnan(z[10].float()).all() and torch.isfinite(torch.cat([z[:10], z[11:]]).float()).all()


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()


@pytest.mark.parametrize("T,chunk", [(8192, None), (3000, 1024)])
def test_end_to_end_against_the_reference_at_the_qwen3_head(T, chunk):
    from xtuner_b200 import ops

    H, V = 2048, 151936
    h, w = _random(T, H, V, seed=11)
    lab = _labels(T, V, seed=11)
    lw = (lab != IGN).float() / (lab != IGN).sum()
    want = lm_head_ce(h, w, lab, lw, IGN, chunk)
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    loss = ops.lm_head_cross_entropy(hh, ww, lab, lw, IGN, chunk)
    loss.backward()
    rl = abs(loss.item() - want[0].item()) / abs(want[0].item())
    e_dh, e_dw = _rel(hh.grad, want[1]), _rel(ww.grad, want[2])
    print(f"T={T} chunk={chunk}: loss rel {rl:.2e}; max|err|/max|ref| dh {e_dh:.2e} dW {e_dw:.2e}")
    assert rl <= 1e-5
    torch.testing.assert_close(hh.grad.float(), want[1].float(), rtol=2 ** -7, atol=2 ** -7 * want[1].float().abs().max().item())
    torch.testing.assert_close(ww.grad.float(), want[2].float(), rtol=2 ** -7, atol=2 ** -7 * want[2].float().abs().max().item())


def test_64bit_addressing_matches_two_halves():
    T, H, V = 16384, 256, 151936  # T * V = 2.49e9 elements > 2^31
    h, w = _random(T, H, V, seed=5)
    lab = _labels(T, V, seed=5)
    lw = torch.full((T,), 1.0 / T, device=DEV)
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    ce, loss, dh, dw = _raw(h, w, lab, lw, True, z)
    del z
    parts = []
    for s in (0, T // 2):
        zh = torch.empty((T // 2, V), dtype=torch.bfloat16, device=DEV)
        parts.append(_raw(h[s:s + T // 2], w, lab[s:s + T // 2], lw[s:s + T // 2], True, zh))
        del zh
    assert torch.equal(ce, torch.cat([parts[0][0], parts[1][0]]))
    assert torch.equal(dh, torch.cat([parts[0][2], parts[1][2]]))
    assert abs(loss.item() - (parts[0][1] + parts[1][1]).item()) <= 1e-6 * abs(loss.item())
    torch.testing.assert_close(dw.float(), (parts[0][3].float() + parts[1][3].float()), rtol=2 ** -7,
                               atol=2 ** -7 * dw.float().abs().max().item())


def test_all_rows_ignored_gives_exact_zeros():
    T, H, V = 500, 256, 1024
    h, w = _random(T, H, V, seed=9)
    lab = torch.full((T,), IGN, device=DEV)
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    ce, loss, dh, dw = _raw(h, w, lab, torch.zeros(T, device=DEV), True, z)
    assert loss.item() == 0.0 and (ce == 0).all() and (z == 0).all() and (dh == 0).all() and (dw == 0).all()


def test_two_calls_give_identical_bits():
    T, H, V = 4096, 1024, 32768
    h, w = _random(T, H, V, seed=13)
    lab = _labels(T, V, seed=13)
    lw = torch.rand(T, device=DEV)
    outs = []
    for _ in range(2):
        z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
        outs.append(_raw(h, w, lab, lw, True, z) + (z,))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_cuda_graph_replay_equals_the_eager_call():
    from xtuner_b200 import ops

    T, H, V = 2048, 512, 16384
    h, w = _random(T, H, V, seed=17)
    lab = _labels(T, V, seed=17)
    lw = torch.rand(T, device=DEV)

    def step(hh, ww):
        loss = ops.lm_head_cross_entropy(hh, ww, lab, lw, IGN, 1024)
        loss.backward()
        return loss, hh.grad, ww.grad

    eager = [t.clone() for t in step(h.clone().requires_grad_(True), w.clone().requires_grad_(True))]
    # the capture's leaves are first used on a side stream (torch.cuda.graph's warm-up rule): a leaf first used on the
    # legacy default stream would accumulate its gradient there, which a capture cannot depend on
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(hh, ww)
    torch.cuda.current_stream().wait_stream(side)
    hh.grad = ww.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step(hh, ww)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref absent (oracle/make_ref.py places the reference package there)")
@pytest.mark.parametrize("mode", ["eager", "chunk"])
def test_plugin_on_the_reference_lm_head(mode):
    from tests.golden import ref_shim
    from xtuner_b200 import plugin

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    ref_shim.import_reference()
    from xtuner.v1.loss.ce_loss import CELossConfig, CELossKwargs, LMHeadLossContext
    from xtuner.v1.module.lm_head.lm_head import LMHead

    T, H, V = 2500, 1024, 32768
    torch.manual_seed(0)
    head = LMHead(H, V, bias=False).to(DEV, torch.bfloat16)
    x = torch.randn(1, T, H, device=DEV).to(torch.bfloat16)
    lab = _labels(T, V, seed=19).view(1, T)

    def run():
        cfg = CELossConfig(mode=mode, chunk_size=1024, ignore_idx=IGN)
        (ctx,) = LMHeadLossContext.build_batches([LMHeadLossContext(cfg, CELossKwargs(shifted_labels=lab))])
        xx = x.clone().requires_grad_(True)
        head.zero_grad()
        loss, (logits, _) = head(xx, ctx)
        loss.backward()
        return loss.detach(), xx.grad, head.weight.grad.clone(), logits

    from xtuner_b200 import _capi

    lib = _capi.load()
    n0 = lib.xtb_launch_count()
    want = run()
    assert lib.xtb_launch_count() == n0  # the reference's own path
    plugin.install_lm_head_loss()
    try:
        got = run()
    finally:
        plugin.uninstall_lm_head_loss()
    assert got[3] is None and lib.xtb_launch_count() > n0, "the installed path did not run xtb_lm_head_ce"
    rl = abs(got[0].item() - want[0].item()) / abs(want[0].item())
    print(f"plugin {mode}: loss rel {rl:.2e}, dh {_rel(got[1], want[1]):.2e}, dW {_rel(got[2], want[2]):.2e}")
    assert rl <= 1e-5
    for a, b in zip(got[1:3], want[1:3]):
        torch.testing.assert_close(a.float(), b.float(), rtol=2 ** -7, atol=2 ** -7 * b.float().abs().max().item())
