"""xtb_lm_head_logprob / xtb_lm_head_logprob_bwd and ``ops.lm_head_logprobs`` on an H100:

* logp and G from the kernel's own logits against float64 formulas; dh and dW from the kernel's own G against the
  scale-aware bound of ``tests/gemm_reference.py``;
* label -100 reads token 0, a label >= V gives NaN in its row only;
* bit equality with ``xtb_lm_head_ce``: -logp == row_ce, and the backward with c = -w gives its G, dh and dW;
* the op end to end at the Qwen3-MoE head against the reference's arithmetic (F.linear -> .float() -> log_softmax ->
  gather, torch autograd) in eager and chunk mode; chunked == unchunked and no-grad == grad logprobs, bit for bit;
* determinism, CUDA-graph capture, 64-bit addressing, T = 0, and the plugin on the reference's own ``LMHead``."""
import os

import pytest
import torch
from torch.nn import functional as F

from tests import gemm_reference as R
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "xtuner", "v1"))
DEV = "cuda"
IGN = -100


def _fwd(h, w, lab, z, stats=True):
    """one xtb_lm_head_logprob call -> (logp, row_stats or None); z receives the logits"""
    lib = ensure_init()
    T, H = h.shape
    V = w.shape[0]
    ws = torch.empty(max(int(lib.xtb_lm_head_logprob_workspace_bytes(T, V)), 16), dtype=torch.uint8, device=DEV)
    logp = torch.empty(T, dtype=torch.float32, device=DEV)
    rs = torch.empty((T, 2), dtype=torch.float32, device=DEV) if stats else None
    check(lib.xtb_lm_head_logprob(ptr(h), ptr(w), ptr(lab), T, H, V, ptr(z), ptr(ws), ptr(logp), ptr(rs),
                                  current_stream()), "xtb_lm_head_logprob")
    return logp, rs


def _bwd(z, rs, lab, c, h, w):
    """one xtb_lm_head_logprob_bwd call -> (dh, dW); z receives G"""
    lib = ensure_init()
    T, H = h.shape
    V = w.shape[0]
    ws = torch.empty(max(int(lib.xtb_lm_head_logprob_workspace_bytes(0, V)), 16), dtype=torch.uint8, device=DEV)
    dh, dw = torch.empty_like(h), torch.empty_like(w)
    check(lib.xtb_lm_head_logprob_bwd(ptr(z), ptr(rs), ptr(lab), ptr(c), ptr(h), ptr(w), T, H, V, ptr(ws), ptr(dh),
                                      ptr(dw), current_stream()), "xtb_lm_head_logprob_bwd")
    return dh, dw


def _ce(h, w, lab, lw, z):
    lib = ensure_init()
    T, H = h.shape
    V = w.shape[0]
    ws = torch.empty(max(int(lib.xtb_lm_head_ce_workspace_bytes(T, V)), 16), dtype=torch.uint8, device=DEV)
    row_ce = torch.empty(T, dtype=torch.float32, device=DEV)
    loss = torch.empty((), dtype=torch.float32, device=DEV)
    dh, dw = torch.empty_like(h), torch.empty_like(w)
    check(lib.xtb_lm_head_ce(ptr(h), ptr(w), ptr(lab), ptr(lw), T, H, V, IGN, 1, ptr(z), ptr(ws), ptr(row_ce),
                             ptr(loss), ptr(dh), ptr(dw), current_stream()), "xtb_lm_head_ce")
    return row_ce, dh, dw


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


def _lsm64(z):
    return torch.log_softmax(z.double(), dim=-1)


@pytest.mark.parametrize("V,scale", [(1152, 1.0), (2048, 1.0), (1152, 2500.0)])  # 2500: logits of magnitude ~1e4
def test_logp_and_grad_from_the_kernels_logits(V, scale):
    T, H = 1000, 256
    h, w = _random(T, H, V, seed=V, scale=scale)
    lab = _labels(T, V, seed=7)
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    logp, rs = _fwd(h, w, lab, z)
    zk = z.clone()
    lsm = _lsm64(zk)
    idx = lab.clip(min=0)
    want = lsm.gather(1, idx[:, None])[:, 0]
    rel = (logp.double() - want).abs() / want.abs().clamp_min(1.0 if scale > 1 else 1e-30)
    print(f"V={V} scale={scale}: max rel logp error {rel.max().item():.2e}")
    assert torch.isfinite(logp).all() and rel.max() <= 1e-6
    assert torch.equal(rs[:, 0], zk.float().amax(1))
    c = torch.randn(T, device=DEV)
    dh, dw = _bwd(z, rs, lab, c, h, w)
    g64 = -torch.exp(lsm) * c.double()[:, None]
    g64.scatter_add_(1, idx[:, None], c.double()[:, None])
    d = R.ulp_distance(z, R.bf16_rn(g64))
    print(f"V={V} scale={scale}: G max ulp {d.max().item()}, exact share {(d == 0).double().mean().item():.6f}")
    assert torch.isfinite(z.float()).all() and d.max() <= 1 and (d == 0).double().mean() >= 0.999
    r1 = R.check_bound(dh, "nn", z, w[None], [T], what="dh")
    r2 = R.check_bound(dw[None], "tn", z, h, [T], what="dW")
    print(f"dh worst |err|/bound {r1:.3f}, dW {r2:.3f}")


def test_ignored_label_reads_token_0_and_label_V_gives_nan_in_its_row_only():
    T, H, V = 300, 256, 1024
    h, w = _random(T, H, V, seed=3)
    lab = _labels(T, V, seed=3)
    lab[10], lab[11], lab[12] = V, IGN, 0
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    logp, rs = _fwd(h, w, lab, z)
    torch.cuda.synchronize()
    want = _lsm64(z[11])[0].item()  # the row's log-probability of token 0
    assert abs(logp[11].item() - want) <= 1e-6 * abs(want)
    ok = torch.ones(T, dtype=torch.bool, device=DEV)
    ok[10] = False
    assert torch.isnan(logp[10]) and torch.isfinite(logp[ok]).all()
    _bwd(z, rs, lab, torch.ones(T, device=DEV), h, w)
    torch.cuda.synchronize()
    assert torch.isnan(z[10].float()).all() and torch.isfinite(z[ok].float()).all()


@pytest.mark.parametrize("T,H,V", [(1000, 512, 32768), (777, 256, 1152)])  # 256- and 128-column vocab tiles
def test_bit_equal_to_the_cross_entropy_entry(T, H, V):
    h, w = _random(T, H, V, seed=T)
    lab = _labels(T, V, seed=T)
    lw = (torch.rand(T, device=DEV) + 0.5) * (lab != IGN)
    zc = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    row_ce, dh_ce, dw_ce = _ce(h, w, lab, lw, zc)
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    logp, rs = _fwd(h, w, lab, z)
    keep = lab != IGN
    assert torch.equal(-logp[keep], row_ce[keep])
    dh, dw = _bwd(z, rs, lab, -lw, h, w)
    assert torch.equal(z, zc) and torch.equal(dh, dh_ce) and torch.equal(dw, dw_ce)


def _ref_logprobs(h, w, lab):
    return F.log_softmax(F.linear(h, w).float(), dim=-1).gather(-1, lab.clip(min=0)[..., None])[..., 0]


def _policy_like_loss(logp, old, adv, wt):
    """a per-token loss of logp with a coefficient that depends on logp (an importance ratio times an advantage)"""
    return -(torch.exp(logp - old) * adv * wt).sum()


def _fwd_bwd(logprobs_fn, h, w, lab, old, adv, wt, chunk):
    """loss, dh, dW: eager (one call) or chunked as ChunkLoss does it (per-chunk grad, dW added in bf16)"""
    T = h.shape[0]
    step = T if chunk is None else chunk
    loss, dh, dw = torch.zeros((), device=DEV), torch.empty_like(h), torch.zeros_like(w)
    for s in range(0, T, step):
        hc = h[s:s + step].detach().requires_grad_(True)
        ww = w.detach().requires_grad_(True)
        lc = _policy_like_loss(logprobs_fn(hc, ww, lab[s:s + step]), old[s:s + step], adv[s:s + step], wt[s:s + step])
        gh, gw = torch.autograd.grad(lc, (hc, ww))
        loss.add_(lc.detach())
        dh[s:s + step] = gh
        dw.add_(gw)
    return loss, dh, dw


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()


def _rl_inputs(T, V, seed):
    h, w = _random(T, 2048, V, seed=seed)
    lab = _labels(T, V, seed=seed)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    old = _ref_logprobs(h, w, lab) + 0.2 * torch.randn(T, generator=g, device=DEV)
    adv = torch.randn(T, generator=g, device=DEV)
    wt = (lab != IGN).float() / (lab != IGN).sum()
    return h, w, lab, old, adv, wt


@pytest.mark.parametrize("T,chunk", [(8192, None), (3000, 1024)])
def test_end_to_end_against_the_reference_at_the_qwen3_head(T, chunk):
    from xtuner_b200 import ops

    h, w, lab, old, adv, wt = _rl_inputs(T, 151936, seed=11)
    want = _fwd_bwd(_ref_logprobs, h, w, lab, old, adv, wt, chunk)
    got = _fwd_bwd(ops.lm_head_logprobs, h, w, lab, old, adv, wt, chunk)
    rl = abs(got[0].item() - want[0].item()) / abs(want[0].item())
    print(f"T={T} chunk={chunk}: loss rel {rl:.2e}; max|err|/max|ref| dh {_rel(got[1], want[1]):.2e} "
          f"dW {_rel(got[2], want[2]):.2e}")
    assert rl <= 1e-5
    for a, b in zip(got[1:], want[1:]):
        torch.testing.assert_close(a.float(), b.float(), rtol=2 ** -7, atol=2 ** -7 * b.float().abs().max().item())
    with torch.no_grad():
        lp_ref = _ref_logprobs(h, w, lab)
        lp = ops.lm_head_logprobs(h, w, lab)
        lp_chunked = ops.lm_head_logprobs(h, w, lab, chunk_size=1000)
    print(f"T={T}: logp max |err| vs reference {(lp - lp_ref).abs().max().item():.2e}")
    torch.testing.assert_close(lp, lp_ref, rtol=2 ** -7, atol=2 ** -7)  # one bf16 ulp of a logit moves logp by as much
    assert torch.equal(lp, lp_chunked)
    lp_grad = ops.lm_head_logprobs(h.detach().requires_grad_(True), w, lab)
    assert lp_grad.requires_grad and torch.equal(lp_grad.detach(), lp)


def test_two_calls_give_identical_bits():
    from xtuner_b200 import ops

    T, H, V = 4096, 1024, 32768
    h, w = _random(T, H, V, seed=13)
    lab = _labels(T, V, seed=13)
    c = torch.randn(T, device=DEV)
    outs = []
    for _ in range(2):
        hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
        lp = ops.lm_head_logprobs(hh, ww, lab)
        lp.backward(c)
        outs.append((lp.detach(), hh.grad, ww.grad))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_cuda_graph_replay_of_the_grpo_step_equals_the_eager_call():
    from xtuner_b200 import ops

    T, H, V = 2048, 512, 16384
    h, w = _random(T, H, V, seed=17)
    lab = _labels(T, V, seed=17)
    g = torch.Generator(device=DEV).manual_seed(17)
    old = torch.randn(T, generator=g, device=DEV) - 9.0
    adv = torch.randn(T, generator=g, device=DEV)
    wt = (lab != IGN).float() / (lab != IGN).sum()

    def step(hh, ww):
        loss = _policy_like_loss(ops.lm_head_logprobs(hh, ww, lab), old, adv, wt)
        loss.backward()
        return loss, hh.grad, ww.grad

    eager = [t.clone() for t in step(h.clone().requires_grad_(True), w.clone().requires_grad_(True))]
    hh, ww = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    side = torch.cuda.Stream()  # warm-up on a side stream, as torch.cuda.graph requires of the capture's leaves
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


def test_64bit_addressing_matches_two_halves():
    T, H, V = 16384, 256, 151936  # T * V = 2.49e9 elements > 2^31
    h, w = _random(T, H, V, seed=5)
    lab = _labels(T, V, seed=5)
    c = torch.randn(T, device=DEV)
    z = torch.empty((T, V), dtype=torch.bfloat16, device=DEV)
    logp, rs = _fwd(h, w, lab, z)
    dh, dw = _bwd(z, rs, lab, c, h, w)
    del z
    parts = []
    for s in (0, T // 2):
        zh = torch.empty((T // 2, V), dtype=torch.bfloat16, device=DEV)
        sl = slice(s, s + T // 2)
        lp_h, rs_h = _fwd(h[sl], w, lab[sl], zh)
        parts.append((lp_h, rs_h) + _bwd(zh, rs_h, lab[sl], c[sl], h[sl], w))
        del zh
    assert torch.equal(logp, torch.cat([parts[0][0], parts[1][0]]))
    assert torch.equal(rs, torch.cat([parts[0][1], parts[1][1]]))
    assert torch.equal(dh, torch.cat([parts[0][2], parts[1][2]]))
    torch.testing.assert_close(dw.float(), parts[0][3].float() + parts[1][3].float(), rtol=2 ** -7,
                               atol=2 ** -7 * dw.float().abs().max().item())


def test_zero_rows_write_nothing_forward_and_a_zero_weight_gradient_backward():
    from xtuner_b200 import ops

    H, V = 256, 1024
    _, w = _random(1, H, V, seed=21)
    h = torch.empty((0, H), dtype=torch.bfloat16, device=DEV).requires_grad_(True)
    ww = w.clone().requires_grad_(True)
    lp = ops.lm_head_logprobs(h, ww, torch.empty((0,), dtype=torch.int64, device=DEV))
    assert lp.shape == (0,)
    lp.sum().backward()
    assert h.grad.shape == (0, H) and (ww.grad == 0).all()


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref absent (oracle/make_ref.py places the reference package there)")
@pytest.mark.parametrize("mode", ["eager", "chunk"])
def test_plugin_on_the_reference_lm_head(mode):
    from tests.golden import ref_shim
    from xtuner_b200 import _capi, plugin

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    ref_shim.import_reference()
    from xtuner.v1.loss.rl_loss import LogProbConfig, LogProbContext, LogProbKwargs
    from xtuner.v1.module.lm_head.lm_head import LMHead
    from xtuner.v1.rl.loss.grpo_loss import GRPOLossConfig, GRPOLossContext, GRPOLossKwargs

    T, H, V = 2500, 1024, 32768
    torch.manual_seed(0)
    head = LMHead(H, V, bias=False).to(DEV, torch.bfloat16)
    x = torch.randn(1, T, H, device=DEV).to(torch.bfloat16)
    lab = _labels(T, V, seed=19).view(1, T)
    g = torch.Generator(device=DEV).manual_seed(19)
    adv = torch.randn(1, T, generator=g, device=DEV)
    noise = 0.3 * torch.randn(1, T, generator=g, device=DEV)

    def logprobs():
        ctx = LogProbContext(LogProbConfig(mode=mode, chunk_size=1024, ignore_idx=IGN), LogProbKwargs(shifted_labels=lab))
        with torch.no_grad():
            lp, (logits, extra) = head(x, ctx)
        return lp, logits, extra

    def grpo(old):
        cfg = GRPOLossConfig(policy_loss_cfg={"loss_type": "vanilla", "cliprange_low": 0.2, "cliprange_high": 0.28},
                             use_kl_loss=True, kl_loss_coef=0.001, kl_loss_type="low_var_kl", mode=mode, chunk_size=1024,
                             ignore_idx=IGN)
        kw = GRPOLossKwargs(shifted_labels=lab, old_logprobs=old, advantages=adv, ref_logprobs=old + noise)
        (ctx,) = GRPOLossContext.build_batches([GRPOLossContext(cfg, kw)])
        xx = x.clone().requires_grad_(True)
        head.zero_grad()
        loss, (logits, extra) = head(xx, ctx)
        loss.backward()
        return loss.detach(), xx.grad, head.weight.grad.clone(), logits, extra

    lib = _capi.load()
    n0 = lib.xtb_launch_count()
    want_lp = logprobs()
    old = want_lp[0] - 0.1 * noise
    want = grpo(old)
    assert lib.xtb_launch_count() == n0  # the reference's own path
    plugin.install_rl_lm_head()
    try:
        got_lp = logprobs()
        n1 = lib.xtb_launch_count()
        got = grpo(old)
    finally:
        plugin.uninstall_rl_lm_head()
    assert n1 > n0 and lib.xtb_launch_count() > n1, "the installed path did not run the logprob entries"
    assert got_lp[1] is None and got[3] is None
    rl = abs(got[0].item() - want[0].item()) / abs(want[0].item())
    print(f"plugin {mode}: logp max |err| {(got_lp[0] - want_lp[0]).abs().max().item():.2e}, loss rel {rl:.2e}, "
          f"dh {_rel(got[1], want[1]):.2e}, dW {_rel(got[2], want[2]):.2e}")
    torch.testing.assert_close(got_lp[0], want_lp[0], rtol=2 ** -7, atol=2 ** -7)
    assert rl <= 5e-5  # mixed-sign advantages: the loss is a cancelling sum, its relative error is larger than a CE's
    for a, b in zip(got[1:3], want[1:3]):
        torch.testing.assert_close(a.float(), b.float(), rtol=2 ** -7, atol=2 ** -7 * b.float().abs().max().item())
    assert set(got[4]) == set(want[4])
    assert torch.equal(got[4]["reduced_train_policy_valid_count"], want[4]["reduced_train_policy_valid_count"])
