"""GPU parity of dispatch (permute) / combine (unpermute) kernels: golden vectors from the reference,
the reference's known-answer test, and size-independent properties at BASELINE.json's full size."""
import pytest
import torch

from oracle import moe_oracle as O
from tests.conftest import load_golden

pytestmark = pytest.mark.gpu


def test_noep_known_answer_through_dispatcher():
    """tests/module/dispatcher/test_noep.py:19-87 replayed through FusedDispatcher."""
    from xtuner_b200.dispatcher import FusedDispatcher

    g = load_golden("noep_kat")
    d = FusedDispatcher(n_routed_experts=4)
    hidden, ids, w = g["hidden_states"].cuda(), g["topk_ids"].cuda(), g["topk_weights"].cuda()
    pre = d.dispatch_preprocess(hidden_states=hidden, topk_ids=ids, topk_weights=w)
    dis = d.dispatch(pre_dispatched=pre, topk_weights=w, decoding=False)
    post = d.dispatch_postprocess(pre_dispatched=pre, dispatched=dis)
    assert torch.equal(post["hidden_states"].cpu(), g["permuted"])
    assert torch.equal(post["tokens_per_expert"].cpu(), g["tokens_per_expert"])
    prec = d.combine_preprocess(hidden_states=post["hidden_states"], pre_dispatched=pre, dispatched=dis, post_dispatched=post)
    comb = d.combine(pre_dispatched=pre, dispatched=dis, post_dispatched=post, pre_combined=prec, decoding=False)
    out = d.combine_postprocess(pre_dispatched=pre, dispatched=dis, post_dispatched=post, pre_combined=prec, combined=comb)
    assert torch.equal(out["hidden_states"].cpu(), g["target"])


@pytest.mark.parametrize("tag", ["c2", "k8", "empty_expert"])
def test_permute_unpermute_golden(tag):
    from xtuner_b200 import ops

    g = load_golden(f"dispatch_{tag}")
    K = g["topk_ids"].shape[1]
    exact = K <= 2  # fp32-accumulate pin: identical to the fallback's bf16 index_add only for K<=2
    x = g["x"].cuda().requires_grad_(True)
    perm, rmap, sorted_idx, tpe = ops.permute(x, g["topk_ids"].cuda().int(), n_experts=g["n_experts"], return_extra=True)
    assert torch.equal(perm.cpu(), g["permuted"])
    assert torch.equal(sorted_idx.cpu(), g["row_id_map"])  # == reference fallback's row_id_map (row -> flat)
    assert torch.equal(tpe.cpu(), g["tokens_per_expert"])
    inv = torch.empty_like(g["row_id_map"])
    inv[g["row_id_map"]] = torch.arange(inv.numel())
    assert torch.equal(rmap.cpu().long(), inv)
    (gx,) = torch.autograd.grad(perm, x, g["grad_permuted"].cuda())
    if exact:
        assert torch.equal(gx.cpu(), g["grad_x"])
    else:
        torch.testing.assert_close(gx.float().cpu(), g["grad_x"].float(), rtol=2e-2, atol=2e-2)
    y = g["y"].cuda().requires_grad_(True)
    p = g["probs"].cuda().requires_grad_(True)
    out = ops.unpermute(y, rmap, p)
    if exact:
        assert torch.equal(out.cpu(), g["out"])
    else:
        torch.testing.assert_close(out.float().cpu(), g["out"].float(), rtol=1e-2, atol=1e-2)
    gy, gp = torch.autograd.grad(out, (y, p), g["grad_out"].cuda())
    assert torch.equal(gy.cpu(), g["grad_y"])
    torch.testing.assert_close(gp.cpu(), g["grad_probs"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("T,H,E,K", [(8192, 2048, 8, 2), (4099, 1024, 128, 8), (1, 256, 8, 2), (7, 64, 4, 3), (2048, 7168, 256, 8),
                                     (300, 12776, 8, 2), (300, 12800, 8, 2)])
def test_dispatch_properties_full_size(T, H, E, K):
    """Bit-exact against the oracle at config sizes + round trip + histogram/sortedness properties.  H = 12776 is the
    longest bf16 row at K = 2 that the row gather stages in shared memory; H = 12800 takes the register-staged gather."""
    from xtuner_b200 import ops

    g = torch.Generator().manual_seed(T * 3 + K)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16)
    ids = torch.rand(T, E, generator=g).topk(K, dim=1)[1].int()
    xd = x.cuda()
    perm, rmap, sorted_idx, tpe = ops.permute(xd, ids.cuda(), n_experts=E, return_extra=True)
    ref_perm, ref_sorted = O.permute(x, ids)
    assert torch.equal(sorted_idx.cpu(), ref_sorted)
    assert torch.equal(perm.cpu(), ref_perm)
    assert torch.equal(tpe.cpu(), O.tokens_per_expert_hist(ids, E))
    # sortedness: expert id along permuted rows is non-decreasing, stable inside an expert
    e_of_row = ids.reshape(-1)[sorted_idx.cpu()]
    assert (e_of_row[1:] >= e_of_row[:-1]).all()
    same = e_of_row[1:] == e_of_row[:-1]
    assert (sorted_idx.cpu()[1:][same] > sorted_idx.cpu()[:-1][same]).all()
    # round trip: combine with probs = 1/K of the permuted copies of x returns x*1 (exact in bf16 for K=2^n)
    probs = torch.full((T, K), 1.0 / K)
    back = ops.unpermute(perm, rmap, probs.cuda())
    if K in (1, 2, 4, 8):
        assert torch.equal(back.cpu(), x)
    else:
        torch.testing.assert_close(back.float().cpu(), x.float(), rtol=1e-2, atol=1e-2)
    # combine vs oracle with random probs
    p = torch.rand(T, K, generator=g)
    y = torch.randn(T * K, H, generator=g).to(torch.bfloat16)
    out = ops.unpermute(y.cuda(), rmap, p.cuda())
    ref = O.unpermute(y, ref_sorted, p)
    if K <= 2:
        assert torch.equal(out.cpu(), ref)
    else:
        torch.testing.assert_close(out.float().cpu(), ref.float(), rtol=1e-2, atol=1e-2)


def test_zero_tokens_and_errors():
    from xtuner_b200 import _capi, ops

    x = torch.empty(0, 128, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    perm, rmap = ops.permute(x, torch.empty(0, 2, dtype=torch.int32, device="cuda"), n_experts=8)
    assert perm.shape[0] == 0 and rmap is None
    with pytest.raises(_capi.XtbError):
        ops.permute(torch.zeros(4, 128, dtype=torch.bfloat16), torch.zeros(4, 2, dtype=torch.int32), n_experts=8)
    with pytest.raises(_capi.XtbError):  # row bytes not a multiple of 16
        ops.permute(torch.zeros(4, 9, dtype=torch.bfloat16, device="cuda"), torch.zeros(4, 2, dtype=torch.int32, device="cuda"), n_experts=8)


@pytest.mark.parametrize("M,I", [(16384, 768), (100, 128), (3, 8)])
def test_swiglu(M, I):
    from xtuner_b200 import ops

    g = torch.Generator().manual_seed(M)
    h = (torch.randn(M, 2 * I, generator=g) * 2).to(torch.bfloat16)
    go = torch.randn(M, I, generator=g).to(torch.bfloat16)
    hr = h.clone().requires_grad_(True)
    ref = O.swiglu(hr)
    (gref,) = torch.autograd.grad(ref, hr, go)
    hd = h.cuda().requires_grad_(True)
    out = ops.swiglu(hd)
    (gh,) = torch.autograd.grad(out, hd, go.cuda())
    # bf16 results: identical up to rare 1-ulp flips from exp ulp differences between CPU and GPU
    mism = (out.cpu() != ref.detach()).float().mean().item()
    assert mism < 1e-3, mism
    torch.testing.assert_close(out.float().cpu(), ref.detach().float(), rtol=8e-3, atol=1e-6)
    torch.testing.assert_close(gh.float().cpu(), gref.float(), rtol=1.6e-2, atol=1e-5)
