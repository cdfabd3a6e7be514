"""The MoE auxiliary-loss statistics kernels (``xtb_moe_aux_stats`` / ``xtb_moe_aux_stats_bwd``) on an H100, through the
C-ABI with guard-banded outputs:

* counts bit-equal to ``torch.histc(ids.float(), bins=E, min=0, max=E).long()`` on the device, with ids equal to E,
  negative and above E in the input;
* ``rw_sum``, ``lse``, ``z_sum`` and ``g_logits`` against float64 with bounds derived from the number of terms (the
  worst |err| / bound is printed), ``g_rw`` bit-equal to the broadcast, two calls bit-identical;
* NaN and infinite logits rows as ``torch.logsumexp`` gives them, argument checks, and two layers of forward and backward
  captured in a CUDA graph;
* the install inside the reference's tiny MoE model (``tests/workers/moe_aux_loss_worker.py``)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests.gpu_harness import XTB_ERR_INVALID, Guarded, Worst
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "xtuner", "v1"))
U = 2.0 ** -24
E_MAX = 512
WORST = Worst("moe_aux_loss")
_report = WORST.fixture()


def _workspace(N, E):
    return torch.zeros(int(ensure_init().xtb_moe_aux_stats_workspace_bytes(N, E)), dtype=torch.uint8, device="cuda")


def _inputs(N, E, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = torch.randn(N, E, device="cuda", generator=g) * 3
    rw = torch.softmax(logits, -1)
    ids = torch.randint(-2, E + 3, (N, K), device="cuda", generator=g)  # E, negatives and ids above E included
    return rw, logits, ids


def _fwd(rw, logits, ids, E, ws):
    N, K = ids.shape
    tpe, rw_sum, z_sum, lse = Guarded(E, 1, torch.int64), Guarded(E, 1, torch.float32), Guarded(1, 1, torch.float32), \
        Guarded(N, 1, torch.float32)
    check(ensure_init().xtb_moe_aux_stats(ptr(rw), ptr(logits), ptr(ids), N, E, K, ptr(tpe.v), ptr(rw_sum.v), ptr(z_sum.v),
                                          ptr(lse.v), ptr(ws), current_stream()), "xtb_moe_aux_stats")
    torch.cuda.synchronize()
    return (tpe.check("tokens_per_expert").view(-1), rw_sum.check("rw_sum").view(-1), z_sum.check("z_sum").view(()),
            lse.check("lse").view(-1))


def _bwd(g_rw_sum, g_z, logits, lse, N, E):
    g_rw, g_logits = Guarded(N, E, torch.float32), Guarded(N, E, torch.float32)
    check(ensure_init().xtb_moe_aux_stats_bwd(ptr(g_rw_sum), ptr(g_z), ptr(logits), ptr(lse), N, E, ptr(g_rw.v),
                                              ptr(g_logits.v), current_stream()), "xtb_moe_aux_stats_bwd")
    torch.cuda.synchronize()
    return g_rw.check("g_rw"), g_logits.check("g_logits")


def _lse_bound(E, lse64):
    """fp32 logsumexp: the max-shifted exp sum carries about (E + 2) u relative error (expf within 2 ulp, the rounded
    shift), its log that absolutely, plus the roundings of the log and the final add; taken twice over"""
    return (2 * E + 8) * U + 2 * U * lse64.abs()


@pytest.mark.parametrize("N", [0, 1, 33, 8192, 100003])
@pytest.mark.parametrize("K", [1, 2, 8])
@pytest.mark.parametrize("E", [1, 8, 128, 256, E_MAX])
def test_stats_and_gradients_against_histc_and_float64(E, K, N):
    rw, logits, ids = _inputs(N, E, K, seed=E * 1000 + K * 10 + N % 7)
    ws = _workspace(N, E)
    tpe, rw_sum, z_sum, lse = _fwd(rw, logits, ids, E, ws)
    assert torch.equal(tpe, torch.histc(ids.float(), bins=E, min=0, max=E).long()), "counts differ from torch.histc"
    again = _fwd(rw, logits, ids, E, ws)
    for a, b, name in zip((tpe, rw_sum, z_sum, lse), again, ("tpe", "rw_sum", "z_sum", "lse")):
        bits = (lambda t: t.reshape(-1).view(torch.int32)) if a.is_floating_point() else (lambda t: t)
        assert torch.equal(bits(a), bits(b)), f"{name}: two calls differ"
    rw64, x64 = rw.double(), logits.double()
    ref_rw = rw64.sum(0)
    bound = max(N, 1) * U * rw64.abs().sum(0) + 1e-30
    WORST.note("rw_sum |err| / bound", ((rw_sum.double() - ref_rw).abs() / bound).max())
    assert bool(((rw_sum.double() - ref_rw).abs() <= bound).all()), "rw_sum outside its bound"
    lse64 = torch.logsumexp(x64, -1)
    lb = _lse_bound(E, lse64)
    if N:
        WORST.note("lse |err| / bound", ((lse.double() - lse64).abs() / lb).max())
        assert bool(((lse.double() - lse64).abs() <= lb).all()), "lse outside its bound"
    zb = (2 * lse64.abs() * lb).sum() + max(N, 1) * U * lse64.square().sum() + 1e-30
    WORST.note("z_sum |err| / bound", (z_sum.double() - lse64.square().sum()).abs() / zb)
    assert float((z_sum.double() - lse64.square().sum()).abs()) <= float(zb), "z_sum outside its bound"

    g = torch.Generator(device="cuda").manual_seed(N + E)
    g_rw_sum = torch.randn(E, device="cuda", generator=g)
    g_z = torch.rand((), device="cuda", generator=g) + 0.5
    g_rw, g_logits = _bwd(g_rw_sum, g_z, logits, lse, N, E)
    assert torch.equal(g_rw, g_rw_sum.expand(N, E)), "g_rw is not the broadcast of g_rw_sum"
    p64 = torch.exp(x64 - lse64[:, None])
    ref_g = g_z.double() * 2 * lse64[:, None] * p64
    gb = 2 * g_z.double() * p64 * (lb[:, None] * (1 + lse64.abs()[:, None]) + 4 * U * lse64.abs()[:, None]) + 1e-30
    if N:
        WORST.note("g_logits |err| / bound", ((g_logits.double() - ref_g).abs() / gb).max())
        assert bool(((g_logits.double() - ref_g).abs() <= gb).all()), "g_logits outside its bound"
    g_rw2, g_logits2 = _bwd(g_rw_sum, g_z, logits, lse, N, E)
    assert torch.equal(g_logits2.view(torch.int32), g_logits.view(torch.int32)) and torch.equal(g_rw2, g_rw)


def test_nan_and_infinite_rows_follow_torch_logsumexp():
    E, N = 8, 5
    logits = torch.randn(N, E, device="cuda")
    logits[1, 3] = float("nan")
    logits[2] = -float("inf")
    logits[3, 0] = float("inf")
    logits[4, :4] = -float("inf")
    rw, ids = torch.softmax(logits, -1), torch.randint(0, E, (N, 2), device="cuda")
    _, _, z_sum, lse = _fwd(rw, logits, ids, E, _workspace(N, E))
    ref = torch.logsumexp(logits, -1)
    assert torch.equal(lse.isnan(), ref.isnan()), (lse, ref)
    inf = ref.isinf()
    assert torch.equal(lse[inf], ref[inf]), (lse, ref)
    fin = ref.isfinite()
    assert bool(((lse[fin] - ref[fin]).abs() <= 1e-6 * (1 + ref[fin].abs())).all()), (lse, ref)
    assert bool(z_sum.isnan())
    g_rw, g_logits = _bwd(torch.ones(E, device="cuda"), torch.ones((), device="cuda"), logits, lse, N, E)
    x = logits.clone().requires_grad_(True)
    torch.logsumexp(x, -1).square().sum().backward()
    assert torch.equal(g_logits.isnan(), x.grad.isnan()), "NaN pattern of g_logits differs from autograd's"


def test_rejects_what_it_does_not_cover():
    lib = ensure_init()
    ids = torch.zeros(4, 2, dtype=torch.int64, device="cuda")
    out = torch.empty(E_MAX + 1, dtype=torch.int64, device="cuda")
    ws = _workspace(4, E_MAX)
    for E, K in ((0, 2), (E_MAX + 1, 2), (8, 0)):
        assert lib.xtb_moe_aux_stats(None, None, ptr(ids), 4, E, K, ptr(out), None, None, None, ptr(ws),
                                     current_stream()) == XTB_ERR_INVALID
    assert lib.xtb_moe_aux_stats(None, None, ptr(ids), 4, 8, 2, ptr(out), ptr(out), None, None, ptr(ws),
                                 current_stream()) == XTB_ERR_INVALID  # rw_sum without rw
    assert lib.xtb_moe_aux_stats_bwd(None, None, None, None, 4, 8, ptr(out), None, current_stream()) == XTB_ERR_INVALID
    assert lib.xtb_moe_aux_stats_bwd(None, None, None, None, 4, 8, None, None, current_stream()) == XTB_ERR_INVALID  # no gradient in


def test_two_layers_forward_and_backward_replay_in_a_cuda_graph():
    from xtuner_b200 import ops

    N, E, K = 4099, 128, 8
    layers = [_inputs(N, E, K, seed=s) for s in (1, 2)]

    def step():
        outs = []
        for rw, logits, ids in layers:
            rw, logits = rw.clone().requires_grad_(True), logits.clone().requires_grad_(True)
            tpe, rw_sum, z_sum = ops.moe_aux_stats(rw, logits, ids, E, need_z=True)
            (rw_sum * torch.arange(E, device="cuda")).sum().add(z_sum * 1e-3).backward()
            outs += [tpe, rw_sum.detach(), z_sum.detach(), rw.grad, logits.grad]
        return outs

    eager = [t.clone() for t in step()]  # also places the workspace, its ticket at zero
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()  # warm-up on the capture stream (its own workspace)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(captured, eager):
        assert torch.equal(a, b), "a replay differs from the eager step"


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref absent (oracle/make_ref.py places the reference package there)")
def test_install_in_the_reference_model_matches_the_reference():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "workers", "moe_aux_loss_worker.py")], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    lines = [l for l in r.stdout.splitlines() if l.startswith("MOEAUXLOSS ")]
    if r.returncode != 0 or not lines:
        err = "\n".join(l for l in r.stderr.splitlines() if "Warning" not in l and l.strip())
        raise AssertionError("aux loss worker failed\nSTDOUT:\n" + r.stdout[-2000:] + "\nSTDERR:\n" + err[-6000:])
    d = json.loads(lines[-1][len("MOEAUXLOSS "):])
    for name, m in d.items():
        assert m["aux_calls"] == m["layers"], (name, m)
        assert m["tpe_equal"], f"{name}: tokens_per_expert_global differs"
        for k, v in m["loss_rel_diff"].items():
            assert v <= max(1e-5, 2 * m["noise"][k]), f"{name}: {k} differs by {v:.3e}"
        assert m["same_grad_keys"], name
        assert m["worst_grad_rel_to_max"] <= max(5e-3, 2 * m["grad_noise"]), (name, m["worst_grad"], m["worst_grad_rel_to_max"])
