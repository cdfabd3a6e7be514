"""Selective recompute of the fused MoE nodes on an H100 (``recompute="act"`` / ``"experts"``, ``xtuner_b200/fused.py``):

* ``xtb_swiglu_bwd_act``: its ``a`` equals ``xtb_swiglu`` and its ``g_h`` equals ``xtb_swiglu_bwd`` bit for bit, at
  every bf16 gate value and at edge widths and row counts, writing nothing outside its rows;
* both nodes, at C2 and at the Qwen3-30B-A3B MoE geometry (E = 128, K = 8), routed and replayed: every output and
  every gradient of each mode equals ``recompute=None`` bit for bit (the permute is a stable sort, the grouped GEMMs run
  no split-K and no atomics, so the rebuilt intermediates are the forward's);
* a two-layer forward + backward captured in a CUDA graph and replayed equals the eager run in each mode;
* over an 8-layer C2 stack, each mode's peak allocated memory lies at least 6 x the per-layer dropped bytes below
  ``recompute=None``."""
import pytest
import torch

from tests.gpu_harness import Guarded
from xtuner_b200._capi import check, current_stream, ensure_init

pytestmark = pytest.mark.gpu

DEV = "cuda"
MODES = ("act", "experts")
C2 = (8192, 2048, 768, 8, 2)
QWEN3_30B_A3B = (4096, 2048, 768, 128, 8)


def _call(name, *args):
    check(getattr(ensure_init(), name)(*args, current_stream()), name)


def _bits(t):
    return t.view(torch.int16)


# ---- the kernel ---------------------------------------------------------------------------------------------------------


def _swiglu_pair(h, d):
    """(a, g_h) of xtb_swiglu_bwd_act in guarded buffers, and (a, g_h) of xtb_swiglu and xtb_swiglu_bwd"""
    M, I = d.shape
    a, gh = Guarded(M, I, torch.bfloat16), Guarded(M, 2 * I, torch.bfloat16)
    _call("xtb_swiglu_bwd_act", d.data_ptr(), h.data_ptr(), gh.v.data_ptr(), a.v.data_ptr(), M, I)
    a_ref = torch.empty(M, I, dtype=torch.bfloat16, device=DEV)
    gh_ref = torch.empty(M, 2 * I, dtype=torch.bfloat16, device=DEV)
    _call("xtb_swiglu", h.data_ptr(), a_ref.data_ptr(), M, I)
    _call("xtb_swiglu_bwd", d.data_ptr(), h.data_ptr(), gh_ref.data_ptr(), M, I)
    torch.cuda.synchronize()
    return (a.check("act"), gh.check("grad_h")), (a_ref, gh_ref)


def test_swiglu_bwd_act_at_every_gate_value():
    """every bf16 bit pattern as the gate (±0, subnormals, ±inf, NaNs, the band where the sigmoid's reciprocal goes
    subnormal), against up values and output gradients that hold 0, NaN and the largest bf16"""
    I = 64
    gate = torch.arange(-32768, 32768, dtype=torch.int32, device=DEV).to(torch.int16).view(torch.bfloat16).view(-1, I)
    M = gate.shape[0]
    gen = torch.Generator(DEV).manual_seed(3)
    up = (torch.randn(M, I, generator=gen, device=DEV) * 4).to(torch.bfloat16)
    d = torch.randn(M, I, generator=gen, device=DEV).to(torch.bfloat16)
    for t in (up, d):
        t.view(-1)[::97] = 0
        t.view(-1)[5::101] = float("nan")
        t.view(-1)[7::103] = torch.finfo(torch.bfloat16).max
    h = torch.cat([gate, up], 1).contiguous()
    (a, gh), (a_ref, gh_ref) = _swiglu_pair(h, d)
    assert torch.equal(_bits(a), _bits(a_ref)) and torch.equal(_bits(gh), _bits(gh_ref))


@pytest.mark.parametrize("M,I", [(1, 8), (7, 8), (9, 24), (17, 136), (4099, 768), (3, 8 * 23170)])
def test_swiglu_bwd_act_at_edge_widths(M, I):
    """I = 8 (the special-cased row split), non-power-of-two I / 8, the widest row the host accepts, and row counts that
    are not a multiple of the 8-row block"""
    gen = torch.Generator(DEV).manual_seed(M + I)
    h = (torch.randn(M, 2 * I, generator=gen, device=DEV) * 3).to(torch.bfloat16)
    d = torch.randn(M, I, generator=gen, device=DEV).to(torch.bfloat16)
    (a, gh), (a_ref, gh_ref) = _swiglu_pair(h, d)
    assert torch.equal(_bits(a), _bits(a_ref)) and torch.equal(_bits(gh), _bits(gh_ref))


def test_swiglu_bwd_act_equals_the_gemm_epilogue():
    """``a`` as the w13 grouped GEMM's SwiGLU epilogue writes it in the forward, from the h that GEMM writes beside it"""
    T, H, I, E, K = 1024, 1024, 768, 8, 2
    M = T * K
    gen = torch.Generator(DEV).manual_seed(5)
    x = torch.randn(M, H, generator=gen, device=DEV).to(torch.bfloat16)
    w13 = (torch.randn(E, 2 * I, H, generator=gen, device=DEV) * H**-0.5).to(torch.bfloat16)
    tpe = torch.full((E,), M // E, dtype=torch.int64, device=DEV)
    tpe[0] += 5
    tpe[1] -= 5
    h = torch.empty(M, 2 * I, dtype=torch.bfloat16, device=DEV)
    a_gemm = torch.empty(M, I, dtype=torch.bfloat16, device=DEV)
    _call("xtb_group_gemm_nt_swiglu", x.data_ptr(), w13.data_ptr(), tpe.data_ptr(), M, I, H, E, h.data_ptr(),
          a_gemm.data_ptr())
    d = torch.randn(M, I, generator=gen, device=DEV).to(torch.bfloat16)
    (a, _), _ = _swiglu_pair(h, d)
    assert torch.equal(_bits(a), _bits(a_gemm))


# ---- the nodes ----------------------------------------------------------------------------------------------------------


def _inputs(T, H, I, E, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    return dict(
        h=torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16),
        res=torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16),
        nw=1 + 0.1 * torch.randn(H, generator=g, device=DEV),
        gw=torch.randn(E, H, generator=g, device=DEV) * 0.02,
        w13=(torch.randn(E, 2 * I, H, generator=g, device=DEV) * H**-0.5).to(torch.bfloat16),
        w2=(torch.randn(E, H, I, generator=g, device=DEV) * I**-0.5).to(torch.bfloat16),
        go=torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16),
        g_rw=torch.randn(T, E, generator=g, device=DEV) * 0.01,
    )


def _run(node, p, K, replay, recompute):
    from xtuner_b200 import fused

    if node == "block":
        leaves = [p[k].clone().requires_grad_(True) for k in ("h", "nw", "gw", "w13", "w2")]
        out, rr = fused.fused_moe_block(leaves[0], leaves[1], 1e-6, *leaves[2:], top_k=K, rollout_routed_experts=replay,
                                        recompute=recompute)
    else:
        leaves = [p[k].clone().requires_grad_(True) for k in ("h", "res", "gw", "w13", "w2")]
        out, rr = fused.fused_moe(leaves[0], leaves[1], *leaves[2:], top_k=K, rollout_routed_experts=replay,
                                  recompute=recompute)
    torch.autograd.backward([out, rr["router_weights"]], [p["go"], p["g_rw"]])
    return [out.detach(), rr["logits"].detach(), rr["router_weights"].detach(), rr["topk_ids"]] + [t.grad for t in leaves]


@pytest.mark.parametrize("shape", [C2, QWEN3_30B_A3B], ids=["c2", "qwen3_30b_a3b"])
@pytest.mark.parametrize("node", ["block", "residual"])
def test_each_mode_equals_the_saved_path(shape, node):
    T, H, I, E, K = shape
    p = _inputs(T, H, I, E, E + K)
    want = _run(node, p, K, None, None)
    # replayed: ids unlike the router's own (a few duplicates in a row included), so the expert groups change size
    ids = torch.randint(0, E, (T, K), generator=torch.Generator(DEV).manual_seed(1), device=DEV)
    ids[::5, 0] = ids[::5, -1]
    want_replayed = _run(node, p, K, ids, None)
    assert not torch.equal(want_replayed[0], want[0])
    for mode in MODES:
        for replay, ref in ((None, want), (ids, want_replayed)):
            got = _run(node, p, K, replay, mode)
            for i, (a, b) in enumerate(zip(got, ref)):
                assert torch.equal(a, b), f"{mode}, replay {replay is not None}: output {i} differs"
    torch.cuda.synchronize()


def _stack(layers, mode, go):
    """forward + backward of a stack of fused blocks; returns the output and every leaf gradient"""
    from xtuner_b200 import fused

    h0, params = layers
    x = h0.clone().requires_grad_(True)
    leaves = [[t.clone().requires_grad_(True) for t in ps] for ps in params]
    h = x
    for nw, gw, w13, w2 in leaves:
        h, _ = fused.fused_moe_block(h, nw, 1e-6, gw, w13, w2, top_k=2, recompute=mode)
    h.backward(go)
    return [h.detach(), x.grad] + [t.grad for ps in leaves for t in ps]


def _layers(n, T, H, I, E, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    h0 = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    params = [(1 + 0.1 * torch.randn(H, generator=g, device=DEV), torch.randn(E, H, generator=g, device=DEV) * 0.02,
               (torch.randn(E, 2 * I, H, generator=g, device=DEV) * H**-0.5).to(torch.bfloat16),
               (torch.randn(E, H, I, generator=g, device=DEV) * I**-0.5).to(torch.bfloat16)) for _ in range(n)]
    return h0, params


@pytest.mark.parametrize("mode", MODES)
def test_two_layers_in_a_cuda_graph(mode):
    """no host synchronisation and no memset between the kernels of either mode: the step captures and replays"""
    T, H, I, E, K = 1024, 1024, 512, 8, 2
    layers = _layers(2, T, H, I, E, 11)
    go = torch.randn(T, H, generator=torch.Generator(DEV).manual_seed(12), device=DEV).to(torch.bfloat16)
    want = _stack(layers, mode, go)
    assert all(torch.equal(a, b) for a, b in zip(want, _stack(layers, None, go)))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _stack(layers, mode, go)  # warm-up on a side stream, as torch.cuda.graph asks of work it captures
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        got = _stack(layers, mode, go)
    graph.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), f"graph replay, tensor {i}"


def test_peak_memory_of_an_eight_layer_stack():
    """C2 per layer: "act" drops x_perm and a (92.3 MB), "experts" all four intermediates (209.7 MB); over 8 layers the
    peak must fall by at least 6 x that (the last layer's rebuilt tensors and the forward's transients take the rest)"""
    T, H, I, E, K = C2
    M = T * K
    dropped = {"act": (M * H + M * I) * 2, "experts": (2 * M * H + 3 * M * I) * 2}
    layers = _layers(8, T, H, I, E, 21)
    go = torch.randn(T, H, generator=torch.Generator(DEV).manual_seed(22), device=DEV).to(torch.bfloat16)
    peak = {}
    for mode in (None, *MODES, None):
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = _stack(layers, mode, go)
        torch.cuda.synchronize()
        peak[mode] = torch.cuda.max_memory_allocated() - base
        del out
    for mode in MODES:
        saved = peak[None] - peak[mode]
        assert saved >= 6 * dropped[mode], (mode, saved / 1e6, dropped[mode] / 1e6, {k: v / 1e6 for k, v in peak.items()})
