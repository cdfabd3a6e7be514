"""Both fused MoE autograd nodes (``FusedMoEFunction`` behind ``fused_moe``, ``FusedMoEBlockFunction`` behind
``fused_moe_block``) against the float64 restatement of tests/fused_node_reference.py: every forward stage from the
node's own saved tensors, every gradient end to end against the propagated bound, and the loss.  Every case runs twice
and the two runs must be bit-identical.

Which case reaches which branch of xtuner_b200/fused.py:

* one-launch gate + route (E <= 8, H <= 4096) and the fused router-gate backward (E <= 8): C2, the T tails at E = 8,
  the replay cases, the block cases;
* two-call gate and router, two-call router and gate backward: Qwen3-30B-A3B (E = 128, K = 8) and the T tails at
  E = 128; the two-call gate at E <= 8 with the fused backward: H = 4224;
* xtb_group_gemm_tn_pair as one launch (I % 256 and H % 256 alike): C2, Qwen3; split into two (I = 384, H = 1024);
* the block's fused norm at H = 256 / 512 / 1024 / 2048 with and without a norm weight gradient; its F.rms_norm
  fallback at H = 3072;
* residual given and absent, hidden_factor 1 and 0.5, GRAD_SINK, T = 0: the moe cases below say which.

The worst |err| / bound per quantity and the module's wall time are printed at the end."""
import contextlib
import time

import pytest
import torch

from oracle import moe_oracle as O
from tests import fused_node_reference as FN
from tests import gemm_reference as G
from tests.gpu_harness import Worst

pytestmark = pytest.mark.gpu

DEV = "cuda"
WORST = Worst("fused_node_edges")


@contextlib.contextmanager
def _wall_time():
    t0 = time.time()
    yield
    print(f"fused_node_edges: wall time {time.time() - t0:.1f} s")


_report = WORST.fixture(_wall_time)


def _note(r):
    for k, v in r.items():
        WORST.note(k, v)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def weights(H, I, E, seed, flat=False, gate_bf16=False):
    g = _gen(seed)
    gw = torch.randn(E, H, generator=g, device=DEV) * (2 / H ** 0.5)
    w13 = (torch.randn(E, 2 * I, H, generator=g, device=DEV) * H ** -0.5).to(torch.bfloat16)
    w2 = (torch.randn(E, H, I, generator=g, device=DEV) * I ** -0.5).to(torch.bfloat16)
    if flat:
        w13, w2 = w13.view(E * 2 * I, H), w2.view(E * H, I)
    return (gw.to(torch.bfloat16) if gate_bf16 else gw), w13, w2


def replay_ids(T, E, K, pattern, seed):
    g = torch.Generator().manual_seed(seed)
    if pattern == "random":
        ids = torch.randint(0, E, (T, K), generator=g)
    elif pattern == "last":
        ids = torch.full((T, K), E - 1)
    elif pattern == "expert0_empty":
        ids = torch.randint(1, E, (T, K), generator=g)
    elif pattern == "half_empty":
        ids = torch.randint(0, E // 2, (T, K), generator=g) * 2
    elif pattern == "dup":
        ids = torch.randint(0, E, (T, K), generator=g)
        ids[::2, 1] = ids[::2, 0]
    else:
        raise ValueError(pattern)
    return ids.to(DEV)


def route_grads(route, logits, rw, tpe, K):
    """(g_logits, g_rw) of a z-loss on logits and a balancing loss on router_weights, as the route asks."""
    lg = logits.detach().clone().requires_grad_(True)
    w = rw.detach().clone().requires_grad_(True)
    g_lg = torch.autograd.grad(O.z_loss(lg, 1e-2), lg)[0] if route == "all" else None
    g_rw = torch.autograd.grad(O.balancing_loss(w, tpe, K, 0.1), w)[0] if route in ("all", "rw") else None
    return g_lg, g_rw


def _bits(a, b, what):
    if a is None or b is None:
        assert a is None and b is None, what
        return
    a, b = a.contiguous(), b.contiguous()
    assert a.shape == b.shape and torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{what}: the two runs differ"


def run_moe(x, res, gw, w13, w2, K, opts, replay=None, route="out", go=None):
    from xtuner_b200.fused import fused_moe

    leaves = [t.detach().clone().requires_grad_(True) if t is not None else None for t in (x, res, gw, w13, w2)]
    xl, rl, gl, l13, l2 = leaves
    out, rr = fused_moe(xl, rl, gl, l13, l2, top_k=K, rollout_routed_experts=replay, **opts)
    node = FN.from_autograd(out, rr["logits"], residual=rl)
    g_lg, g_rw = route_grads(route, rr["logits"], rr["router_weights"], rr["topkens_per_expert"], K)
    outs, gos = [], []
    if route != "rw":
        outs.append(out), gos.append(go)
    for o, g in ((rr["logits"], g_lg), (rr["router_weights"], g_rw)):
        if g is not None:
            outs.append(o), gos.append(g)
    wrt = [t for t in leaves if t is not None]
    gr = dict(zip(["g_x"] + (["g_res"] if rl is not None else []) + ["g_gate_w", "g_w13", "g_w2"],
                  torch.autograd.grad(outs, wrt, gos)))
    g_out = go if route != "rw" else torch.zeros_like(go)
    return node, out.detach(), rr, gr, g_out, g_lg, g_rw


def twice(fn, *a, **kw):
    r1, r2 = fn(*a, **kw), fn(*a, **kw)
    _, out1, rr1, gr1 = r1[:4]
    _, out2, rr2, gr2 = r2[:4]
    _bits(out1, out2, "out")
    for k in ("logits", "router_weights", "topk_ids", "topkens_per_expert"):
        _bits(rr1[k], rr2[k], k)
    for k in gr1:
        _bits(gr1[k], gr2[k], k)
    return r1


def check_moe(node, out, gr, g_out, g_lg, g_rw, x, res, gw, w13, w2, opts, replay=None, gate_bf16=False):
    T, H = node.t["x"].shape
    E = node.t["gate_w"].shape[0]
    r = FN.check_forward(node, replay)
    grads = dict(gr)
    grads["g_x"] = gr["g_x"].reshape(T, H)
    r.update(FN.check_backward(node, grads, g_out.reshape(T, H), g_lg, g_rw, gate_bf16=gate_bf16))
    inp = {"x": x.reshape(T, H), "gate_w": gw.float(), "w13": w13.reshape(E, -1, H), "w2": w2.reshape(E, H, -1),
           "residual": None if res is None else res.reshape(T, H)}
    fw = FN.forward64(inp, node.t["ids"], node.K, node.norm, node.scaling, node.hf, node.scoring, rounded=True)
    loss = FN.check_loss(out.reshape(T, H), fw["out"])
    if loss is not None:
        r["loss sum(out^2)"] = loss / FN.LOSS_REL
    _note(r)
    return r


def moe_case(T, H, I, E, K, opts, *, seed=0, residual=True, replay=None, route="out", flat=False, gate_bf16=False,
             shape=None, strided_res=False):
    g = _gen(seed + 1)
    x = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    res = None
    if residual:
        res = torch.randn(H, T, generator=g, device=DEV).to(torch.bfloat16).T if strided_res else \
            torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    go = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    if shape is not None:  # reshape keeps the strided residual a non-contiguous view
        x, go = x.view(shape), go.view(shape)
        res = None if res is None else res.reshape(shape)
    gw, w13, w2 = weights(H, I, E, seed, flat, gate_bf16)
    node, out, rr, gr, g_out, g_lg, g_rw = twice(run_moe, x, res, gw, w13, w2, K, opts, replay, route, go)
    check_moe(node, out, gr, g_out, g_lg, g_rw, x, res, gw, w13, w2, opts, replay, gate_bf16)
    return node, gr


SOFTMAX = dict(norm_topk_prob=True, router_scaling_factor=1.0, hidden_factor=1.0, scoring_func="softmax")
SIGMOID = dict(norm_topk_prob=False, router_scaling_factor=2.5, hidden_factor=0.5, scoring_func="sigmoid")


# ---- FusedMoEFunction ------------------------------------------------------------------------------------------------


def test_c2():
    """T = 8192, H = 2048, I = 768, E = 8, K = 2 (the benchmark's shape): one-launch gate + route, fused router-gate
    backward, paired dW; residual, z-loss and balancing gradients, flat weights as the layer holds them."""
    moe_case(8192, 2048, 768, 8, 2, SOFTMAX, route="all", flat=True)


def test_qwen3_30b_a3b():
    """E = 128, K = 8: two-call gate and router, two-call router and gate backward; sigmoid unnormalised at scaling
    2.5, hidden_factor 0.5, no residual, a bf16 gate parameter."""
    moe_case(1024, 2048, 768, 128, 8, SIGMOID, seed=1, residual=False, route="all", gate_bf16=True)


@pytest.mark.parametrize("replayed", [False, True])
def test_wide_hidden_two_call_gate(replayed):
    """H = 4224 > 4096 at E = 8: the two-call gate with the router (xtb_router_greedy_dispatch) or its replay entry,
    the fused backward."""
    replay = replay_ids(256, 8, 2, "random", 2) if replayed else None
    moe_case(256, 4224, 256, 8, 2, SOFTMAX, seed=2, replay=replay, route="all")


def test_split_weight_gradients():
    """I = 384, H = 1024: I % 256 != H % 256, so xtb_group_gemm_tn_pair runs as two launches; router_weights-only
    gradient, x as [B, S, H], a non-contiguous residual."""
    moe_case(512, 1024, 384, 8, 2, SOFTMAX, seed=3, route="rw", shape=(2, 256, 1024), strided_res=True)


@pytest.mark.parametrize("T", [1, 7, 33, 255])
@pytest.mark.parametrize("E,K", [(8, 2), (128, 8)])
def test_token_tails(T, E, K):
    """T tails at both gate paths; at E = 128 the routing is the router's own at T = 1 and 33, replayed with ids
    repeated in a row at T = 7 and 255."""
    if E == 8:
        moe_case(T, 256, 128, E, K, SOFTMAX, seed=T, route="all")
    else:
        replay = replay_ids(T, E, K, "dup", T) if T in (7, 255) else None
        moe_case(T, 256, 128, E, K, SIGMOID, seed=T, residual=False, replay=replay, route="all")


@pytest.mark.parametrize("pattern", ["random", "last", "expert0_empty", "half_empty", "dup"])
def test_replayed_routing(pattern):
    """Replayed ids: every token to the last expert (one expert holds all M rows), expert 0 empty, half the experts
    empty, the same id twice in a row.  Options alternate: softmax with residual and hidden_factor 1, sigmoid without
    residual at hidden_factor 0.5; the routes alternate too."""
    T, E, K = 300, 8, 2
    i = ["random", "last", "expert0_empty", "half_empty", "dup"].index(pattern)
    opts = SOFTMAX if i % 2 == 0 else SIGMOID
    moe_case(T, 512, 256, E, K, opts, seed=10 + i, residual=i % 2 == 0, replay=replay_ids(T, E, K, pattern, i),
             route=["out", "all", "rw"][i % 3], flat=i % 2 == 1)


def test_grad_sink():
    """GRAD_SINK set: the expert weight gradients land in the sink's buffers, bit-equal to a run without it.  Every
    backward gets fresh NaN-filled buffers, so the two runs' gradients are compared across separate memory."""
    from xtuner_b200 import fused

    T, H, I, E, K = 300, 512, 256, 8, 2
    _, plain = moe_case(T, H, I, E, K, SOFTMAX, seed=20, route="all")
    sinks = []

    def sink():
        sinks.append((torch.full((E * 2 * I * H,), float("nan"), dtype=torch.bfloat16, device=DEV),
                      torch.full((E * H * I,), float("nan"), dtype=torch.bfloat16, device=DEV)))
        return sinks[-1]

    fused.GRAD_SINK = sink
    try:
        _, sunk = moe_case(T, H, I, E, K, SOFTMAX, seed=20, route="all")
    finally:
        fused.GRAD_SINK = None
    assert len(sinks) == 2  # one backward per run of twice()
    for k in plain:
        _bits(plain[k], sunk[k], f"{k} with GRAD_SINK")
    assert sunk["g_w13"].data_ptr() == sinks[0][0].data_ptr() and sunk["g_w2"].data_ptr() == sinks[0][1].data_ptr()


@pytest.mark.parametrize("E,K", [(8, 2), (128, 8)])
@pytest.mark.parametrize("block", [False, True])
def test_no_tokens(E, K, block):
    """T = 0 (a micro-batch that brings no tokens): empty outputs, zero weight gradients, zero tokens_per_expert, for
    the layer node with a residual and for the block node with its norm weight."""
    from tests import norm_combine_reference as NC
    from xtuner_b200.fused import fused_moe, fused_moe_block

    H, I = 256, 128
    gw, w13, w2 = weights(H, I, E, 0)
    x = torch.empty(0, H, dtype=torch.bfloat16, device=DEV).requires_grad_(True)
    other = NC.norm_weight(H, 0, DEV) if block else torch.empty(0, H, dtype=torch.bfloat16, device=DEV)
    other.requires_grad_(True)
    ps = [t.clone().requires_grad_(True) for t in (gw, w13, w2)]
    out, rr = fused_moe_block(x, other, 1e-6, *ps, top_k=K) if block else fused_moe(x, other, *ps, top_k=K)
    assert out.shape == (0, H) and rr["logits"].shape == (0, E) and rr["topk_ids"].shape == (0, K)
    assert torch.equal(rr["topkens_per_expert"], torch.zeros(E, dtype=torch.int64, device=DEV))
    g_lg = torch.zeros(0, E, device=DEV)
    grads = torch.autograd.grad([out, rr["logits"]], [x, other] + ps, [torch.zeros_like(out), g_lg])
    assert grads[0].shape == (0, H) and grads[1].shape == other.shape
    for g in grads[1 if block else 2:]:
        assert bool((g == 0).all()), "a weight gradient is not zero at T = 0"


# ---- FusedMoEBlockFunction -------------------------------------------------------------------------------------------


def run_block(h, nw, gw, w13, w2, K, go, opts, need_nw=True, replay=None, route="out"):
    from xtuner_b200.fused import _FUSED_NORM_H, fused_moe_block

    hl = h.detach().clone().requires_grad_(True)
    nl = nw.detach().clone().requires_grad_(need_nw)
    ps = [t.detach().clone().requires_grad_(True) for t in (gw, w13, w2)]
    out, rr = fused_moe_block(hl, nl, 1e-6, *ps, top_k=K, rollout_routed_experts=replay, **opts)
    H = h.shape[-1]
    kind = "block" if H in _FUSED_NORM_H else "fallback"
    node = FN.from_autograd(out, rr["logits"], kind=kind, h_in=hl, norm_w=nl)
    g_lg, g_rw = route_grads(route, rr["logits"], rr["router_weights"], rr["topkens_per_expert"], K)
    outs, gos = ([out], [go]) if route != "rw" else ([], [])
    for o, g in ((rr["logits"], g_lg), (rr["router_weights"], g_rw)):
        if g is not None:
            outs.append(o), gos.append(g)
    wrt = [hl] + ([nl] if need_nw else []) + ps
    g = torch.autograd.grad(outs, wrt, gos)
    names = ["g_h"] + (["g_norm_w"] if need_nw else []) + ["g_gate_w", "g_w13", "g_w2"]
    g_out = go if route != "rw" else torch.zeros_like(go)
    return node, out.detach(), rr, dict(zip(names, g)), g_out, g_lg, g_rw


SOFTMAX_HF = dict(SOFTMAX, hidden_factor=0.5)
BLOCK_CASES = {  # H: (T, I, options, gradient route, replayed ids)
    256: (300, 256, SOFTMAX, "out", None),
    512: (300, 256, SIGMOID, "all", None),
    1024: (300, 256, SIGMOID, "rw", "random"),
    2048: (8192, 768, SOFTMAX_HF, "all", None),
    3072: (300, 256, SIGMOID, "all", "dup"),
}


@pytest.mark.parametrize("H", list(BLOCK_CASES))
def test_block(H):
    """The fused norm at every H it serves, H = 3072 through F.rms_norm and fused_moe.  Options vary by H: softmax
    normalised, sigmoid unnormalised at scaling 2.5 and hidden_factor 0.5, softmax at hidden_factor 0.5 (the benchmark's
    shape); gradients through out only, through out, logits and router_weights, or through router_weights only;
    replayed random ids and ids repeated in a row.  The norm weight is fp32 and not bf16-representable; a second run
    without its gradient gives the other gradients bit for bit."""
    from tests import norm_combine_reference as NC

    T, I, opts, route, pattern = BLOCK_CASES[H]
    E, K = 8, 2
    g = _gen(H)
    h = (torch.randn(T, H, generator=g, device=DEV) * 2).to(torch.bfloat16)
    nw = NC.norm_weight(H, H, DEV)
    go = torch.randn(T, H, generator=g, device=DEV).to(torch.bfloat16)
    gw, w13, w2 = weights(H, I, E, H)
    replay = None if pattern is None else replay_ids(T, E, K, pattern, H)
    node, out, rr, gr, g_out, g_lg, g_rw = twice(run_block, h, nw, gw, w13, w2, K, go, opts, replay=replay, route=route)
    r = FN.check_forward(node, replay)
    r.update(FN.check_backward(node, gr, g_out, g_lg, g_rw))
    fw = FN.forward64({"h_in": h, "norm_w": nw, "gate_w": gw, "w13": w13, "w2": w2}, node.t["ids"], K, node.norm,
                      node.scaling, node.hf, node.scoring, rounded=True)
    r["loss sum(out^2)"] = FN.check_loss(out, fw["out"]) / FN.LOSS_REL  # T H >= 2^14 at every H here
    _note({(f"{k} (fallback)" if node.kind == "fallback" else k): v for k, v in r.items()})
    gr2 = run_block(h, nw, gw, w13, w2, K, go, opts, need_nw=False, replay=replay, route=route)[3]
    assert "g_norm_w" not in gr2
    for k in gr2:
        _bits(gr[k], gr2[k], f"{k} without a norm weight gradient")


def test_fused_norm_and_fallback_differ_by_at_most_one_ulp_of_x():
    """On the same inputs the fused norm (bf16(h rstd w), fp32 w) and the composition the block falls back to
    (F.rms_norm with w cast to bf16) give x at most one bf16 ulp apart, element by element.  Which of the two is
    right is not settled here: each is pinned to its own restatement by test_block."""
    import torch.nn.functional as F

    from tests import norm_combine_reference as NC
    from xtuner_b200.fused import fused_moe_block

    T, H, I, E, K = 300, 1024, 256, 8, 2
    g = _gen(5)
    h = (torch.randn(T, H, generator=g, device=DEV) * 2).to(torch.bfloat16)
    nw = NC.norm_weight(H, 5, DEV)
    gw, w13, w2 = weights(H, I, E, 5)
    out, rr = fused_moe_block(h.requires_grad_(True), nw, 1e-6, gw, w13, w2, top_k=K)
    x_fused = FN.from_autograd(out, rr["logits"], kind="block").t["x"]
    x_fb = F.rms_norm(h.detach(), (H,), nw.to(torch.bfloat16), 1e-6)
    d = G.ulp_distance(x_fused, x_fb)
    print(f"fused_node_edges: fused norm vs F.rms_norm: {int((d > 0).sum())} of {d.numel()} elements one ulp apart")
    assert int(d.max()) <= 1
