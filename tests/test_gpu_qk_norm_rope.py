"""The fused q/k RMSNorm + rotary embedding kernels (``csrc/qk_norm_rope.cu``) on an H100, against the exact restatements
and float64 references of ``tests/qk_norm_rope_reference.py``:

* forward outputs bit-exact given the kernel's own rstd, and rstd within its fp64 bound;
* the gradient at the norm output exact, seen directly where there is no norm (dx = gn);
* dx by the near-tie checker (every mismatch a near tie, no fraction tolerated), dw within its bound;
* the Qwen3-30B-A3B attention input (Hq 32, Hkv 4, D 128) at T = 8192, D = 64 and 256, T = 1, a T that is not a multiple
  of the CTA's token group, ``with_gate`` strides, no norm, and rows from 2^-60 to 2^40, all-zero and eps-dominated;
* 64-bit addressing (T Hq D > 2^31), run-to-run identical bits, CUDA-graph replay, ``opcheck`` on both custom ops;
* with the reference package present: its ``MultiHeadAttention`` with and without the plugin, and its q/k steps under
  ``torch.compile(fullgraph=True)``."""
import math
import os

import pytest
import torch

from tests import qk_norm_rope_reference as R
from tests.gpu_harness import sm_count
from tests.norm_combine_reference import assert_bits_equal, check_bound, check_near_tie, norm_rows, norm_weight, rstd_rel

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "xtuner", "v1"))
EPS = 1e-6


def _cos_sin(T: int, D: int, seed: int):
    """the reference RotaryEmbedding's arithmetic (rope_theta 1e6) over packed documents of random lengths"""
    g = torch.Generator().manual_seed(seed)
    pos, n = [], 0
    while n < T:
        L = int(torch.randint(1, 4097, (1,), generator=g))
        pos.append(torch.arange(min(L, T - n)))
        n += L
    pos = torch.cat(pos).to(DEV).float()
    inv = 1.0 / (1e6 ** (torch.arange(0, D, 2, dtype=torch.int64, device=DEV).float() / D))
    emb = torch.cat([pos[:, None] * inv[None]] * 2, dim=-1)
    return emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)


def _inputs(T, Hq, Hkv, D, seed, gate=False):
    """q [T, Hq, D] (a view with head stride 2D when ``gate``) and k with norm_rows magnitudes, cos, sin, fp32 weights"""
    q_full = norm_rows(T * Hq, 2 * D if gate else D, seed, DEV).view(T, Hq, -1)
    k = norm_rows(T * Hkv, D, seed + 1, DEV).view(T, Hkv, D)
    cos, sin = _cos_sin(T, D, seed)
    return q_full[..., :D], k, cos, sin, norm_weight(D, seed + 2, DEV), norm_weight(D, seed + 3, DEV)


def _fwd(q, k, cos, sin, wq, wk):
    from xtuner_b200 import ops

    return ops._qk_norm_rope_op(q, k, cos, sin, wq, wk, EPS)


def _bwd(gq, gk, q, k, cos, sin, wq, wk, rq, rk):
    from xtuner_b200 import ops

    return ops._qk_norm_rope_bwd_op(gq, gk, q, k, cos, sin, wq, wk, rq, rk, wq is not None)


SHAPES = [  # T, Hq, Hkv, D, norm, with_gate
    pytest.param(8192, 32, 4, 128, True, False, id="qwen3_30b_a3b_T8192"),
    pytest.param(1000, 8, 2, 64, True, False, id="D64"),
    pytest.param(1000, 8, 2, 256, True, False, id="D256"),
    pytest.param(1, 32, 4, 128, True, False, id="T1"),
    pytest.param(1003, 16, 4, 128, True, False, id="T_ragged_group"),
    pytest.param(515, 32, 4, 128, True, True, id="with_gate"),
    pytest.param(777, 32, 4, 128, False, False, id="no_norm"),
    pytest.param(777, 8, 2, 256, False, True, id="no_norm_gate_D256"),
]


@pytest.mark.parametrize("T,Hq,Hkv,D,norm,gate", SHAPES)
def test_forward_and_backward_against_the_references(T, Hq, Hkv, D, norm, gate):
    q, k, cos, sin, wq, wk = _inputs(T, Hq, Hkv, D, seed=T + D, gate=gate)
    if not norm:
        wq = wk = None
    out_q, out_k, rq, rk = _fwd(q, k, cos, sin, wq, wk)
    g = torch.Generator(device=DEV).manual_seed(5)
    g_full = torch.randn((T, Hq, 2 * D if gate else D), generator=g, device=DEV).to(torch.bfloat16)
    gq, gk = g_full[..., :D], torch.randn((T, Hkv, D), generator=g, device=DEV).to(torch.bfloat16)
    dx_q, dx_k, dw = _bwd(gq, gk, q, k, cos, sin, wq, wk, rq, rk)
    torch.cuda.synchronize()
    n_cta = R.bwd_ctas(T, sm_count())
    worst = {}
    for i, (x, out, rstd, w, gg, dx) in enumerate(((q, out_q, rq, wq, gq, dx_q), (k, out_k, rk, wk, gk, dx_k))):
        tag = "qk"[i]
        assert_bits_equal(out, R.forward(x, cos, sin, rstd if norm else None, w), f"out_{tag}")
        gn = R.grad_n(gg, cos, sin)
        if not norm:
            assert_bits_equal(dx, gn, f"dx_{tag} (= gn)")
            continue
        r64 = R.rstd_fp64(x, EPS)
        worst[f"rstd_{tag}"] = check_bound(rstd, r64, rstd_rel(D) * r64, f"rstd_{tag}")
        worst[f"dx_{tag}"] = check_near_tie(dx, *R.dx_ref(gn, x, rstd, w), f"dx_{tag}")[0]
        worst[f"dw_{tag}"] = check_bound(dw[i], *R.dw_ref(gn, x, rstd, n_cta), f"dw_{tag}")
    print(f"T={T} Hq={Hq} Hkv={Hkv} D={D} norm={norm} gate={gate}: largest |err|/bound " +
          ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_64bit_offsets_first_and_last_tokens():
    T, Hq, Hkv, D = (1 << 19) + 5, 32, 4, 128  # T Hq D = 2^31 + 20480 elements
    assert T * Hq * D > 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(11)
    q = torch.randn((T, Hq, D), generator=g, device=DEV, dtype=torch.bfloat16)
    k = torch.randn((T, Hkv, D), generator=g, device=DEV, dtype=torch.bfloat16)
    cos, sin = _cos_sin(T, D, 11)
    wq, wk = norm_weight(D, 12, DEV), norm_weight(D, 13, DEV)
    out_q, out_k, rq, rk = _fwd(q, k, cos, sin, wq, wk)
    torch.cuda.synchronize()
    for sl in (slice(0, 3), slice(T - 3, T)):
        assert_bits_equal(out_q[sl], R.forward(q[sl], cos[sl], sin[sl], rq[sl], wq), f"out_q[{sl}]")
        assert_bits_equal(out_k[sl], R.forward(k[sl], cos[sl], sin[sl], rk[sl], wk), f"out_k[{sl}]")
        r64 = R.rstd_fp64(q[sl], EPS)
        check_bound(rq[sl], r64, rstd_rel(D) * r64, "rstd_q")


def _step(q, k, cos, sin, wq, wk, gq, gk):
    from xtuner_b200 import ops

    qq, kk = q.clone().requires_grad_(True), k.clone().requires_grad_(True)
    wwq, wwk = wq.clone().requires_grad_(True), wk.clone().requires_grad_(True)
    oq, ok = ops.qk_norm_rope(qq, kk, cos, sin, wwq, wwk, EPS)
    torch.autograd.backward((oq, ok), (gq, gk))
    return oq, ok, qq.grad, kk.grad, wwq.grad, wwk.grad


def test_two_calls_give_identical_bits():
    q, k, cos, sin, wq, wk = _inputs(4099, 32, 4, 128, seed=3)
    gq, gk = torch.randn_like(q), torch.randn_like(k)
    a, b = _step(q, k, cos, sin, wq, wk, gq, gk), _step(q, k, cos, sin, wq, wk, gq, gk)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int16) if x.dtype == torch.bfloat16 else x.view(torch.int32),
                           y.view(torch.int16) if y.dtype == torch.bfloat16 else y.view(torch.int32))


def test_cuda_graph_replay_equals_the_eager_call():
    from xtuner_b200 import ops

    T, Hq, Hkv, D = 2048, 32, 4, 128
    q, k, cos, sin, wq, wk = _inputs(T, Hq, Hkv, D, seed=9)
    gq, gk = torch.randn_like(q), torch.randn_like(k)

    def step():
        oq, ok, rq, rk = ops._qk_norm_rope_op(q, k, cos, sin, wq, wk, EPS)
        return (oq, ok) + ops._qk_norm_rope_bwd_op(gq, gk, q, k, cos, sin, wq, wk, rq, rk, True)

    eager = [t.clone() for t in step()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()  # warm-up on a side stream, as torch.cuda.graph asks of work it captures
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(static, eager):
        assert torch.equal(a, b)


def test_opcheck_both_custom_ops():
    from xtuner_b200 import ops

    q, k, cos, sin, wq, wk = _inputs(64, 8, 2, 128, seed=21, gate=True)
    torch.library.opcheck(ops._qk_norm_rope_op, (q, k, cos, sin, wq, wk, EPS))
    torch.library.opcheck(ops._qk_norm_rope_op, (q, k, cos, sin, None, None, EPS))
    _, _, rq, rk = ops._qk_norm_rope_op(q, k, cos, sin, wq, wk, EPS)
    gq, gk = torch.randn_like(q), torch.randn_like(k)
    torch.library.opcheck(ops._qk_norm_rope_bwd_op, (gq, gk, q, k, cos, sin, wq, wk, rq, rk, True))


# ---- the reference's attention with and without the plugin -----------------------------------------------------------


def _rel(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-30))


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref absent (oracle/make_ref.py places the reference package there)")
@pytest.mark.parametrize("compiled", [False, True])
def test_plugin_on_the_reference_attention(compiled):
    from tests.golden import ref_shim
    from xtuner_b200 import _capi, plugin

    ref_shim.REFERENCE_ROOT = os.path.join(ROOT, "oracle", "_ref")
    ref_shim.import_reference()
    from xtuner.v1.data_proto import SequenceContext
    from xtuner.v1.module.attention import MHAConfig

    torch.manual_seed(0)
    S, hidden = 2048, 2048
    attn = MHAConfig(num_attention_heads=32, num_key_value_heads=4, head_dim=128, qk_norm=True,
                     attn_impl="eager_attention").build(hidden_size=hidden, layer_idx=0)
    with torch.no_grad():
        for p in attn.parameters():
            p.copy_(torch.randn_like(p) * hidden ** -0.5 if p.dim() > 1 else 1.0 + 0.3 * torch.randn_like(p))
    attn = attn.to(DEV, torch.bfloat16)
    docs = (700, 800, S - 1500)  # packed documents: position ids restart at each
    seq_ctx = SequenceContext.from_input_ids(input_ids=tuple(torch.zeros(1, n, dtype=torch.long) for n in docs), device=DEV)
    pos = seq_ctx.position_ids.view(-1).to(DEV)
    inv = 1.0 / (1e6 ** (torch.arange(0, 128, 2, dtype=torch.int64, device=DEV).float() / 128))
    emb = torch.cat([pos[:, None].float() * inv[None]] * 2, -1)[None]
    cos, sin = emb.cos().to(torch.bfloat16), emb.sin().to(torch.bfloat16)
    h = (torch.randn(1, S, hidden, device=DEV)).to(torch.bfloat16)
    gout = torch.randn(1, S, hidden, device=DEV).to(torch.bfloat16)
    if compiled:
        # the q/k steps of MultiHeadAttention.forward (mha.py:335-363) under fullgraph: the reference's eager_attention
        # builds its mask with data-dependent shapes that inductor does not take, so the attention stays outside
        def qk(x):
            q = attn.q_norm(attn.q_proj(x).view(1, S, -1, 128)).transpose(1, 2)
            k = attn.k_norm(attn.k_proj(x).view(1, S, -1, 128)).transpose(1, 2)
            return attn.apply_rotary_emb(q, k, cos, sin)

        qk = torch.compile(qk, fullgraph=True)
        gq = torch.randn(1, 32, S, 128, device=DEV).to(torch.bfloat16)
        gk = torch.randn(1, 4, S, 128, device=DEV).to(torch.bfloat16)

    def run():
        attn.zero_grad(set_to_none=True)
        x = h.clone().requires_grad_(True)
        if compiled:
            oq, ok = qk(x)
            torch.autograd.backward((oq, ok), (gq, gk))
            out = torch.cat([oq.reshape(-1), ok.reshape(-1)])
        else:
            out = attn(x, (cos, sin), seq_ctx)["projected_output"]
            out.backward(gout)
        return [out.detach(), x.grad] + [getattr(attn, m).weight.grad.clone() for m in ("q_proj", "k_proj", "q_norm", "k_norm")]

    lib = _capi.load()
    want = run()
    n0 = lib.xtb_launch_count()
    assert plugin.install_qk_norm_rope(attn) == 1
    try:
        if compiled:
            torch._dynamo.reset()
        got = run()
    finally:
        plugin.uninstall_qk_norm_rope(attn)
    assert lib.xtb_launch_count() > n0, "the installed path did not run xtb_qk_norm_rope"
    names = ["out", "dh", "q_proj.w", "k_proj.w", "q_norm.w", "k_norm.w"]
    rels = {n: _rel(a, b) for n, a, b in zip(names, got, want)}
    print(f"plugin on MultiHeadAttention (compiled={compiled}): largest |err| / max|ref|: " +
          ", ".join(f"{n} {r:.2e}" for n, r in rels.items()))
    for n, r in rels.items():
        assert math.isfinite(r) and r <= 2e-2, f"{n}: {r}"
