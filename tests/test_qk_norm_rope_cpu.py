"""CPU coverage of the fused q/k RMSNorm + rotary embedding (``ops.qk_norm_rope``, ``plugin.install_qk_norm_rope``):

* the restatement in ``tests/qk_norm_rope_reference.py`` against fixtures made by the reference's own ``RMSNorm``,
  ``apply_rotary_pos_emb_cuda`` and ``RotaryEmbedding`` (``tests/golden/make_qk_norm_rope_golden.py``): outputs and the
  gradient at the norm outputs bit for bit, input and weight gradients within their float64 bounds;
* the shipped host layers (custom ops, autograd node, strides, weight dtypes) over a host-memory emulation of the two
  C entries written from the header's contract (``QKNormRopeEmulatedLib``, on top of ``tests/cabi_emulator.py``);
* the plugin on the reference's ``MultiHeadAttention``: which layers it takes, per-call fallback, exact restore.

The kernels themselves are covered on an H100 by ``tests/test_gpu_qk_norm_rope.py``."""
import os
import sys

import pytest
import torch

from tests import qk_norm_rope_reference as R
from tests.cabi_emulator import EmulatedLib, _view
from tests.conftest import load_golden
from tests.norm_combine_reference import BF16_U, check_bound, check_near_tie, rstd_rel

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = ["d128", "d64", "d128_bf16w", "d128_gate", "d128_nonorm"]


@pytest.fixture(scope="module")
def gold():
    return load_golden("qk_norm_rope")


def _case(gold, name):
    """(q [T, Hq, D] view (the with_gate half of the stored projection), k, cos, sin, w_q, w_k)"""
    k = gold[f"{name}.k"]
    D = k.shape[-1]
    return (gold[f"{name}.q"][..., :D], k, gold[f"{name}.cos"], gold[f"{name}.sin"], gold.get(f"{name}.w_q"),
            gold.get(f"{name}.w_k"))


def _dw_bound(dw64, bound, dtype):
    """a bf16 weight's gradient is the fp32 sum rounded once more"""
    return bound * 1.01 + (BF16_U * dw64.abs() if dtype == torch.bfloat16 else 0)


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_the_reference(gold, name):
    q, k, cos, sin, w_q, w_k = _case(gold, name)
    eps = gold["eps"]
    for x, w, tag in ((q, w_q, "q"), (k, w_k, "k")):
        rstd = R.rstd_torch(x, eps) if w is not None else None
        assert torch.equal(R.forward(x, cos, sin, rstd, w), gold[f"{name}.out_{tag}"]), f"out_{tag}"
        gn = R.grad_n(gold[f"{name}.g_{tag}"], cos, sin)
        D = x.shape[-1]
        dx = gold[f"{name}.dx_{tag}"][..., :D]
        if w is None:
            assert torch.equal(gn, dx), f"dx_{tag} = gn without the norm"
            continue
        assert torch.equal(gn, gold[f"{name}.gn_{tag}"]), f"gn_{tag}"
        ref64 = R.rstd_fp64(x, eps)
        check_bound(rstd, ref64, rstd_rel(D) * ref64, f"rstd_{tag}")
        check_near_tie(dx, *R.dx_ref(gn, x, rstd, w), f"dx_{tag}")
        dw64, bound = R.dw_ref(gn, x, rstd, n_cta=1)
        dw = gold[f"{name}.dw_{tag}"]
        check_bound(dw.float(), dw64, _dw_bound(dw64, bound, dw.dtype), f"dw_{tag}")
    if name == "d128_gate":  # the gate half of the projection gets nothing from this step
        assert gold[f"{name}.dx_q"][..., q.shape[-1]:].count_nonzero() == 0


# ---- host layers over the emulated entries -------------------------------------------------------------------------------


class QKNormRopeEmulatedLib(EmulatedLib):
    """``xtb_qk_norm_rope`` / ``xtb_qk_norm_rope_bwd`` computed on host memory as the header states them: the
    restatement for the forward and the gradient at the norm output, plain fp32 torch for the norm backward."""

    @staticmethod
    def _rows(addr, T, H, D, st, sh):
        """bf16 [T, H, D] view with token stride ``st`` and head stride ``sh`` (elements) of host memory at ``addr``"""
        flat = _view(addr, torch.bfloat16, (T - 1) * st + (H - 1) * sh + D)
        return flat.as_strided((T, H, D), (st, sh, 1))

    def xtb_qk_norm_rope_bwd_workspace_bytes(self, T, D):
        return self._real.xtb_qk_norm_rope_bwd_workspace_bytes(T, D)

    def xtb_qk_norm_rope(self, q, q_st, q_sh, k, k_st, k_sh, cos, sin, w_q, w_k, eps, T, Hq, Hkv, D, out_q, out_k, rstd_q,
                         rstd_k, stream):
        self.calls.append("xtb_qk_norm_rope")
        if D not in (64, 128, 256) or (w_q is None) != (w_k is None):
            return 1
        if T == 0:
            return 0
        c, s = _view(cos, torch.bfloat16, T, D), _view(sin, torch.bfloat16, T, D)
        for x, st, sh, H, w, out, rstd in ((q, q_st, q_sh, Hq, w_q, out_q, rstd_q), (k, k_st, k_sh, Hkv, w_k, out_k, rstd_k)):
            xv = self._rows(x, T, H, D, st, sh)
            r = None
            if w is not None:
                r = R.rstd_torch(xv, eps)
                _view(rstd, torch.float32, T, H).copy_(r)
            _view(out, torch.bfloat16, T, H, D).copy_(R.forward(xv, c, s, r, None if w is None else _view(w, torch.float32, D)))
        return 0

    def xtb_qk_norm_rope_bwd(self, g_q, gq_st, gq_sh, g_k, gk_st, gk_sh, q, q_st, q_sh, k, k_st, k_sh, cos, sin, w_q, w_k,
                             rstd_q, rstd_k, T, Hq, Hkv, D, dx_q, dx_k, dw, ws, stream):
        self.calls.append("xtb_qk_norm_rope_bwd")
        if D not in (64, 128, 256) or (w_q is None) != (w_k is None) or (dw is not None and (w_q is None or ws is None)):
            return 1
        dws = []
        c, s = (_view(cos, torch.bfloat16, T, D), _view(sin, torch.bfloat16, T, D)) if T else (None, None)
        for gp, gst, gsh, x, st, sh, H, w, rstd, dx in ((g_q, gq_st, gq_sh, q, q_st, q_sh, Hq, w_q, rstd_q, dx_q),
                                                         (g_k, gk_st, gk_sh, k, k_st, k_sh, Hkv, w_k, rstd_k, dx_k)):
            if T == 0:
                dws.append(torch.zeros(D))
                continue
            gn = R.grad_n(self._rows(gp, T, H, D, gst, gsh), c, s)
            if w is None:
                _view(dx, torch.bfloat16, T, H, D).copy_(gn)
                continue
            xv, r, wv = self._rows(x, T, H, D, st, sh).float(), _view(rstd, torch.float32, T, H)[..., None], _view(w, torch.float32, D)
            wg = gn.float() * wv
            c_term = (wg * xv).sum(-1, keepdim=True) * r * r / D
            _view(dx, torch.bfloat16, T, H, D).copy_(((wg - xv * c_term) * r).to(torch.bfloat16))
            dws.append((gn.float() * r * xv).sum((0, 1)))
        if dw is not None:
            _view(dw, torch.float32, 2, D).copy_(torch.stack(dws))
        return 0


@pytest.fixture
def emu(monkeypatch):
    from xtuner_b200 import _capi, ops

    lib = QKNormRopeEmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    monkeypatch.setattr(ops, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "_scratch", lambda tag, n, dev: torch.empty(max(int(n), 16), dtype=torch.uint8))
    return lib


@pytest.mark.parametrize("name", CASES)
def test_op_gives_the_reference_forward_and_routes_the_gradients(gold, emu, name):
    from xtuner_b200 import ops

    D = gold[f"{name}.k"].shape[-1]
    q_full = gold[f"{name}.q"].clone().requires_grad_(True)  # [T, Hq, D] or, with_gate, [T, Hq, 2D]
    k = gold[f"{name}.k"].clone().requires_grad_(True)
    _, _, cos, sin, w_q, w_k = _case(gold, name)
    wq = None if w_q is None else w_q.clone().requires_grad_(True)
    wk = None if w_k is None else w_k.clone().requires_grad_(True)
    q = q_full[..., :D]
    out_q, out_k = ops.qk_norm_rope(q, k, cos, sin, wq, wk, gold["eps"])
    assert out_q.is_contiguous() and out_k.is_contiguous()
    assert torch.equal(out_q, gold[f"{name}.out_q"]) and torch.equal(out_k, gold[f"{name}.out_k"])
    assert emu.calls == ["xtb_qk_norm_rope"]
    (out_q.float() * gold[f"{name}.g_q"].float()).sum().add((out_k.float() * gold[f"{name}.g_k"].float()).sum()).backward()
    assert emu.calls == ["xtb_qk_norm_rope", "xtb_qk_norm_rope_bwd"]
    for x, g, tag in ((q_full, q_full.grad, "q"), (k, k.grad, "k")):
        assert g.shape == x.shape and g.dtype == torch.bfloat16
        want = gold[f"{name}.dx_{tag}"]
        if w_q is None:
            assert torch.equal(g, want)
        else:
            xx = x.detach()[..., :D]
            gn = gold[f"{name}.gn_{tag}"]
            check_near_tie(g[..., :D], *R.dx_ref(gn, xx, R.rstd_torch(xx, gold["eps"]), gold[f"{name}.w_{tag}"]), f"dx_{tag}")
        if name == "d128_gate" and tag == "q":
            assert g[..., D:].count_nonzero() == 0
    if w_q is not None:
        for w, tag in ((wq, "q"), (wk, "k")):
            ref = gold[f"{name}.dw_{tag}"]
            assert w.grad.dtype == w.dtype == ref.dtype
            dw64, bound = R.dw_ref(gold[f"{name}.gn_{tag}"], _case(gold, name)[0 if tag == "q" else 1],
                                   R.rstd_torch(_case(gold, name)[0 if tag == "q" else 1], gold["eps"]), n_cta=1)
            check_bound(w.grad.float(), dw64, _dw_bound(dw64, bound, w.dtype), f"dw_{tag}")


def test_op_without_weight_grad_skips_dw_and_rejects_bad_shapes(gold, emu):
    from xtuner_b200 import _capi, ops

    q, k, cos, sin, w_q, w_k = _case(gold, "d128")
    qq = q.clone().requires_grad_(True)
    out_q, out_k = ops.qk_norm_rope(qq, k, cos, sin, w_q, w_k)
    out_q.float().sum().backward()  # k's output unused: its gradient enters as zeros
    assert qq.grad is not None and w_q.grad is None
    with pytest.raises(_capi.XtbError):
        ops.qk_norm_rope(q[..., :96], k[..., :96], cos[:, :96], sin[:, :96])
    with pytest.raises(ValueError):
        ops.qk_norm_rope(q, k, cos, sin, w_q, None)
    with pytest.raises(_capi.XtbError):
        ops.qk_norm_rope(q, k, cos[:-1], sin[:-1], w_q, w_k)


# ---- plugin on the reference's MultiHeadAttention -----------------------------------------------------------------------

sys.path.insert(0, os.path.join(HERE, "golden"))
import ref_shim  # noqa: E402


@pytest.fixture
def ref():
    if not ref_shim.reference_available():
        pytest.skip("no reference checkout found")
    ref_shim.apply_cpu_patches()
    import importlib

    return importlib.import_module("xtuner.v1.module.attention.mha")


def _attn(ref, seed=0, qk_norm=True, head_dim=64, norm_type="default", with_gate=False):
    from xtuner.v1.module.attention import MHAConfig

    torch.manual_seed(seed)
    cfg = MHAConfig(num_attention_heads=4, num_key_value_heads=2, head_dim=head_dim, qk_norm=qk_norm,
                    rms_norm_type=norm_type, with_gate=with_gate, attn_impl="eager_attention")
    attn = cfg.build(hidden_size=128, layer_idx=0)
    with torch.no_grad():
        for p in attn.parameters():
            p.copy_(torch.randn_like(p) * (0.2 if p.dim() > 1 else 1.0) + (1.0 if p.dim() == 1 else 0.0))
    return attn.to(torch.bfloat16)


def _run(attn, S=24):
    from types import SimpleNamespace

    from xtuner.v1.data_proto import SequenceContext

    torch.manual_seed(7)
    h = torch.randn(1, S, 128).to(torch.bfloat16).requires_grad_(True)
    ids = torch.zeros(1, S, dtype=torch.long)
    seq_ctx = SequenceContext.from_input_ids(input_ids=(ids,), device="cpu")
    cfg = SimpleNamespace(max_position_embeddings=4096, rope_parameters_cfg=None, rope_scaling_cfg=None, rope_theta=1e6,
                          head_dim=attn.head_dim)
    from xtuner.v1.module.rope.rope import RotaryEmbedding

    cos, sin = RotaryEmbedding(cfg).forward(h, seq_ctx.position_ids)
    attn.zero_grad(set_to_none=True)
    out = attn(h, (cos, sin), seq_ctx)["projected_output"]
    (out.float() * torch.linspace(-1, 1, out.numel()).view_as(out)).sum().backward()
    grads = {n: p.grad.clone() for n, p in attn.named_parameters() if p.grad is not None}
    return out.detach(), h.grad, grads


@pytest.fixture
def on_device(monkeypatch):
    from xtuner_b200 import plugin

    monkeypatch.setattr(plugin, "_on_device", lambda t: True)  # host tensors: the eligibility predicate's only device question


@pytest.mark.parametrize("with_gate", [False, True])
def test_plugin_runs_the_fused_op_in_the_reference_attention(ref, emu, on_device, with_gate):
    from xtuner_b200 import plugin

    attn = _attn(ref, with_gate=with_gate)
    want_out, want_dh, want_g = _run(attn)
    assert plugin.install_qk_norm_rope(attn) == 1
    try:
        out, dh, grads = _run(attn)
    finally:
        plugin.uninstall_qk_norm_rope(attn)
    assert emu.calls == ["xtb_qk_norm_rope", "xtb_qk_norm_rope_bwd"]
    assert torch.equal(out, want_out)  # the emulated forward has the reference's roundings
    assert set(grads) == set(want_g)
    for n, g in [("h", dh), *grads.items()]:
        w = want_dh if n == "h" else want_g[n]
        torch.testing.assert_close(g.float(), w.float(), rtol=2e-2, atol=2e-2 * float(w.abs().max()), msg=n)


def test_plugin_skips_ineligible_layers(ref):
    from xtuner.v1.ops.rotary_emb import apply_rotary_pos_emb_cuda_for_partial_rotary

    from xtuner_b200 import plugin

    partial = _attn(ref)
    partial.apply_rotary_emb = apply_rotary_pos_emb_cuda_for_partial_rotary
    layers = torch.nn.ModuleList([partial, _attn(ref, norm_type="zero_centered"), _attn(ref, head_dim=32), _attn(ref),
                                  _attn(ref, qk_norm=False)])
    assert plugin.install_qk_norm_rope(layers) == 2
    assert plugin.install_qk_norm_rope(layers) == 0  # installed layers are not wrapped twice
    assert [plugin._SAVED in vars(a) for a in layers] == [False, False, False, True, True]
    plugin.uninstall_qk_norm_rope(layers)


def test_plugin_falls_back_per_call(ref, emu):
    from xtuner.v1.ops.rotary_emb import apply_rotary_pos_emb_cuda

    from xtuner_b200 import plugin

    attn = _attn(ref)
    torch.manual_seed(3)
    q = torch.randn(2, 4, 8, 64).to(torch.bfloat16)
    k = torch.randn(2, 2, 8, 64).to(torch.bfloat16)
    cos, sin = torch.rand(2, 8, 64).to(torch.bfloat16), torch.rand(2, 8, 64).to(torch.bfloat16)
    want = apply_rotary_pos_emb_cuda(attn.q_norm(q), attn.k_norm(k), cos, sin)
    plugin.install_qk_norm_rope(attn)
    try:
        # host tensors (the predicate is not patched here), batch 2, and unsqueeze_dim=2 on [b, s, h, d] tensors
        got = attn.apply_rotary_emb(q, k, cos, sin)
        got2 = attn.apply_rotary_emb(q.transpose(1, 2), k.transpose(1, 2), cos, sin, unsqueeze_dim=2)
        assert attn.q_norm(q) is q  # the norm itself is a pass-through while installed
    finally:
        plugin.uninstall_qk_norm_rope(attn)
    assert emu.calls == []
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    for a, b in zip(got2, want):
        assert torch.equal(a.transpose(1, 2), b)


def test_plugin_restores_the_modules_exactly(ref):
    from xtuner_b200 import plugin

    attn = _attn(ref)
    cls_dict = dict(vars(type(attn)))
    before = {m: dict(vars(m)) for m in (attn, attn.q_norm, attn.k_norm)}
    keys = list(attn.state_dict())
    assert plugin.install_qk_norm_rope(attn) == 1
    assert list(attn.state_dict()) == keys
    assert "forward" in vars(attn.q_norm) and attn.apply_rotary_emb is not before[attn]["apply_rotary_emb"]
    plugin.uninstall_qk_norm_rope(attn)
    for m, d in before.items():
        assert dict(vars(m)) == d
    assert dict(vars(type(attn))) == cls_dict and list(attn.state_dict()) == keys
