"""CPU coverage of the lm_head cross-entropy (``ops.lm_head_cross_entropy``, ``plugin.install_lm_head_loss``):

* the plain-torch restatement in ``tests/lm_head_ce_reference.py`` against fixtures made by the reference's own
  ``LMHeadLossContext`` (``tests/golden/make_lm_head_ce_golden.py``), bit for bit, in modes "eager" and "chunk";
* the shipped host orchestration (chunk loop, bf16 ``dW`` accumulation, fp32 loss accumulation, ``grad_output``
  scaling, ``need_grad``) over a host-memory emulation of ``xtb_lm_head_ce`` written from the header's contract;
* the plugin's dispatch: eligible calls to ours, everything else to the reference's methods, and an exact restore.

The kernels themselves are covered on an H100 by ``tests/test_gpu_lm_head_ce.py``."""
import os
import sys

import pytest
import torch
from torch.nn import functional as F

from tests.cabi_emulator import EmulatedLib, _view
from tests.conftest import load_golden
from tests.lm_head_ce_reference import lm_head_ce

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def gold():
    g = load_golden("lm_head_ce")
    g["hidden"] = g["hidden"].view(-1, g["hidden"].shape[-1])
    g["labels"] = g["labels"].view(-1)
    return g


CASES = [("eager", "token"), ("eager", "sample"), ("chunk", "token"), ("chunk", "sample")]


@pytest.mark.parametrize("mode,reduction", CASES)
def test_reference_restatement_matches_the_reference_bit_for_bit(gold, mode, reduction):
    lw = gold[f"{mode}.{reduction}.loss_weight"]
    loss, dh, dw = lm_head_ce(gold["hidden"], gold["weight"], gold["labels"], lw, gold["ignore_index"],
                              None if mode == "eager" else gold["chunk_size"])
    assert torch.equal(loss, gold[f"{mode}.{reduction}.loss"])
    assert torch.equal(dh, gold[f"{mode}.{reduction}.dh"].view_as(dh))
    assert torch.equal(dw, gold[f"{mode}.{reduction}.dw"])


@pytest.mark.parametrize("mode", ["eager", "chunk"])
def test_reference_restatement_all_ignored(gold, mode):
    labels = torch.full_like(gold["labels"], gold["ignore_index"])
    lw = torch.zeros(labels.shape)
    loss, dh, dw = lm_head_ce(gold["hidden"], gold["weight"], labels, lw, gold["ignore_index"],
                              None if mode == "eager" else gold["chunk_size"])
    assert float(loss) == 0.0 and float(gold[f"{mode}.all_ignored.loss"]) == 0.0
    assert gold[f"{mode}.all_ignored.grad_nonzero"] == 0
    assert dh.count_nonzero() == 0 and dw.count_nonzero() == 0


# ---- host orchestration over an emulated xtb_lm_head_ce ------------------------------------------------------------------


class LMHeadEmulatedLib(EmulatedLib):
    """``xtb_lm_head_ce`` computed as the header states it, with the reference's own arithmetic for one chunk."""

    def xtb_lm_head_ce_workspace_bytes(self, T, V):
        return self._real.xtb_lm_head_ce_workspace_bytes(T, V)

    def xtb_lm_head_ce(self, h, w, labels, loss_weight, T, H, V, ignore_index, need_grad, z_or_G, ws, row_ce, loss, dh,
                       dw, stream):
        self.calls.append(("xtb_lm_head_ce", T, need_grad))
        assert ws is not None
        hh = _view(h, torch.bfloat16, T, H).clone().requires_grad_(True)
        ww = _view(w, torch.bfloat16, V, H).clone().requires_grad_(True)
        lab, lw = _view(labels, torch.int64, T), _view(loss_weight, torch.float32, T)
        with torch.enable_grad():
            z = F.linear(hh, ww)
            logits = z.float()
            if int((lab != ignore_index).sum()) == 0:
                ce, out = torch.zeros(T), logits.sum() * 0
            else:
                ce = F.cross_entropy(logits, lab, reduction="none", ignore_index=ignore_index)
                out = (ce * lw).sum()
            if need_grad:
                G, gh, gw = torch.autograd.grad(out, (z, hh, ww))
        _view(loss, torch.float32, 1).copy_(out.detach().view(1))
        _view(row_ce, torch.float32, T).copy_(ce.detach())
        _view(z_or_G, torch.bfloat16, T, V).copy_(G if need_grad else z.detach())
        if need_grad:
            _view(dh, torch.bfloat16, T, H).copy_(gh)
            _view(dw, torch.bfloat16, V, H).copy_(gw)
        return 0


@pytest.fixture
def emu(monkeypatch):
    from xtuner_b200 import _capi, ops

    lib = LMHeadEmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    monkeypatch.setattr(ops, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "_scratch", lambda tag, n, dev: torch.empty(max(int(n), 16), dtype=torch.uint8))
    return lib


def _ours(gold, lw, chunk, grad_output, labels=None):
    from xtuner_b200 import ops

    h = gold["hidden"].clone().requires_grad_(True)
    w = gold["weight"].clone().requires_grad_(True)
    loss = ops.lm_head_cross_entropy(h, w, gold["labels"] if labels is None else labels, lw, gold["ignore_index"], chunk)
    loss.backward(torch.tensor(grad_output))
    return loss.detach(), h.grad, w.grad


@pytest.mark.parametrize("grad_output", [1.0, 2.0 ** -3])
@pytest.mark.parametrize("mode,reduction", CASES)
def test_host_orchestration_gives_the_reference_bits(gold, emu, mode, reduction, grad_output):
    """Power-of-two loss gradients scale every rounding exactly, so both modes keep the reference's bits."""
    lw = gold[f"{mode}.{reduction}.loss_weight"]
    chunk = None if mode == "eager" else gold["chunk_size"]
    loss, dh, dw = _ours(gold, lw, chunk, grad_output)
    want = lm_head_ce(gold["hidden"], gold["weight"], gold["labels"], lw, gold["ignore_index"], chunk, grad_output)
    assert torch.equal(loss, want[0]) and torch.equal(dh, want[1]) and torch.equal(dw, want[2])
    if grad_output == 1.0:
        assert torch.equal(loss, gold[f"{mode}.{reduction}.loss"]) and torch.equal(dw, gold[f"{mode}.{reduction}.dw"])
    # chunks of 128, 128 and 44 rows: the ragged last chunk is its own call
    rows = [c[1] for c in emu.calls]
    assert rows == ([300] if chunk is None else [128, 128, 44]) and all(c[2] == 1 for c in emu.calls)


def test_chunk_dw_is_accumulated_in_bf16_in_chunk_order(gold, emu):
    lw = gold["chunk.token.loss_weight"]
    _, _, dw = _ours(gold, lw, 128, 1.0)
    parts = [lm_head_ce(gold["hidden"][s:s + 128], gold["weight"], gold["labels"][s:s + 128], lw.view(-1)[s:s + 128],
                        gold["ignore_index"])[2] for s in (0, 128, 256)]
    assert torch.equal(dw, (parts[0] + parts[1]) + parts[2])
    assert not torch.equal(dw, (parts[0].float() + parts[1].float() + parts[2].float()).to(torch.bfloat16)), \
        "inputs too tame: fp32 accumulation would give the same bits"


def test_no_grad_skips_the_gradients(gold, emu):
    from xtuner_b200 import ops

    lw = gold["eager.token.loss_weight"]
    with torch.no_grad():
        loss = ops.lm_head_cross_entropy(gold["hidden"].requires_grad_(False), gold["weight"], gold["labels"], lw)
    assert emu.calls == [("xtb_lm_head_ce", 300, 0)]
    assert torch.equal(loss, gold["eager.token.loss"])
    emu.calls.clear()
    ops.lm_head_cross_entropy(gold["hidden"], gold["weight"], gold["labels"], lw, chunk_size=128)  # nothing requires grad
    assert [c[2] for c in emu.calls] == [0, 0, 0]


@pytest.mark.parametrize("mode", ["eager", "chunk"])
def test_all_ignored_gives_zero_loss_and_zero_gradients(gold, emu, mode):
    labels = torch.full_like(gold["labels"], gold["ignore_index"])
    loss, dh, dw = _ours(gold, torch.zeros(labels.shape), None if mode == "eager" else 128, 1.0, labels)
    assert float(loss) == 0.0 and dh.count_nonzero() == 0 and dw.count_nonzero() == 0


def test_shape_errors_are_raised_on_the_host(gold, emu):
    from xtuner_b200 import _capi, ops

    with pytest.raises(_capi.XtbError):
        ops.lm_head_cross_entropy(gold["hidden"], gold["weight"][:, :128], gold["labels"], torch.ones(300))
    with pytest.raises(_capi.XtbError):
        ops.lm_head_cross_entropy(gold["hidden"], gold["weight"], gold["labels"][:10], torch.ones(300))
    with pytest.raises(ValueError):
        ops.lm_head_cross_entropy(gold["hidden"], gold["weight"], gold["labels"], torch.ones(300), chunk_size=0)
    assert emu.calls == []


# ---- plugin dispatch ---------------------------------------------------------------------------------------------------

sys.path.insert(0, os.path.join(HERE, "golden"))
import ref_shim  # noqa: E402


@pytest.fixture
def ce_mod(monkeypatch):
    if not ref_shim.reference_available():
        pytest.skip("no reference checkout found")
    import importlib

    from xtuner_b200 import plugin

    ref_shim.apply_cpu_patches()
    monkeypatch.setattr(plugin, "_on_device", lambda t: True)  # host tensors: the eligibility predicate's only device question
    return importlib.import_module("xtuner.v1.loss.ce_loss")


def _ctx(ce_mod, gold, mode, cls=None, V=None, kwargs_cls=None):
    cfg = ce_mod.CELossConfig(mode=mode, chunk_size=128, loss_reduction="token", ignore_idx=gold["ignore_index"])
    labels = gold["labels"].view(1, -1).clone()
    if V is not None:
        labels = labels.clamp(max=V - 1)
    ctx = (cls or ce_mod.LMHeadLossContext)(cfg, (kwargs_cls or ce_mod.CELossKwargs)(shifted_labels=labels))
    (ctx,) = ce_mod.LMHeadLossContext.build_batches([ctx])
    return ctx


def test_plugin_install_and_uninstall_restore_the_class_exactly(ce_mod):
    from xtuner_b200 import plugin

    cls = ce_mod.LMHeadLossContext
    before = dict(vars(cls))
    plugin.install_lm_head_loss()
    plugin.install_lm_head_loss()  # idempotent
    assert vars(cls)["eager_mode"] is not before["eager_mode"] and vars(cls)["chunk_mode"] is not before["chunk_mode"]
    plugin.uninstall_lm_head_loss()
    assert dict(vars(cls)) == before


def test_plugin_dispatch(ce_mod, gold, emu, monkeypatch):
    from xtuner_b200 import ops, plugin

    cls = ce_mod.LMHeadLossContext
    orig = []
    for name in ("eager_mode", "chunk_mode"):  # record which calls reach the reference's methods
        f = vars(cls)[name]
        monkeypatch.setattr(cls, name, lambda self, *a, _f=f, _n=name: (orig.append(_n), _f(self, *a))[1])
    ours = []
    real = ops.lm_head_cross_entropy
    monkeypatch.setattr(ops, "lm_head_cross_entropy", lambda *a, **k: (ours.append(a[-1]), real(*a, **k))[1])
    plugin.install_lm_head_loss()
    try:
        hidden = gold["hidden"].view(1, 300, -1)
        for mode, chunk in (("eager", None), ("chunk", 128)):
            ctx = _ctx(ce_mod, gold, mode)
            h = hidden.clone().requires_grad_(True)
            w = gold["weight"].clone().requires_grad_(True)
            loss, (logits, extra) = ctx.forward(h, w)
            loss.backward()
            assert ours[-1] == chunk and logits is None and orig == []
            assert torch.equal(loss.detach(), gold[f"{mode}.token.loss"])
            assert torch.equal(h.grad, gold[f"{mode}.token.dh"]) and torch.equal(w.grad, gold[f"{mode}.token.dw"])
        n = len(ours)
        kw = lambda c: c.loss_kwargs  # noqa: E731
        # MTP: a subclass with its own loss_fn
        from xtuner.v1.loss.mtp_loss import MTPLossContext, MTPLossKwargs

        mtp = _ctx(ce_mod, gold, "eager", cls=MTPLossContext, kwargs_cls=MTPLossKwargs)
        mtp.eager_mode(hidden, gold["weight"], None, kw(mtp))
        # a head bias
        ctx = _ctx(ce_mod, gold, "eager")
        ctx.eager_mode(hidden, gold["weight"], torch.zeros(gold["weight"].shape[0], dtype=torch.bfloat16), kw(ctx))
        # an fp32 head (fp32_lm_head)
        ctx.eager_mode(hidden.float(), gold["weight"].float(), None, kw(ctx))
        # V % 128 != 0
        ctxv = _ctx(ce_mod, gold, "chunk", V=1000)
        ctxv.chunk_mode(hidden, gold["weight"][:1000], None, kw(ctxv))
        # chunk mode over a batch of two sequences (ChunkLoss splits each along the sequence)
        ctx2 = _ctx(ce_mod, gold, "chunk")
        ctx2.loss_kwargs.shifted_labels = ctx2.loss_kwargs.shifted_labels.view(2, 150)
        ctx2.loss_kwargs.loss_weight = ctx2.loss_kwargs.loss_weight.view(2, 150)
        ctx2.chunk_mode(hidden.view(2, 150, -1), gold["weight"], None, kw(ctx2))
        # liger: the original chunk_mode (which needs the liger kernel, absent here)
        liger = _ctx(ce_mod, gold, "chunk")
        object.__setattr__(liger.loss_cfg, "mode", "liger")
        with pytest.raises(AssertionError, match="liger"):
            liger.chunk_mode(hidden, gold["weight"], None, kw(liger))
        assert len(ours) == n
        assert orig == ["eager_mode", "eager_mode", "eager_mode", "chunk_mode", "chunk_mode", "chunk_mode"]
    finally:
        plugin.uninstall_lm_head_loss()
