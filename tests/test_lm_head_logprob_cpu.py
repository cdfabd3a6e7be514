"""CPU coverage of the lm_head log-probabilities (``ops.lm_head_logprobs``, ``plugin.install_rl_lm_head``):

* the shipped host orchestration (chunk loop, autograd node, the single backward) over a host-memory emulation of
  ``xtb_lm_head_logprob`` / ``xtb_lm_head_logprob_bwd`` written from the header's contract with the reference's own
  arithmetic, against fixtures made by the reference's ``LogProbContext`` and ``GRPOLossContext``
  (``tests/golden/make_lm_head_logprob_golden.py``), bit for bit;
* the plugin's dispatch: eligible calls to ours, everything else to the reference's methods, and an exact restore.

The kernels themselves are covered on an H100 by ``tests/test_gpu_lm_head_logprob.py``."""
import os
import sys

import pytest
import torch
from torch.nn import functional as F

from tests.cabi_emulator import EmulatedLib, _view
from tests.conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
GRPO_CASES = [(m, kl) for m in ("eager", "chunk") for kl in ("none", "k1", "low_var_kl")]


@pytest.fixture(scope="module")
def gold():
    return load_golden("lm_head_logprob")


def _lsm_at_label(z, lab):
    return F.log_softmax(z.float(), dim=-1).gather(-1, lab.clip(min=0).unsqueeze(-1)).squeeze(-1)


class LogProbEmulatedLib(EmulatedLib):
    """The two entries computed as the header states them, with gather_logprobs' own arithmetic."""

    def xtb_lm_head_logprob_workspace_bytes(self, T, V):
        return self._real.xtb_lm_head_logprob_workspace_bytes(T, V)

    def xtb_lm_head_logprob(self, h, w, labels, T, H, V, z, ws, logp, row_stats, stream):
        self.calls.append(("xtb_lm_head_logprob", T, row_stats is None))
        assert ws is not None
        zz = F.linear(_view(h, torch.bfloat16, T, H), _view(w, torch.bfloat16, V, H))
        _view(z, torch.bfloat16, T, V).copy_(zz)
        _view(logp, torch.float32, T).copy_(_lsm_at_label(zz, _view(labels, torch.int64, T)))
        if row_stats is not None:
            m = zz.float().amax(-1)
            _view(row_stats, torch.float32, T, 2).copy_(torch.stack([m, (zz.float() - m[:, None]).logsumexp(-1)], -1))
        return 0

    def xtb_lm_head_logprob_bwd(self, z_or_G, row_stats, labels, grad_logp, h, w, T, H, V, ws, dh, dw, stream):
        self.calls.append(("xtb_lm_head_logprob_bwd", T))
        assert ws is not None and row_stats is not None
        zbuf = _view(z_or_G, torch.bfloat16, T, V)
        hh = _view(h, torch.bfloat16, T, H).clone().requires_grad_(True)
        ww = _view(w, torch.bfloat16, V, H).clone().requires_grad_(True)
        with torch.enable_grad():
            zz = zbuf.clone().requires_grad_(True)
            (G,) = torch.autograd.grad(_lsm_at_label(zz, _view(labels, torch.int64, T)), zz,
                                       _view(grad_logp, torch.float32, T))
            gh, gw = torch.autograd.grad(F.linear(hh, ww), (hh, ww), G)
        zbuf.copy_(G)
        _view(dh, torch.bfloat16, T, H).copy_(gh)
        _view(dw, torch.bfloat16, V, H).copy_(gw)
        return 0


@pytest.fixture
def emu(monkeypatch):
    from xtuner_b200 import _capi, ops

    lib = LogProbEmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    monkeypatch.setattr(ops, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "_scratch", lambda tag, n, dev: torch.empty(max(int(n), 16), dtype=torch.uint8))
    return lib


# ---- host op -----------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("chunk", [None, 48, 1000])
def test_no_grad_logprobs_run_forward_entries_only_and_give_the_reference_bits(gold, emu, chunk):
    from xtuner_b200 import ops

    with torch.no_grad():
        logp = ops.lm_head_logprobs(gold["hidden"].clone().requires_grad_(True), gold["weight"], gold["labels"], chunk)
    assert logp.shape == gold["labels"].shape and logp.dtype == torch.float32
    assert torch.equal(logp, gold["logprob.eager"]) and torch.equal(logp, gold["logprob.chunk"])
    rows = [c[1] for c in emu.calls]
    assert rows == ({48: [48, 48, 32]}.get(chunk, [128]))
    assert all(c[0] == "xtb_lm_head_logprob" and c[2] for c in emu.calls), "row_stats must be NULL without grad"


def test_nothing_requiring_grad_is_the_no_grad_path(gold, emu):
    from xtuner_b200 import ops

    logp = ops.lm_head_logprobs(gold["hidden"], gold["weight"], gold["labels"], 48)
    assert logp.grad_fn is None and torch.equal(logp, gold["logprob.chunk"])
    assert [c[2] for c in emu.calls] == [True, True, True]


def test_grad_path_gives_the_same_logprobs_and_one_backward_only(gold, emu):
    from xtuner_b200 import ops

    h = gold["hidden"].clone().requires_grad_(True)
    w = gold["weight"].clone().requires_grad_(True)
    logp = ops.lm_head_logprobs(h, w, gold["labels"], chunk_size=48)  # one node: chunking only bounds no-grad memory
    assert torch.equal(logp.detach(), gold["logprob.eager"])
    assert emu.calls == [("xtb_lm_head_logprob", 128, False)]
    c = torch.linspace(-1, 1, 128).view(1, 128)
    (logp * c).sum().backward(retain_graph=True)
    assert h.grad.shape == h.shape and w.grad.shape == w.shape
    assert emu.calls[-1] == ("xtb_lm_head_logprob_bwd", 128)
    with pytest.raises(RuntimeError, match="runs once"):
        (logp * c).sum().backward()
    assert len(emu.calls) == 2


def test_shape_errors_are_raised_on_the_host(gold, emu):
    from xtuner_b200 import _capi, ops

    with pytest.raises(_capi.XtbError):
        ops.lm_head_logprobs(gold["hidden"], gold["weight"][:, :64], gold["labels"])
    with pytest.raises(_capi.XtbError):
        ops.lm_head_logprobs(gold["hidden"], gold["weight"], gold["labels"][:, :10])
    with pytest.raises(ValueError):
        ops.lm_head_logprobs(gold["hidden"], gold["weight"], gold["labels"], chunk_size=0)
    assert emu.calls == []


# ---- plugin over the reference's contexts ------------------------------------------------------------------------------

sys.path.insert(0, os.path.join(HERE, "golden"))
import ref_shim  # noqa: E402


@pytest.fixture
def rl(monkeypatch):
    if not ref_shim.reference_available():
        pytest.skip("no reference checkout found")
    import importlib

    from xtuner_b200 import plugin

    ref_shim.apply_cpu_patches()
    monkeypatch.setattr(plugin, "_on_device", lambda t: True)  # host tensors: the eligibility predicate's only device question
    return importlib.import_module("xtuner.v1.loss.rl_loss"), importlib.import_module("xtuner.v1.rl.loss.grpo_loss")


def _logprob_ctx(rl, gold, mode, cls=None):
    cfg = rl[0].LogProbConfig(mode=mode, chunk_size=gold["chunk_size"], ignore_idx=gold["ignore_index"])
    return (cls or rl[0].LogProbContext)(cfg, rl[0].LogProbKwargs(shifted_labels=gold["labels"].clone()))


def _grpo_ctx(rl, gold, mode, kl, cls=None):
    g = rl[1]
    cfg = g.GRPOLossConfig(policy_loss_cfg=dict(gold["policy_loss_cfg"]), use_kl_loss=kl != "none",
                           kl_loss_coef=gold["kl_loss_coef"], kl_loss_type=None if kl == "none" else kl, mode=mode,
                           chunk_size=gold["chunk_size"], ignore_idx=gold["ignore_index"])
    kw = g.GRPOLossKwargs(shifted_labels=gold["labels"].clone(), old_logprobs=gold["old_logprobs"].clone(),
                          advantages=gold["advantages"].clone(), ref_logprobs=gold["ref_logprobs"].clone())
    (ctx,) = g.GRPOLossContext.build_batches([(cls or g.GRPOLossContext)(cfg, kw)])
    return ctx


def _run_grpo(ctx, gold, grad_output):
    h = gold["hidden"].clone().requires_grad_(True)
    w = gold["weight"].clone().requires_grad_(True)
    loss, (logits, extra) = ctx.forward(h, w)
    loss.backward(torch.tensor(grad_output))
    return loss.detach(), logits, extra, h.grad, w.grad


@pytest.mark.parametrize("mode", ["eager", "chunk"])
def test_plugin_logprob_context_gives_the_reference_bits(rl, gold, emu, mode):
    from xtuner_b200 import plugin

    plugin.install_rl_lm_head()
    try:
        ctx = _logprob_ctx(rl, gold, mode)
        with torch.no_grad():
            logp, (logits, extra) = ctx.forward(gold["hidden"], gold["weight"])
    finally:
        plugin.uninstall_rl_lm_head()
    assert logits is None and extra == {}
    assert torch.equal(logp, gold[f"logprob.{mode}"])
    assert [c[1] for c in emu.calls] == ([128] if mode == "eager" else [48, 48, 32]) and all(c[2] for c in emu.calls)


@pytest.mark.parametrize("mode,kl", GRPO_CASES)
def test_plugin_grpo_gives_the_reference_bits(rl, gold, emu, mode, kl):
    """Loss, every extra_info entry and, where the fixture holds them, both gradients (two of those cases with a loss
    gradient other than 1)."""
    from xtuner_b200 import plugin

    key = f"grpo.{mode}.{kl}"
    plugin.install_rl_lm_head()
    try:
        loss, logits, extra, dh, dw = _run_grpo(_grpo_ctx(rl, gold, mode, kl), gold, gold[f"{key}.grad_output"])
    finally:
        plugin.uninstall_rl_lm_head()
    assert logits is None
    assert torch.equal(loss, gold[f"{key}.loss"])
    want = gold[f"{key}.extra_info"]
    assert set(extra) == set(want)
    for k, v in want.items():
        assert torch.equal(extra[k], v), k
    if f"{key}.dh" in gold:
        assert torch.equal(dh, gold[f"{key}.dh"]) and torch.equal(dw, gold[f"{key}.dw"])
    n_chunks = 1 if mode == "eager" else 3
    assert [c[0] for c in emu.calls] == ["xtb_lm_head_logprob", "xtb_lm_head_logprob_bwd"] * n_chunks


def test_plugin_install_and_uninstall_restore_the_classes_exactly(rl):
    from xtuner_b200 import plugin

    lp, grpo = rl[0].LogProbContext, rl[1].GRPOLossContext
    ce = sys.modules["xtuner.v1.loss.ce_loss"].LMHeadLossContext
    before = [dict(vars(c)) for c in (lp, grpo, ce)]
    plugin.install_rl_lm_head()
    plugin.install_rl_lm_head()  # idempotent
    assert vars(lp)["loss_fn"] is not before[0]["loss_fn"] and vars(lp)["chunk_mode"] is not before[0]["chunk_mode"]
    assert vars(grpo)["loss_fn"] is not before[1]["loss_fn"]
    plugin.uninstall_rl_lm_head()
    assert [dict(vars(c)) for c in (lp, grpo, ce)] == before
    for first, second in ((plugin.install_lm_head_loss, plugin.install_rl_lm_head),
                          (plugin.install_rl_lm_head, plugin.install_lm_head_loss)):
        first()
        second()
        plugin.uninstall_lm_head_loss()
        plugin.uninstall_rl_lm_head()
        assert [dict(vars(c)) for c in (lp, grpo, ce)] == before


@pytest.mark.parametrize("order", ["ce_first", "rl_first"])
def test_plugin_composes_with_the_cross_entropy_install(rl, gold, emu, order):
    from xtuner_b200 import plugin

    installs = [plugin.install_lm_head_loss, plugin.install_rl_lm_head]
    for f in installs if order == "ce_first" else installs[::-1]:
        f()
    try:
        for mode in ("eager", "chunk"):
            key = f"grpo.{mode}.low_var_kl"
            loss, _, extra, _, _ = _run_grpo(_grpo_ctx(rl, gold, mode, "low_var_kl"), gold, gold[f"{key}.grad_output"])
            assert torch.equal(loss, gold[f"{key}.loss"])
            assert torch.equal(extra["reduced_train_policy_kl3_sum"], gold[f"{key}.extra_info"]["reduced_train_policy_kl3_sum"])
    finally:
        plugin.uninstall_rl_lm_head()
        plugin.uninstall_lm_head_loss()
    assert sum(c[0] == "xtb_lm_head_logprob_bwd" for c in emu.calls) == 4


def test_plugin_sends_every_ineligible_call_to_the_original_methods(rl, gold, emu, monkeypatch):
    from xtuner_b200 import plugin

    lp, grpo = rl[0].LogProbContext, rl[1].GRPOLossContext
    orig = []
    for cls, name in ((lp, "loss_fn"), (lp, "chunk_mode"), (grpo, "loss_fn")):  # record calls reaching the reference
        f = vars(cls)[name]
        monkeypatch.setattr(cls, name, lambda self, *a, _f=f, _n=f"{cls.__name__}.{name}": (orig.append(_n), _f(self, *a))[1])

    class OwnGRPO(grpo):  # a subclass with its own loss_fn
        def loss_fn(self, *a):
            orig.append("OwnGRPO.loss_fn")
            return grpo.loss_fn(self, *a)

    class OwnLogProb(lp):
        pass

    class NotPlain(torch.Tensor):
        pass

    plugin.install_rl_lm_head()
    try:
        h, w, V = gold["hidden"], gold["weight"], gold["weight"].shape[0]
        bias = torch.zeros(V, dtype=torch.bfloat16)
        with torch.no_grad():
            for mode, method in (("eager", "loss_fn"), ("chunk", "chunk_mode")):
                ctx = _logprob_ctx(rl, gold, mode)
                kw = ctx.loss_kwargs
                getattr(ctx, method)(h, w, bias, kw)  # a head bias
                getattr(ctx, method)(h.float(), w.float(), None, kw)  # an fp32 head
                getattr(ctx, method)(h, w.as_subclass(NotPlain), None, kw)  # not a plain tensor
                getattr(ctx, method)(h[..., :64].contiguous(), w[:, :64].contiguous(), None, kw)  # H % 128 != 0
                sub = _logprob_ctx(rl, gold, mode, cls=OwnLogProb)
                getattr(sub, method)(h, w, None, sub.loss_kwargs)  # a subclass
            assert orig == ["LogProbContext.loss_fn"] * 5 + ["LogProbContext.chunk_mode"] * 5
            orig.clear()
            ctx = _grpo_ctx(rl, gold, "eager", "none")
            kw = ctx.loss_kwargs
            ctx.loss_fn(h, w, bias, kw)
            ctx.loss_fn(h.float(), w.float(), None, kw)
            ctx.loss_fn(h, w.as_subclass(NotPlain), None, kw)
            lab = kw.shifted_labels.clamp(max=199)
            ctx.loss_fn(h, w[:200], None, kw.model_copy(update={"shifted_labels": lab}))  # V % 128 != 0
            liger = _grpo_ctx(rl, gold, "eager", "none")
            object.__setattr__(liger.loss_cfg, "mode", "liger")
            liger.loss_fn(h, w, None, liger.loss_kwargs)
            own = _grpo_ctx(rl, gold, "eager", "none", cls=OwnGRPO)
            own.loss_fn(h, w, None, own.loss_kwargs)
        assert orig == ["GRPOLossContext.loss_fn"] * 5 + ["OwnGRPO.loss_fn", "GRPOLossContext.loss_fn"]
        assert emu.calls == []
    finally:
        plugin.uninstall_rl_lm_head()
