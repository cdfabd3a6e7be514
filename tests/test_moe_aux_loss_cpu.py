"""CPU coverage of the MoE auxiliary-loss statistics (``ops.moe_aux_stats``, ``plugin.install_moe_aux_loss``):

* the op and the install, over a host-memory emulation of ``xtb_moe_aux_stats`` / ``xtb_moe_aux_stats_bwd`` written from
  the header's contract (``AuxStatsEmulatedLib``), reproduce the fixture the reference's own ``AuxLossContext``,
  ``BalancingLossContext`` and ``ZLossContext`` made (``tests/golden/make_moe_aux_loss_golden.py``): counts exactly,
  losses and gradients within fp32 summation tolerance;
* calls the kernels do not cover run the original ``accumulate``; install and uninstall restore the class attribute;
* engine level: the reference's MoE model with both losses, ``convert_model(fused=True)`` over the emulated C-ABI, with
  and without the install, against the unconverted model.

The kernels themselves are covered on an H100 by ``tests/test_gpu_moe_aux_loss.py``."""
import os
import sys

import pytest
import torch

from tests.cabi_emulator import EmulatedLib, _view
from tests.conftest import load_golden

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import ref_shim  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_shim.reference_available(), reason="no reference checkout found")


class AuxStatsEmulatedLib(EmulatedLib):
    """The two entries computed on host memory as the header states them."""

    def xtb_moe_aux_stats_workspace_bytes(self, N, E):
        return self._real.xtb_moe_aux_stats_workspace_bytes(N, E)

    def xtb_moe_aux_stats(self, rw, logits, ids, N, E, K, tpe, rw_sum, z_sum, lse, ws, stream):
        self.calls.append("xtb_moe_aux_stats")
        if not (1 <= E <= 512 and K >= 1 and N >= 0 and tpe is not None and ws is not None):
            return 1
        idv = _view(ids, torch.int64, N, K).reshape(-1) if N else torch.zeros(0, dtype=torch.int64)
        keep = idv[(idv >= 0) & (idv <= E)].clamp(max=E - 1)
        _view(tpe, torch.int64, E).copy_(torch.bincount(keep, minlength=E))
        if rw_sum is not None:
            _view(rw_sum, torch.float32, E).copy_(_view(rw, torch.float32, N, E).sum(0) if N else torch.zeros(E))
        if z_sum is not None:
            l = torch.logsumexp(_view(logits, torch.float32, N, E), dim=-1) if N else torch.zeros(0)
            if N:
                _view(lse, torch.float32, N).copy_(l)
            _view(z_sum, torch.float32, 1).copy_(l.square().sum())
        return 0

    def xtb_moe_aux_stats_bwd(self, g_rw_sum, g_z, logits, lse, N, E, g_rw, g_logits, stream):
        self.calls.append("xtb_moe_aux_stats_bwd")
        if N == 0:
            return 0
        if g_rw is not None:
            _view(g_rw, torch.float32, N, E).copy_(_view(g_rw_sum, torch.float32, E).expand(N, E))
        if g_logits is not None:
            l = _view(lse, torch.float32, N)[:, None]
            gz = _view(g_z, torch.float32, 1)
            _view(g_logits, torch.float32, N, E).copy_((gz * (2 * l)) * (_view(logits, torch.float32, N, E) - l).exp())
        return 0


@pytest.fixture
def emulated(monkeypatch):
    ref_shim.apply_cpu_patches()
    from xtuner_b200 import _capi, ops, plugin

    lib = AuxStatsEmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    monkeypatch.setattr(ops, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "_moe_aux_workspace", lambda N, E, dev: torch.zeros(
        int(lib.xtb_moe_aux_stats_workspace_bytes(N, E)), dtype=torch.uint8))
    monkeypatch.setattr(plugin, "_on_device", lambda t: True)
    yield lib
    plugin.uninstall_moe_aux_loss()


@pytest.fixture(scope="module")
def gold():
    return load_golden("moe_aux_loss")


@pytest.fixture(scope="module")
def gloo():
    import torch.distributed as dist

    if not dist.is_initialized():
        import socket

        with socket.socket() as s:  # a free port: other modules of the suite bring up their own groups
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
        dist.init_process_group("gloo", rank=0, world_size=1)
    yield
    if dist.is_initialized():
        dist.destroy_process_group()


def _close(a, b, what, rtol=2e-6, atol=1e-9):
    torch.testing.assert_close(a, b, rtol=rtol, atol=atol, msg=lambda m: f"{what}: {m}")


CASES = ["e8k2", "e128k8", "batch2", "zalpha0", "n0"]


@pytest.mark.parametrize("name", CASES)
def test_install_reproduces_the_reference_fixture(emulated, gold, gloo, name):
    import make_moe_aux_loss_golden as G

    from xtuner_b200 import plugin

    plugin.install_moe_aux_loss()
    spec = gold[f"{name}.spec"]
    got = G.run_case(2000 + gold["cases"].index(name), *spec, G.CASES[name][7])
    layers = spec[3]
    assert emulated.calls.count("xtb_moe_aux_stats") == layers
    for l in range(layers):
        for k in ("rw", "logits", "ids"):
            assert torch.equal(got[f"{k}{l}"], gold[f"{name}.{k}{l}"]), f"input {k}{l} differs from the fixture"
        assert torch.equal(got[f"tpe{l}"], gold[f"{name}.tpe{l}"]), f"counts of layer {l}"
        _close(got[f"g_rw{l}"], gold[f"{name}.g_rw{l}"], f"g_rw{l}")
        _close(got[f"g_logits{l}"], gold[f"{name}.g_logits{l}"], f"g_logits{l}", atol=1e-10)
    assert torch.equal(got["tpe_global"], gold[f"{name}.tpe_global"])
    for k in ("balancing_loss", "z_loss", "hidden_grad"):
        _close(got[k], gold[f"{name}.{k}"], k)


@pytest.mark.parametrize("name", CASES)
def test_op_reproduces_the_reference_statistics(emulated, gold, name):
    from xtuner_b200 import ops

    E = gold[f"{name}.spec"][0]
    rw = gold[f"{name}.rw0"].clone().requires_grad_(True)
    logits = gold[f"{name}.logits0"].clone().requires_grad_(True)
    tpe, rw_sum, z_sum = ops.moe_aux_stats(rw, logits, gold[f"{name}.ids0"], E, need_rw_sum=True, need_z=True)
    assert torch.equal(tpe, gold[f"{name}.tpe0"]) and not tpe.requires_grad
    _close(rw_sum, rw.detach().sum(0), "rw_sum")
    _close(z_sum, torch.logsumexp(logits.detach(), -1).square().sum(), "z_sum")
    (rw_sum * torch.arange(E)).sum().add(z_sum * 3).backward()
    assert torch.equal(rw.grad, torch.arange(E, dtype=torch.float32).expand_as(rw))
    l = torch.logsumexp(logits.detach(), -1, keepdim=True)
    assert torch.equal(logits.grad, (3 * (2 * l)) * (logits.detach() - l).exp())


def test_counts_follow_histc_at_its_edges(emulated):
    from xtuner_b200 import ops

    ids = torch.tensor([[0, 3], [4, 5], [-1, 4], [2, 2]], dtype=torch.int64)
    tpe, rw_sum, z_sum = ops.moe_aux_stats(None, None, ids, 4, need_rw_sum=False)
    assert rw_sum is None and z_sum is None
    assert torch.equal(tpe, torch.histc(ids.float(), bins=4, min=0, max=4).long())
    assert tpe.tolist() == [1, 0, 2, 3]


def test_an_output_without_gradient_gives_its_input_none(emulated):
    from xtuner_b200 import ops

    rw = torch.rand(6, 8).requires_grad_(True)
    logits = torch.randn(6, 8).requires_grad_(True)
    ids = torch.randint(0, 8, (6, 2))
    _, rw_sum, z_sum = ops.moe_aux_stats(rw, logits, ids, 8, need_z=True)
    z_sum.backward()
    assert rw.grad is None and logits.grad is not None
    _, rw_sum, z_sum = ops.moe_aux_stats(rw, logits.detach(), ids, 8, need_z=True)
    calls = len(emulated.calls)
    z_sum.backward(retain_graph=True)  # the logits need no gradient and rw_sum got none: nothing to launch
    assert emulated.calls[calls:] == [] and rw.grad is None
    rw_sum.sum().backward()
    assert emulated.calls[calls:] == ["xtb_moe_aux_stats_bwd"] and torch.equal(rw.grad, torch.ones(6, 8))


def test_op_refuses_what_the_kernels_do_not_take(emulated):
    from xtuner_b200 import _capi, ops

    ids = torch.zeros(4, 2, dtype=torch.int64)
    with pytest.raises(_capi.XtbError):
        ops.moe_aux_stats(torch.rand(4, 600), None, ids, 600)
    with pytest.raises(_capi.XtbError):
        ops.moe_aux_stats(torch.rand(4, 8, dtype=torch.float64), None, ids, 8)
    with pytest.raises(_capi.XtbError):
        ops.moe_aux_stats(torch.rand(4, 8), None, ids.int(), 8)


def test_op_has_no_cpu_fallback():
    from xtuner_b200 import _capi, ops

    with pytest.raises(_capi.XtbError):
        ops.moe_aux_stats(torch.rand(4, 8), None, torch.zeros(4, 2, dtype=torch.int64), 8)


def _one_layer(aux_cls, bal_ctx, z_ctx, rw, logits, ids):
    from xtuner.v1.loss.aux_loss import AuxLossConfig

    aux = AuxLossConfig().build(n_routed_experts=rw.shape[1], num_experts_per_tok=ids.shape[1])
    aux.__class__ = aux_cls
    aux.accumulate(selected_router_weights=rw, selected_router_logits=logits, selected_experts=ids,
                   hidden_states=torch.zeros(rw.shape[0], 4), balancing_ctx=bal_ctx, z_ctx=z_ctx, num_tokens_local=rw.shape[0])
    return aux


def test_calls_outside_the_kernels_run_the_original(emulated):
    from xtuner.v1.loss.aux_loss import AuxLossContext
    from xtuner.v1.loss.moe_loss import BalancingLossConfig, BalancingLossContext, ZLossConfig

    from xtuner_b200 import plugin

    plugin.install_moe_aux_loss()
    N, E, K = 6, 8, 2
    rw, logits, ids = torch.rand(N, E), torch.randn(N, E), torch.randint(0, E, (N, K))

    class MyBalancing(BalancingLossContext):
        pass

    class MyAux(AuxLossContext):
        pass

    sub = BalancingLossConfig().build()
    sub.__class__ = MyBalancing
    big = torch.randint(0, 600, (N, K))
    for args in (
        (AuxLossContext, [sub], None, rw, logits, ids),  # a context subclass
        (MyAux, BalancingLossConfig().build(), None, rw, logits, ids),  # an AuxLossContext subclass
        (AuxLossContext, BalancingLossConfig().build(), None, rw.double(), logits, ids),  # not fp32
        (AuxLossContext, BalancingLossConfig().build(), None, rw, logits, ids.int()),  # int32 ids
        (AuxLossContext, BalancingLossConfig().build(), ZLossConfig().build(), rw, logits[:, :4], ids),  # logits shape
        (AuxLossContext, None, None, torch.rand(N, 600), torch.randn(N, 600), big),  # E above the kernel's range
    ):
        aux = _one_layer(*args)
        assert len(aux._local_load_logits_list) == 1
    assert emulated.calls == []
    plugin._on_device = lambda t: False  # host tensors (the fixture's monkeypatch restores it)
    _one_layer(AuxLossContext, BalancingLossConfig().build(), None, rw, logits, ids)
    assert emulated.calls == []


def test_install_and_uninstall_restore_the_class_attribute():
    ref_shim.apply_cpu_patches()
    from xtuner.v1.loss.aux_loss import AuxLossContext

    from xtuner_b200 import plugin

    orig = vars(AuxLossContext)["accumulate"]
    plugin.install_moe_aux_loss()
    installed = vars(AuxLossContext)["accumulate"]
    plugin.install_moe_aux_loss()
    assert installed is not orig and vars(AuxLossContext)["accumulate"] is installed and installed.__wrapped__ is orig
    plugin.uninstall_moe_aux_loss()
    plugin.uninstall_moe_aux_loss()
    assert vars(AuxLossContext)["accumulate"] is orig and plugin._SAVED not in vars(AuxLossContext)


# ---- engine level -----------------------------------------------------------------------------------------------------


def _model_step(model, cfg):
    from xtuner.v1.loss.ce_loss import CELossConfig
    from xtuner.v1.loss.moe_loss import BalancingLossConfig, ZLossConfig
    from xtuner.v1.model.moe.moe import SequenceContext

    torch.manual_seed(123)
    input_ids = torch.randint(0, cfg.vocab_size, (1, 65), dtype=torch.int64)
    seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cpu")
    loss_cfg = CELossConfig()
    lctx = loss_cfg.loss_ctx_cls.build_batches([loss_cfg.build(data={"shifted_labels": input_ids[:, 1:]}, sp_mesh=None)])[0]
    loss_ctx = {"lm": lctx, "balancing": BalancingLossConfig().build(), "z_loss": ZLossConfig(z_loss_alpha=1e-2).build()}
    model.zero_grad(set_to_none=True)
    out = model(seq_ctx=seq_ctx, loss_ctx=loss_ctx)
    fields = {k: getattr(out, k) for k in type(out).model_fields}
    total = sum(v for k, v in fields.items() if "loss" in k and isinstance(v, torch.Tensor) and v.requires_grad)
    total.backward()
    grads = {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}
    losses = {k: fields[k].detach().clone() for k in ("loss", "balancing_loss", "z_loss")}
    return losses, grads, fields["tokens_per_expert_global"].clone()


def test_reference_model_with_both_losses_fused_and_installed(monkeypatch, gloo):
    from tests.test_plugin_reference_cpu import _build_reference_model, _install_emulated_cabi
    from xtuner_b200 import fused, ops, plugin

    model, cfg = _build_reference_model(0, hidden=256)
    ref_losses, ref_grads, ref_tpe = _model_step(model, cfg)
    assert float(ref_losses["z_loss"]) > 0 and float(ref_losses["balancing_loss"]) > 0
    lib = _install_emulated_cabi(monkeypatch)
    lib.__class__ = AuxStatsEmulatedLib
    monkeypatch.setattr(fused, "current_stream", lambda: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    monkeypatch.setattr(ops, "_moe_aux_workspace", lambda N, E, dev: torch.zeros(
        int(lib.xtb_moe_aux_stats_workspace_bytes(N, E)), dtype=torch.uint8))
    assert plugin.convert_model(model, fused=True) == cfg.num_hidden_layers
    try:
        runs = {}
        for installed in (False, True):
            if installed:
                plugin.install_moe_aux_loss()
            lib.calls.clear()
            runs[installed] = _model_step(model, cfg)
            n_aux = lib.calls.count("xtb_moe_aux_stats")
            assert n_aux == (cfg.num_hidden_layers if installed else 0)
            assert lib.calls.count("xtb_moe_aux_stats_bwd") == n_aux
        for installed, (losses, grads, tpe) in runs.items():
            assert torch.equal(tpe, ref_tpe), f"tokens_per_expert_global (installed={installed})"
            for k, v in ref_losses.items():
                _close(losses[k], v, f"{k} (installed={installed})", rtol=2e-4, atol=1e-5)
            assert set(grads) == set(ref_grads)
            for k in ref_grads:
                a, b = grads[k], ref_grads[k]
                bad = ((a - b).abs() > 3e-2 * (b.abs() + b.abs().mean())).float().mean()
                assert bad < 5e-3, f"grad {k} (installed={installed}): {bad:.4f} of elements off"
        # the install changes only how the statistics are computed: the same step as the reference's accumulate
        for k in ref_losses:
            _close(runs[True][0][k], runs[False][0][k], f"{k}: installed vs not", rtol=1e-5, atol=1e-8)
        for k in ref_grads:
            _close(runs[True][1][k], runs[False][1][k], f"grad {k}: installed vs not", rtol=1e-3, atol=1e-6)
    finally:
        plugin.uninstall_moe_aux_loss()
        plugin.restore_model(model)
