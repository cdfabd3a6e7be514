"""Selective recompute of the fused MoE nodes (``recompute="act"`` / ``"experts"`` in ``xtuner_b200/fused.py``) on the CPU,
over the host-memory emulation of the C-ABI: each mode gives the outputs and gradients of ``recompute=None`` exactly,
keeps exactly the tensors it is meant to keep, runs the launches it is meant to run, and reaches the reference's own
model through ``plugin.convert_model``.  The kernels' bits are the GPU suite's (tests/test_gpu_moe_recompute.py)."""
import os

import pytest
import torch
from torch import nn

from oracle import moe_oracle as O
from tests.cabi_emulator import _view
from tests.test_router_replay_cpu import ReplayEmulatedLib

MODES = ("act", "experts")


class RecomputeEmulatedLib(ReplayEmulatedLib):
    """The emulated C-ABI plus xtb_swiglu_bwd_act, computed on host memory as include/xtuner_b200.h states it."""

    def xtb_swiglu_bwd_act(self, grad_out, h, grad_h, act_out, M, I, stream):
        self.calls.append("xtb_swiglu_bwd_act")
        hv = _view(h, torch.bfloat16, M, 2 * I)
        _view(grad_h, torch.bfloat16, M, 2 * I).copy_(self._swiglu_bwd(_view(grad_out, torch.bfloat16, M, I), hv))
        _view(act_out, torch.bfloat16, M, I).copy_(O.swiglu(hv))
        return 0


@pytest.fixture
def emu(monkeypatch):
    from xtuner_b200 import _capi, fused, ops, router

    lib = RecomputeEmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    for mod in (ops, router, fused):
        monkeypatch.setattr(mod, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "permute_workspace", lambda T, K, E, dev: torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8))
    monkeypatch.setattr(ops, "_scratch", lambda tag, n, dev: torch.empty(max(int(n), 16), dtype=torch.uint8))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))  # the public entries' guards
    return lib


def _inputs(T, H, I, E, seed):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(T, H, generator=g).to(torch.bfloat16)
    res = torch.randn(T, H, generator=g).to(torch.bfloat16)
    nw = 1 + 0.1 * torch.randn(H, generator=g)
    gw = torch.randn(E, H, generator=g) * 0.05
    w13 = (torch.randn(E, 2 * I, H, generator=g) * H**-0.5).to(torch.bfloat16)
    w2 = (torch.randn(E, H, I, generator=g) * I**-0.5).to(torch.bfloat16)
    go = torch.randn(T, H, generator=g).to(torch.bfloat16)
    g_rw = torch.randn(T, E, generator=g) * 0.01
    return h, res, nw, gw, w13, w2, go, g_rw


def _replay_ids(T, E, K, seed):
    ids = torch.randint(0, E, (T, K), generator=torch.Generator().manual_seed(seed))
    ids[::3, 0] = ids[::3, -1]  # duplicates inside a row, as replayed ids may hold
    return ids


def _run(node, inputs, K, replay, recompute):
    """(outputs, gradients) of one forward + backward of a node through its public entry"""
    from xtuner_b200 import fused

    h, res, nw, gw, w13, w2, go, g_rw = inputs
    if node == "block":
        leaves = [t.clone().requires_grad_(True) for t in (h, nw, gw, w13, w2)]
        out, rr = fused.fused_moe_block(leaves[0], leaves[1], 1e-6, *leaves[2:], top_k=K, rollout_routed_experts=replay,
                                        recompute=recompute)
    else:
        leaves = [t.clone().requires_grad_(True) for t in (h, gw, w13, w2)] + ([res.clone().requires_grad_(True)]
                                                                               if node == "residual" else [])
        out, rr = fused.fused_moe(leaves[0], leaves[4] if node == "residual" else None, *leaves[1:4], top_k=K,
                                  rollout_routed_experts=replay, recompute=recompute)
    torch.autograd.backward([out, rr["router_weights"]], [go, g_rw])
    return [out.detach(), rr["logits"].detach(), rr["router_weights"].detach(), rr["topk_ids"]], [t.grad for t in leaves]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("replay", [False, True])
@pytest.mark.parametrize("node", ["block", "residual", "plain"])
@pytest.mark.parametrize("E", [8, 16])
def test_each_mode_equals_the_saved_path(emu, node, replay, mode, E):
    """E = 8 takes the one-launch gate and route entries, E = 16 the separate ones"""
    T, H, I, K = 48, 256, 128, 2
    inputs = _inputs(T, H, I, E, E + len(node))
    ids = _replay_ids(T, E, K, 7) if replay else None
    want_out, want_g = _run(node, inputs, K, ids, None)
    emu.calls.clear()
    out, grads = _run(node, inputs, K, ids, mode)
    for a, b in zip(out + grads, want_out + want_g):
        assert torch.equal(a, b)
    rebuilt = {"act": "xtb_swiglu_bwd_act", "experts": "xtb_group_gemm_nt_swiglu"}[mode]
    assert emu.calls.count("xtb_moe_permute") == 1 and rebuilt in emu.calls


def _backward_calls(emu, node, mode):
    T, H, I, E, K = 32, 256, 128, 8, 2
    inputs = _inputs(T, H, I, E, 3)
    emu.calls.clear()
    from xtuner_b200 import fused

    h, res, nw, gw, w13, w2, go, g_rw = inputs
    x = h.clone().requires_grad_(True)
    if node == "block":
        out, _ = fused.fused_moe_block(x, nw, 1e-6, gw, w13, w2, top_k=K, recompute=mode)
    else:
        out, _ = fused.fused_moe(x, None, gw, w13, w2, top_k=K, recompute=mode)
    n_fwd = len(emu.calls)
    out.backward(go)
    # the emulated xtb_moe_permute logs the xtb_moe_permute_prepared it is built on as well
    return [c for c in emu.calls[n_fwd:] if c != "xtb_moe_permute_prepared"]


@pytest.mark.parametrize("node", ["block", "plain"])
def test_the_backward_rebuilds_in_the_stated_order(emu, node):
    """"act": a from the SwiGLU backward, x_perm permuted again after the dX GEMM of w13, no GEMM of the forward again;
    "experts": permute, both forward GEMMs, then the combine backward that frees y"""
    saved = _backward_calls(emu, node, None)
    act = _backward_calls(emu, node, "act")
    experts = _backward_calls(emu, node, "experts")
    i = saved.index("xtb_swiglu_bwd")
    want_act = saved[:i] + ["xtb_swiglu_bwd_act", "xtb_group_gemm_nn", "xtb_moe_permute"] + saved[i + 2:]
    assert saved[i + 1] == "xtb_group_gemm_nn" and act == want_act, act
    assert experts == ["xtb_moe_permute", "xtb_group_gemm_nt_swiglu", "xtb_group_gemm_nt"] + saved, experts


def _saved_bytes(node, mode, T, H, I, E, K):
    from xtuner_b200 import fused

    h, res, nw, gw, w13, w2, go, g_rw = _inputs(T, H, I, E, 4)
    x = h.clone().requires_grad_(True)
    if node == "block":
        out, _ = fused.fused_moe_block(x, nw, 1e-6, gw, w13, w2, top_k=K, recompute=mode)
    else:
        out, _ = fused.fused_moe(x, res, gw, w13, w2, top_k=K, recompute=mode)
    node_ctx = out.grad_fn.next_functions[0][0]  # the fused node behind the entry's output view
    return sum(t.numel() * t.element_size() for t in node_ctx.saved_tensors if t is not None)


@pytest.mark.parametrize("node", ["block", "plain"])
def test_saved_bytes_drop_by_the_listed_tensors(emu, node):
    """"act" drops x_perm [M, H] and a [M, I], "experts" also h [M, 2I] and y [M, H] (M = T * K, bf16); both keep the
    int32 ids [T, K] the permute runs on again"""
    T, H, I, E, K = 40, 256, 128, 8, 4
    M = T * K
    base = _saved_bytes(node, None, T, H, I, E, K)
    ids32 = T * K * 4
    assert base - _saved_bytes(node, "act", T, H, I, E, K) == (M * H + M * I) * 2 - ids32
    assert base - _saved_bytes(node, "experts", T, H, I, E, K) == (2 * M * H + 3 * M * I) * 2 - ids32


@pytest.mark.parametrize("mode", MODES)
def test_gradient_sink_and_no_tokens(emu, monkeypatch, mode):
    """the expert weight gradients still land in the GRAD_SINK buffers (the FSDP engine's), and T = 0 still runs no
    launch"""
    from xtuner_b200 import fused

    T, H, I, E, K = 32, 256, 128, 8, 2
    inputs = _inputs(T, H, I, E, 5)
    _, want = _run("block", inputs, K, None, None)
    w13, w2 = inputs[4], inputs[5]
    b13, b2 = torch.full((w13.numel(),), 7.0, dtype=torch.bfloat16), torch.full((w2.numel(),), 7.0, dtype=torch.bfloat16)
    monkeypatch.setattr(fused, "GRAD_SINK", lambda: (b13, b2))
    _run("block", inputs, K, None, mode)
    assert torch.equal(b13.view_as(w13), want[3]) and torch.equal(b2.view_as(w2), want[4])
    monkeypatch.setattr(fused, "GRAD_SINK", None)
    emu.calls.clear()
    x = torch.zeros(0, H, dtype=torch.bfloat16, requires_grad=True)
    out, rr = fused.fused_moe_block(x, inputs[2], 1e-6, inputs[3], w13, w2, top_k=K, recompute=mode)
    out.sum().backward()
    assert emu.calls == [] and x.grad.shape == (0, H)


def test_swiglu_bwd_act_refuses_bad_arguments_on_the_host():
    """the pointer values are never dereferenced"""
    from xtuner_b200 import _capi

    lib = _capi.load()
    A = 1 << 20  # a 16-byte aligned fake address
    assert lib.xtb_swiglu_bwd_act(A, A, A, None, 4, 64, None) == 1 and b"null pointer" in lib.xtb_last_error()
    for args in ((A + 8, A, A, A), (A, A + 4, A, A), (A, A, A + 2, A), (A, A, A, A + 8)):
        assert lib.xtb_swiglu_bwd_act(*args, 4, 64, None) == 1 and b"16-byte aligned" in lib.xtb_last_error()
    assert lib.xtb_swiglu_bwd_act(A, A, A, A, 4, 12, None) == 1 and b"bad shape" in lib.xtb_last_error()
    assert lib.xtb_swiglu_bwd_act(A, A, A, A, 4, 8 * 23171, None) == 1 and b"too wide" in lib.xtb_last_error()
    assert lib.xtb_last_error().startswith(b"xtb_swiglu_bwd_act")


@pytest.mark.parametrize("mode", MODES)
def test_modules_pass_the_mode_to_their_node(emu, mode):
    from xtuner_b200 import fused

    kw = dict(hidden_size=256, moe_intermediate_size=128, n_routed_experts=8, num_experts_per_tok=2)
    h, res = _inputs(16, 256, 128, 8, 6)[:2]
    for cls in (fused.FusedMoEBlock, fused.FusedMoELayer):
        mod = cls(**kw, recompute=mode)
        mod.experts.to(torch.bfloat16)
        emu.calls.clear()
        x = h.clone().requires_grad_(True)
        out, _ = mod(x) if cls is fused.FusedMoEBlock else mod(x, res)
        out.float().sum().backward()
        assert "xtb_moe_permute" in emu.calls and x.grad is not None


def test_unknown_modes_are_refused():
    from xtuner_b200 import fused, plugin

    x = torch.zeros(4, 256, dtype=torch.bfloat16)
    for bad in ("all", "", True, "ACT"):
        with pytest.raises(ValueError, match="recompute"):
            fused.fused_moe(x, None, torch.zeros(8, 256), torch.zeros(8, 256, 256), torch.zeros(8, 256, 128), top_k=2,
                            recompute=bad)
        with pytest.raises(ValueError, match="recompute"):
            fused.fused_moe_block(x, torch.ones(256), 1e-6, torch.zeros(8, 256), torch.zeros(8, 256, 256),
                                  torch.zeros(8, 256, 128), top_k=2, recompute=bad)
        for cls in (fused.FusedMoEBlock, fused.FusedMoELayer):
            with pytest.raises(ValueError, match="recompute"):
                cls(hidden_size=256, moe_intermediate_size=128, n_routed_experts=8, num_experts_per_tok=2, recompute=bad)
        with pytest.raises(ValueError, match="recompute"):
            plugin.convert_model(nn.Module(), fused=True, recompute=bad)
    for mode in MODES:
        with pytest.raises(ValueError, match="fused=True"):
            plugin.convert_model(nn.Module(), recompute=mode)
        layer = fused.FusedMoEBlock(hidden_size=256, moe_intermediate_size=128, n_routed_experts=8, num_experts_per_tok=2,
                                    recompute=mode)
        assert layer.recompute == mode
    assert plugin.convert_model(nn.Module(), fused=True, recompute=None) == 0


@pytest.mark.parametrize("mode", MODES)
def test_reference_model_converted_with_recompute(monkeypatch, mode):
    """the reference's own MoE model, ``convert_model(fused=True, recompute=mode)`` over the emulated C-ABI: losses and
    every parameter gradient equal to ``fused=True`` alone, and within the fused path's tolerance of the unconverted
    model"""
    from tests.golden import ref_shim

    if not ref_shim.reference_available():
        pytest.skip("no reference checkout found")
    import torch.distributed as dist

    from tests.test_plugin_reference_cpu import _build_reference_model, _install_emulated_cabi, _loss_and_grads

    if not dist.is_initialized():
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29697", RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
        dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        model, cfg = _build_reference_model(0, hidden=256)
        ref_out, ref_grads = _loss_and_grads(model, cfg)
        from xtuner_b200 import fused, plugin

        import tests.cabi_emulator

        monkeypatch.setattr(tests.cabi_emulator, "EmulatedLib", RecomputeEmulatedLib)  # the helper builds this one
        lib = _install_emulated_cabi(monkeypatch)
        assert isinstance(lib, RecomputeEmulatedLib)
        monkeypatch.setattr(fused, "current_stream", lambda: None)
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        assert plugin.convert_model(model, fused=True) == cfg.num_hidden_layers
        fused_out, fused_grads = _loss_and_grads(model, cfg)
        plugin.restore_model(model)
        lib.calls.clear()
        assert plugin.convert_model(model, fused=True, recompute=mode) == cfg.num_hidden_layers
        our_out, our_grads = _loss_and_grads(model, cfg)
        assert lib.calls.count("xtb_moe_permute") == cfg.num_hidden_layers
        assert set(our_out) == set(fused_out) and set(our_grads) == set(fused_grads) == set(ref_grads)
        for k in fused_out:
            assert torch.equal(our_out[k], fused_out[k]), k
            torch.testing.assert_close(our_out[k], ref_out[k], rtol=2e-4, atol=1e-5)
        for k in fused_grads:
            assert torch.equal(our_grads[k], fused_grads[k]), k
            a, b = our_grads[k].float(), ref_grads[k].float()
            assert ((a - b).abs() > 3e-2 * (b.abs() + b.abs().mean())).float().mean() < 5e-3, k
        plugin.restore_model(model)
        assert not any("_forward" in vars(m) for m in model.modules())
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()
