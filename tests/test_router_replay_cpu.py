"""CPU coverage of routing replay (RL rollout-routed experts):

* the shipped host layers — the two replay custom ops, the routers, ``fused._gate_route`` and the fused node — over a
  host-memory emulation of the three replay entries written from the header's contract (``ReplayEmulatedLib``), against
  the reference's replay arithmetic (greedy.py:70-90, noaux_router.py:78-142) and autograd;
* the reference's MoE model (GreedyRouter) and its DeepSeek-style model (NoAuxRouter) run with
  ``seq_ctx.rollout_routed_experts``, converted per-op and with ``fused=True``, against the unconverted model: losses,
  gradients, the ids that reach the dispatcher, a layer past the tensor's layer count routing normally, and an offloaded
  (host-resident) tensor moved as the reference moves it;
* the fixture made by the reference's own routers (``tests/golden/router_replay.pt``): the restatement above reproduces
  it bit for bit, forward and backward, and the routers over the emulated entries reproduce it.

The kernels themselves are covered on an H100 by ``tests/test_gpu_router_replay.py``."""
import os

import pytest
import torch

from oracle import moe_oracle as O
from tests.cabi_emulator import EmulatedLib, _view


def _rows(addr, T, K, stride):
    """int64 [T, K] view with row stride ``stride`` (elements) of host memory at ``addr``"""
    if T == 0:
        return torch.empty(0, K, dtype=torch.int64)
    return _view(addr, torch.int64, (T - 1) * stride + K).as_strided((T, K), (stride, 1))


def _sanitise(ids, E):
    """the header's rule for ids outside [0, E): id 0, and every topk weight of the token NaN"""
    bad = (ids < 0) | (ids >= E)
    return torch.where(bad, torch.zeros_like(ids), ids), bad.any(1, keepdim=True)


def greedy_replay_reference(logits, ids, norm, scaling, scoring):
    """greedy.py:70-90 with ``rollout_routed_experts``: scores, gather at the given ids, renormalise, scale, histc"""
    p = torch.softmax(logits.float(), 1) if scoring == "softmax" else logits.float().sigmoid()
    w = p.gather(1, ids)
    if norm:
        w = w / w.sum(-1, keepdim=True)
    if scaling != 1.0:
        w = w * scaling
    return p, w, torch.histc(ids.float(), bins=p.shape[1], min=0, max=p.shape[1]).long()


def noaux_replay_reference(logits, bias, ids, K, n_group, topk_group, norm, scaling):
    """noaux_router.py:78-142 with ``rollout_routed_experts`` (the discarded top-k left out)"""
    s = logits.float().sigmoid()
    ch = s + bias.unsqueeze(0)
    if n_group != topk_group:
        T, E = logits.shape
        gsc = ch.view(T, n_group, -1).topk(2, dim=-1)[0].sum(dim=-1)
        gi = torch.topk(gsc, k=topk_group, dim=-1, sorted=False)[1]
        gm = torch.zeros_like(gsc).scatter_(1, gi, 1)
        m = gm.unsqueeze(-1).expand(T, n_group, E // n_group).reshape(T, -1)
        ch = ch.masked_fill(~m.bool(), 0.0)
    w = s.gather(1, ids)
    rw = ch / ch.sum(-1, keepdim=True)
    if K > 1 and norm:
        w = w / (w.sum(-1, keepdim=True) + 1e-20)
    return rw, w * scaling, torch.histc(ids.float(), bins=logits.shape[1], min=0, max=logits.shape[1])


# ---- the fixture made by the reference's own routers (tests/golden/make_router_replay_golden.py) --------------------------

PATTERNS = ("own", "dup", "never", "slice")


@pytest.fixture(scope="module")
def gold():
    from tests.conftest import load_golden

    return load_golden("router_replay")


def fixture_case_names():
    names = [f"greedy.{sc}.{nm}.e{E}.k{K}" for sc in ("softmax", "sigmoid") for nm in ("norm", "raw") for E in (8, 128)
             for K in (1, 2, 8)]
    return names + ["noaux.g8t4", "noaux.g8t8"]


def fixture_config(case):
    """greedy: ("greedy", E, K, scoring, norm, 1.5); noaux: ("noaux", 256, 8, n_group, topk_group, 2.5)"""
    parts = case.split(".")
    if parts[0] == "greedy":
        return "greedy", int(parts[3][1:]), int(parts[4][1:]), parts[1], parts[2] == "norm", 1.5
    g, t = parts[1][1:].split("t")
    return "noaux", 256, 8, int(g), int(t), 2.5


def fixture_ids(gold, case, pat):
    """the pattern's replayed ids; ``slice`` as the strided [:, 1, :] view of the stored [T, 3, K] tensor"""
    return gold[f"{case}.{pat}.full"][:, 1, :] if pat == "slice" else gold[f"{case}.{pat}.ids"]


def _restatement(gold, case, logits, ids):
    kind, E, K, a, b, scaling = fixture_config(case)
    if kind == "greedy":
        return greedy_replay_reference(logits, ids, b, scaling, a)
    return noaux_replay_reference(logits, gold[f"{case}.bias"], ids, K, a, b, True, scaling)


@pytest.mark.parametrize("case", fixture_case_names())
def test_restatement_reproduces_the_fixture_bit_for_bit(gold, case):
    for pat in PATTERNS:
        ids = fixture_ids(gold, case, pat)
        lg = gold[f"{case}.logits"].clone().requires_grad_(True)
        rw, tw, tpe = _restatement(gold, case, lg, ids)
        assert torch.equal(rw, gold[f"{case}.router_weights"]), f"{pat}: router_weights"
        assert torch.equal(tw, gold[f"{case}.{pat}.topk_weights"]), f"{pat}: topk_weights"
        assert torch.equal(tpe.double(), gold[f"{case}.{pat}.tokens_per_expert"].double()), f"{pat}: tokens_per_expert"
        ((tw * gold[f"{case}.{pat}.g_tw"]).sum() + (rw * gold[f"{case}.g_rw"]).sum()).backward()
        assert torch.equal(lg.grad, gold[f"{case}.{pat}.grad_logits"]), f"{pat}: grad_logits"
    if fixture_config(case)[0] == "noaux" and case.endswith("g8t4"):  # the `never` ids sit in masked groups
        assert (gold[f"{case}.router_weights"].gather(1, fixture_ids(gold, case, "never")) == 0).all()


class ReplayEmulatedLib(EmulatedLib):
    """The three replay entries computed on host memory as include/xtuner_b200.h states them."""

    def xtb_router_greedy_replay(self, logits, replay, stride, T, E, K, scoring, norm, scaling, rw, tw, ids, ids32, tpe, ws,
                                 stream):
        self.calls.append("xtb_router_greedy_replay")
        assert ws is None or ids32 is not None
        idx, bad = _sanitise(_rows(replay, T, K, stride).clone(), E)
        p, w, _ = greedy_replay_reference(_view(logits, torch.float32, T, E), idx, bool(norm), scaling,
                                          "softmax" if scoring == 0 else "sigmoid")
        _view(rw, torch.float32, T, E).copy_(p)
        _view(tw, torch.float32, T, K).copy_(torch.where(bad, float("nan"), w))
        _view(ids, torch.int64, T, K).copy_(idx)
        if ids32 is not None:
            _view(ids32, torch.int32, T, K).copy_(idx.int())
        _view(tpe, torch.int64, E).copy_(torch.bincount(idx.flatten(), minlength=E))
        return 0

    def xtb_gate_route_replay_dispatch(self, x, w, replay, stride, T, H, E, K, scoring, norm, scaling, logits, rw, tw, ids,
                                       ids32, tpe, ws, stream):
        self.calls.append("xtb_gate_route_replay_dispatch")
        if E > 8 or K > 8 or H % 128 or H > 4224:
            return 1
        self.xtb_gate_logits(x, w, None, logits, T, H, E, stream)
        rc = self.xtb_router_greedy_replay(logits, replay, stride, T, E, K, scoring, norm, scaling, rw, tw, ids, ids32, tpe,
                                           ws, stream)
        self.calls = self.calls[:-2]
        return rc

    def xtb_router_noaux_replay(self, logits, bias, replay, stride, T, E, K, n_group, topk_group, norm, scaling, rw, tw,
                                ids, ids32, tpe, stream):
        self.calls.append("xtb_router_noaux_replay")
        idx, bad = _sanitise(_rows(replay, T, K, stride).clone(), E)
        r, w, _ = noaux_replay_reference(_view(logits, torch.float32, T, E), _view(bias, torch.float32, E), idx, K, n_group,
                                         topk_group, bool(norm), scaling)
        _view(rw, torch.float32, T, E).copy_(r)
        _view(tw, torch.float32, T, K).copy_(torch.where(bad, float("nan"), w))
        _view(ids, torch.int64, T, K).copy_(idx)
        if ids32 is not None:
            _view(ids32, torch.int32, T, K).copy_(idx.int())
        _view(tpe, torch.float32, E).copy_(torch.bincount(idx.flatten(), minlength=E).float())
        return 0


@pytest.fixture
def emu(monkeypatch):
    from xtuner_b200 import _capi, fused, ops, router

    lib = ReplayEmulatedLib(_capi.load())
    monkeypatch.setattr(_capi, "ensure_init", lambda: lib)
    for mod in (ops, router, fused):
        monkeypatch.setattr(mod, "current_stream", lambda: None)
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "permute_workspace", lambda T, K, E, dev: torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8))
    monkeypatch.setattr(ops, "_scratch", lambda tag, n, dev: torch.empty(max(int(n), 16), dtype=torch.uint8))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))  # the routers' and fused node's guards
    return lib


@pytest.mark.parametrize("case", fixture_case_names())
def test_routers_over_the_emulated_entries_reproduce_the_fixture(emu, gold, case):
    """the shipped routers and custom ops (argument order, strides, autograd wiring, the existing backward entries) on
    the fixture's logits and ids"""
    from xtuner_b200 import router

    kind, E, K, a, b, scaling = fixture_config(case)
    if kind == "greedy":
        r = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K, norm_topk_prob=b, scoring_func=a,
                                router_scaling_factor=scaling)
    else:
        r = router.NoAuxRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=scaling,
                               scoring_func="sigmoid", n_group=a, topk_group=b)
        r.e_score_correction_bias = gold[f"{case}.bias"].clone()
    for pat in PATTERNS:
        ids = fixture_ids(gold, case, pat)
        lg = gold[f"{case}.logits"].clone().requires_grad_(True)
        res = r(lg, ids)
        assert torch.equal(res["topk_ids"], ids) and torch.equal(r.last_topk_ids_i32, ids.int())
        assert torch.equal(res["router_weights"], gold[f"{case}.router_weights"])
        assert torch.equal(res["topk_weights"], gold[f"{case}.{pat}.topk_weights"])
        assert torch.equal(res["topkens_per_expert"].double(), gold[f"{case}.{pat}.tokens_per_expert"].double())
        ((res["topk_weights"] * gold[f"{case}.{pat}.g_tw"]).sum() + (res["router_weights"] * gold[f"{case}.g_rw"]).sum()).backward()
        torch.testing.assert_close(lg.grad, gold[f"{case}.{pat}.grad_logits"], rtol=1e-5, atol=1e-6, msg=lambda m: f"{pat}: {m}")


def _ids(T, E, K, seed, L=3, layer=1):
    """the [:, layer, :] slice of an [T, L, K] id tensor, with duplicates in every third row"""
    g = torch.Generator().manual_seed(seed)
    full = torch.randint(0, E, (T, L, K), generator=g)
    full[::3, layer, 0] = full[::3, layer, -1]
    return full[:, layer, :]


@pytest.mark.parametrize("E,K,scoring,norm,scaling", [(8, 2, "softmax", True, 1.0), (128, 8, "sigmoid", False, 2.5),
                                                      (8, 1, "sigmoid", True, 1.5)])
def test_greedy_router_replays_and_routes_the_gradients(emu, E, K, scoring, norm, scaling):
    from xtuner_b200 import router

    T = 40
    ids = _ids(T, E, K, E + K)
    assert ids.stride() == (3 * K, 1)
    lg = torch.randn(T, E, generator=torch.Generator().manual_seed(1)) * 2
    r = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K, norm_topk_prob=norm, scoring_func=scoring,
                            router_scaling_factor=scaling)
    a = lg.clone().requires_grad_(True)
    res = r(a, ids)
    assert emu.calls == ["xtb_router_greedy_replay"]
    assert torch.equal(res["topk_ids"], ids) and torch.equal(r.last_topk_ids_i32, ids.int())
    b = lg.clone().requires_grad_(True)
    p, w, hist = greedy_replay_reference(b, ids, norm, scaling, scoring)
    assert torch.equal(res["topkens_per_expert"], hist)
    torch.testing.assert_close(res["topk_weights"], w, rtol=0, atol=0)
    g = torch.Generator().manual_seed(2)
    g_tw, g_rw = torch.randn(T, K, generator=g), torch.randn(T, E, generator=g)
    (res["topk_weights"] * g_tw).sum().add((res["router_weights"] * g_rw).sum()).backward()
    (w * g_tw).sum().add((p * g_rw).sum()).backward()
    assert emu.calls == ["xtb_router_greedy_replay", "xtb_router_greedy_bwd"]
    torch.testing.assert_close(a.grad, b.grad, rtol=1e-5, atol=1e-6)
    with pytest.raises(TypeError):
        r(lg, ids.int())


@pytest.mark.parametrize("n_group,topk_group", [(8, 4), (8, 8)])
def test_noaux_router_replays_and_routes_the_gradients(emu, n_group, topk_group):
    from xtuner_b200 import router

    T, E, K = 24, 256, 8
    g = torch.Generator().manual_seed(n_group + topk_group)
    lg = torch.randn(T, E, generator=g)
    r = router.NoAuxRouter(n_routed_experts=E, num_experts_per_tok=K, router_scaling_factor=2.5, scoring_func="sigmoid",
                           n_group=n_group, topk_group=topk_group)
    with torch.no_grad():
        r.e_score_correction_bias.copy_(torch.randn(E, generator=g) * 0.1)
    # ids the router would never pick: the experts of its masked groups and its lowest scores
    ids = _ids(T, E, K, 5).clone()
    ids[:4] = lg[:4].argsort(1)[:, :K]
    a = lg.clone().requires_grad_(True)
    res = r(a, ids)
    assert emu.calls == ["xtb_router_noaux_replay"] and torch.equal(res["topk_ids"], ids)
    b = lg.clone().requires_grad_(True)
    rw, w, hist = noaux_replay_reference(b, r.e_score_correction_bias, ids, K, n_group, topk_group, True, 2.5)
    assert torch.equal(res["topkens_per_expert"], hist)
    torch.testing.assert_close(res["topk_weights"], w, rtol=0, atol=0)
    g_tw, g_rw = torch.randn(T, K, generator=g), torch.randn(T, E, generator=g)
    (res["topk_weights"] * g_tw).sum().add((res["router_weights"] * g_rw).sum()).backward()
    (w * g_tw).sum().add((rw * g_rw).sum()).backward()
    torch.testing.assert_close(a.grad, b.grad, rtol=1e-4, atol=1e-5)


def test_out_of_range_ids_are_sanitised(emu):
    from xtuner_b200 import router

    T, E, K = 6, 8, 2
    ids = torch.tensor([[0, 1], [-1, 2], [3, 8], [4, 2 ** 40], [5, 5], [6, 7]])
    res = router.GreedyRouter(n_routed_experts=E, num_experts_per_tok=K)(torch.randn(T, E), ids)
    assert res["topk_ids"].tolist() == [[0, 1], [0, 2], [3, 0], [4, 0], [5, 5], [6, 7]]
    assert torch.isnan(res["topk_weights"][1:4]).all() and torch.isfinite(res["topk_weights"][[0, 4, 5]]).all()
    assert res["topkens_per_expert"].tolist() == [4, 1, 1, 1, 1, 2, 1, 1]


@pytest.mark.parametrize("E,H", [(8, 256), (16, 256), (8, 192)])
def test_fused_node_replays_on_both_gate_paths(emu, E, H):
    """E <= 8 and H % 128 == 0: the one-launch entry; otherwise the gate and the replay router as two calls"""
    from xtuner_b200 import fused

    T, I, K = 32, 128, 2
    g = torch.Generator().manual_seed(E + H)
    h = torch.randn(T, H, generator=g).to(torch.bfloat16)
    nw = torch.ones(H)
    gw = torch.randn(E, H, generator=g) * 0.05
    w13 = (torch.randn(E, 2 * I, H, generator=g) * 0.05).to(torch.bfloat16)
    w2 = (torch.randn(E, H, I, generator=g) * 0.05).to(torch.bfloat16)
    ids = _ids(T, E, K, 3)
    x = h.clone().requires_grad_(True)
    out, rr = fused.fused_moe(x, None, gw, w13, w2, top_k=K, rollout_routed_experts=ids)
    want = "xtb_gate_route_replay_dispatch" if E <= 8 and H % 128 == 0 else "xtb_router_greedy_replay"
    assert want in emu.calls and torch.equal(rr["topk_ids"], ids)
    # the per-op composition with the same ids
    logits = h.float() @ gw.t()
    p, w, _ = greedy_replay_reference(logits, ids, True, 1.0, "softmax")
    ref = torch.zeros(T, H)
    for e in range(E):
        tok, slot = (ids == e).nonzero(as_tuple=True)
        if tok.numel():
            hh = (h[tok] @ w13[e].t()).float()
            a = O.swiglu(hh.to(torch.bfloat16)).float()
            ref.index_add_(0, tok, (a.to(torch.bfloat16) @ w2[e].t()).float() * w[tok, slot, None])
    torch.testing.assert_close(out.float(), ref, rtol=3e-2, atol=3e-2)
    out.float().sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad.float()).all()


# ---- the reference's models ---------------------------------------------------------------------------------------------


def _ref_helpers():
    from tests import test_plugin_reference_cpu as P

    if not P.ref_shim.reference_available():
        pytest.skip("no reference checkout found")
    return P


def _loss_and_grads(model, cfg, replay, offload=False):
    from xtuner.v1.loss.ce_loss import CELossConfig
    from xtuner.v1.model.moe.moe import SequenceContext

    torch.manual_seed(123)
    input_ids = torch.randint(0, cfg.vocab_size, (1, 65), dtype=torch.int64)
    seq_ctx = SequenceContext.from_input_ids(input_ids=(input_ids[:, :-1],), device="cpu")
    seq_ctx.rollout_routed_experts = replay
    seq_ctx.offload_rollout_routed_experts = offload
    loss_cfg = CELossConfig()
    lctx = loss_cfg.build(data={"shifted_labels": input_ids[:, 1:]}, sp_mesh=None)
    lctx = loss_cfg.loss_ctx_cls.build_batches([lctx])[0]
    model.zero_grad(set_to_none=True)
    out = model(seq_ctx=seq_ctx, loss_ctx={"lm": lctx})
    fields = {k: getattr(out, k) for k in type(out).model_fields} if hasattr(type(out), "model_fields") else dict(out)
    total = sum(v for k, v in fields.items() if "loss" in k and isinstance(v, torch.Tensor) and v.requires_grad)
    total.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    return {k: v.detach().clone() for k, v in fields.items() if isinstance(v, torch.Tensor) and v.numel() == 1}, grads


def _dispatched_ids(model, monkeypatch):
    """records the topk ids every FusedDispatcher / fused node receives"""
    from xtuner_b200 import dispatcher, fused

    seen = []
    orig = dispatcher.FusedDispatcher.dispatch_preprocess

    def spy(self, *, hidden_states, topk_ids, topk_weights, **kw):
        seen.append(topk_ids.clone())
        return orig(self, hidden_states=hidden_states, topk_ids=topk_ids, topk_weights=topk_weights, **kw)

    monkeypatch.setattr(dispatcher.FusedDispatcher, "dispatch_preprocess", spy)
    orig_block = fused.fused_moe_block

    def block_spy(*a, **kw):
        out, rr = orig_block(*a, **kw)
        seen.append(rr["topk_ids"].clone())
        return out, rr

    monkeypatch.setattr(fused, "fused_moe_block", block_spy)
    return seen


def _compare(ref, ours, loss_tol, grad_check):
    ref_out, ref_grads = ref
    our_out, our_grads = ours
    for k, v in ref_out.items():
        torch.testing.assert_close(our_out[k], v, rtol=loss_tol, atol=loss_tol * 0.1, msg=lambda m, k=k: f"{k}: {m}")
    assert set(our_grads) == set(ref_grads)
    for k in ref_grads:
        grad_check(our_grads[k].float(), ref_grads[k].float(), k)


def _close(a, b, k):
    torch.testing.assert_close(a, b, rtol=2e-3, atol=2e-5, msg=lambda m: f"grad {k}: {m}")


def _mostly_close(a, b, k):
    bad = ((a - b).abs() > 3e-2 * (b.abs() + b.abs().mean())).float().mean()
    assert bad < 5e-3, f"grad {k}: {bad:.4f} of elements off"


@pytest.mark.parametrize("mode", ["per_op", "fused"])
@pytest.mark.parametrize("noaux", [False, True])
def test_reference_models_with_rollout_routed_experts(monkeypatch, emu, mode, noaux):
    import torch.distributed as dist

    P = _ref_helpers()
    if noaux and mode == "fused":
        pytest.skip("no-aux layers are not fused-eligible: covered by the per-op case")
    if not dist.is_initialized():
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29711", RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
        dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: False))  # the reference model builds on host
        model, cfg = P._build_reference_model(0, noaux=noaux, hidden=256 if mode == "fused" else 64)
        E, K, S = cfg.n_routed_experts, cfg.num_experts_per_tok, 64
        # ids for layer 0 only: layer 1 (layer_idx >= shape[1]) routes itself, as in the reference
        full = torch.randint(0, E, (S, 1, K), generator=torch.Generator().manual_seed(4))
        full[::3, 0, 0] = full[::3, 0, -1]
        ref = _loss_and_grads(model, cfg, full)
        from xtuner_b200 import plugin

        seen = _dispatched_ids(model, monkeypatch)
        monkeypatch.setattr(plugin, "_gg_eligible", lambda x, w: True)
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
        assert plugin.convert_model(model, fused=(mode == "fused")) == cfg.num_hidden_layers
        ours = _loss_and_grads(model, cfg, full)
        assert torch.equal(seen[0], full[:, 0, :]), "the replayed ids reach the dispatcher"
        assert len(seen) == 2 and not torch.equal(seen[1], full[:, 0, :])
        _compare(ref, ours, 2e-4, _mostly_close if mode == "fused" else _close)
        # with the offload flag set: the result must not change (both sides are host memory here, so nothing moves; the
        # move itself is checked by test_fused_layer_moves_an_offloaded_slice_to_the_device and by the GPU worker)
        seen.clear()
        again = _loss_and_grads(model, cfg, full, offload=True)
        assert torch.equal(seen[0], full[:, 0, :])
        assert torch.equal(again[0]["loss"], ours[0]["loss"])
        plugin.restore_model(model)
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def test_fused_layer_moves_an_offloaded_slice_to_the_device(monkeypatch):
    """``_fused_layer_forward`` slices ``[:, layer_idx, :]`` and, with ``offload_rollout_routed_experts`` and a tensor on
    another device, makes it contiguous and moves it (moe_decoder_layer.py:669-677)"""
    from types import SimpleNamespace

    from xtuner_b200 import fused, plugin

    got = {}

    def block(h, *a, rollout_routed_experts=None, **kw):
        got["ids"] = rollout_routed_experts
        return h, {"logits": None, "router_weights": None, "topk_ids": None}

    monkeypatch.setattr(fused, "fused_moe_block", block)
    moved = []
    full = torch.arange(4 * 3 * 2).view(4, 3, 2)

    class FakeIds:
        shape = full.shape

        def __getitem__(self, idx):
            sl = full[idx]

            class Slice:
                device = torch.device("meta")

                def contiguous(self):
                    moved.append("contiguous")
                    return self

                def to(self, dev):
                    moved.append(dev)
                    return sl.contiguous()

            return Slice()

    norm = SimpleNamespace(weight=torch.ones(8), variance_epsilon=1e-6)
    layer = SimpleNamespace(
        input_layernorm=lambda h: h, self_attn=lambda **kw: {"projected_output": torch.zeros_like(kw["hidden_states"])},
        post_attention_layernorm=norm, gate=SimpleNamespace(weight=torch.ones(2, 8), router=SimpleNamespace(
            top_k=2, norm_topk_prob=True, router_scaling_factor=1.0, scoring_func="softmax")),
        experts=SimpleNamespace(fused_w1w3=SimpleNamespace(weight=None), fused_w2=SimpleNamespace(weight=None)),
        hidden_factor=1.0, layer_idx=1)
    h = torch.zeros(1, 4, 8)
    seq_ctx = SimpleNamespace(rollout_routed_experts=FakeIds(), offload_rollout_routed_experts=True)
    plugin._fused_layer_forward(layer, h, seq_ctx, None)
    assert moved == ["contiguous", h.device] and torch.equal(got["ids"], full[:, 1, :])
    layer.layer_idx = 3  # past the tensor's layer count: no replay
    got.clear()
    plugin._fused_layer_forward(layer, h, seq_ctx, None)
    assert got == {"ids": None}
    seq_ctx = SimpleNamespace(rollout_routed_experts=full, offload_rollout_routed_experts=False)
    layer.layer_idx = 2
    plugin._fused_layer_forward(layer, h, seq_ctx, None)
    assert torch.equal(got["ids"], full[:, 2, :]) and got["ids"].data_ptr() == full[:, 2, :].data_ptr()
