"""The one save-and-restore mechanism behind every reference seam ``xtuner_b200.plugin`` rebinds (``_rebind`` /
``_restore``): first on plain objects, then through each public install / uninstall pair on the reference's own classes,
modules and model, where uninstalling must put back exactly the objects that were there."""
import importlib
import os
import sys
import types

import pytest
from torch import nn

from xtuner_b200 import plugin

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import ref_shim  # noqa: E402


def _neg(x):
    return -x


# ---- the helpers on plain objects --------------------------------------------------------------------------------------


def test_class_entry_keeps_its_descriptor():
    class Base:
        @staticmethod
        def f(x):
            return x + 1

    raw = vars(Base)["f"]
    assert plugin._rebind(Base, f=_neg)
    assert vars(Base)["f"] is _neg and vars(Base)[plugin._SAVED] == {"f": raw}
    plugin._restore(Base)
    assert vars(Base)["f"] is raw and plugin._SAVED not in vars(Base)
    assert Base.f(1) == 2 and Base().f(1) == 2


def test_inherited_class_entry_is_inherited_again():
    class Base:
        def f(self):
            return "base"

    class Sub(Base):
        pass

    assert plugin._rebind(Sub, f=lambda self: "sub")
    assert Sub().f() == "sub" and Base().f() == "base"
    plugin._restore(Sub)
    assert "f" not in vars(Sub) and plugin._SAVED not in vars(Sub) and Sub().f() == "base"


def test_module_attribute():
    mod = types.ModuleType("seam_module")
    mod.fn = abs
    assert plugin._rebind(mod, fn=_neg)
    assert mod.fn is _neg
    plugin._restore(mod)
    assert vars(mod)["fn"] is abs and not hasattr(mod, plugin._SAVED)


def test_submodule_is_registered_again():
    class Parent(nn.Module):
        def __init__(self):
            super().__init__()
            self.child = nn.Linear(2, 2)

    parent = Parent()
    child, keys = parent.child, list(parent.state_dict())
    replacement = nn.Identity()
    assert plugin._rebind(parent, child=replacement)
    assert parent._modules["child"] is replacement and vars(parent)[plugin._SAVED] == {"child": child}
    plugin._restore(parent)
    assert parent._modules["child"] is child and "child" not in vars(parent) and plugin._SAVED not in vars(parent)
    assert list(parent.state_dict()) == keys


def test_instance_name_shadowing_a_class_method_is_absent_again():
    lin = nn.Linear(2, 2)
    assert plugin._rebind(lin, forward=_neg)
    assert vars(lin)["forward"] is _neg
    plugin._restore(lin)
    assert "forward" not in vars(lin) and plugin._SAVED not in vars(lin)
    assert lin.forward.__func__ is nn.Linear.forward


def test_second_rebind_is_refused_and_double_restore_is_harmless():
    obj = types.SimpleNamespace(a=1)
    plugin._restore(obj)  # nothing rebound yet
    assert plugin._rebind(obj, a=2)
    assert not plugin._rebind(obj, a=3)
    assert obj.a == 2 and vars(obj)[plugin._SAVED] == {"a": 1}
    plugin._restore(obj)
    plugin._restore(obj)
    assert vars(obj) == {"a": 1}


# ---- every seam on the reference -----------------------------------------------------------------------------------------

_MISSING = object()


@pytest.fixture
def ref():
    if not ref_shim.reference_available():
        pytest.skip("no reference checkout found")
    ref_shim.apply_cpu_patches()


def _held(owner, name):
    """what ``owner`` itself holds under ``name``: a registered submodule, its own attribute, or _MISSING"""
    if isinstance(owner, nn.Module) and name in owner._modules:
        return owner._modules[name]
    return vars(owner).get(name, _MISSING)


def _snapshot(names):
    return [_held(owner, name) for owner, name in names]


def _assert_held(names, objs):
    for (owner, name), obj in zip(names, objs):
        assert _held(owner, name) is obj, name


def _assert_installed(names, before):
    for (owner, name), obj in zip(names, before):
        assert _held(owner, name) is not obj, name


def _assert_restored(names, before):
    _assert_held(names, before)
    assert not any(plugin._SAVED in vars(owner) for owner, _ in names)


def _cycle(install, uninstall, names):
    """install (every name changes), install again (nothing changes), uninstall (exactly the originals, or the name
    absent again, and no saved dict left), uninstall again"""
    before = _snapshot(names)
    install()
    _assert_installed(names, before)
    installed = _snapshot(names)
    install()
    _assert_held(names, installed)
    uninstall()
    _assert_restored(names, before)
    uninstall()
    _assert_restored(names, before)
    return before


def _model():
    """the reference's MoE model with fused-eligible MoE layers and attention the q/k install takes (head dim 64, qk_norm)"""
    from xtuner.v1.model.moe.moe import MoE, MoEConfig
    from xtuner.v1.module.attention import MHAConfig
    from xtuner.v1.module.router import GreedyRouterConfig

    cfg = MoEConfig(
        vocab_size=512, max_position_embeddings=256, pad_token_id=0, eos_token_id=0, num_hidden_layers=2, hidden_size=64,
        intermediate_size=128, rms_norm_eps=1e-6, rope_theta=1e6, hidden_act="silu",
        attention=MHAConfig(num_attention_heads=4, num_key_value_heads=2, head_dim=64, qk_norm=True,
                            attn_impl="eager_attention"),
        tie_word_embeddings=False, n_routed_experts=8, n_shared_experts=0, num_experts_per_tok=2, first_k_dense_replace=0,
        hidden_factor=1.0, moe_intermediate_size=32,
        router=GreedyRouterConfig(scoring_func="softmax", router_scaling_factor=1.0, norm_topk_prob=True), compile_cfg=False,
    )
    return MoE(config=cfg)


def _moe_names(model):
    mgl = importlib.import_module("xtuner.v1.module.grouped_linear.moe_group_linear")
    layers = [m for m in model.modules() if "dispatcher" in vars(m)]
    assert layers
    return [(mgl, "group_gemm")] + [
        pair for layer in layers
        for pair in ((layer, "dispatcher"), (layer, "_forward"), (layer.gate, "router"), (layer.experts, "moe_act"))]


def _qk_names(model):
    mha = importlib.import_module("xtuner.v1.module.attention.mha")
    attns = [m for m in model.modules() if isinstance(m, mha.MultiHeadAttention)]
    assert attns
    return [pair for a in attns for pair in ((a, "apply_rotary_emb"), (a.q_norm, "forward"), (a.k_norm, "forward"))]


def test_convert_and_restore_model(ref):
    model = _model()
    names = _moe_names(model)
    counts = []

    def convert():
        counts.append(plugin.convert_model(model, fused=True, recompute="act"))

    before = _cycle(convert, lambda: plugin.restore_model(model), names)
    assert counts == [2, 0]
    assert [obj is _MISSING for (_, name), obj in zip(names, before) if name == "_forward"] == [True, True]
    convert()
    for layer in [owner for owner, name in names if name == "dispatcher"]:
        # the saved dict holds originals only: the recompute mode is bound into the installed forward
        assert set(vars(layer)[plugin._SAVED]) == {"dispatcher", "_forward"}
        assert layer._forward.__func__.keywords == {"recompute": "act"}
    plugin.restore_model(model)


def test_install_and_uninstall_qk_norm_rope(ref):
    model = _model()
    names = _qk_names(model)
    counts = []
    before = _cycle(lambda: counts.append(plugin.install_qk_norm_rope(model)),
                    lambda: plugin.uninstall_qk_norm_rope(model), names)
    assert counts == [2, 0]
    assert [obj is _MISSING for (_, name), obj in zip(names, before)] == [False, True, True] * 2


def test_install_and_uninstall_ulysses(ref):
    from xtuner_b200 import comm

    mha = importlib.import_module("xtuner.v1.module.attention.mha")
    _cycle(plugin.install_ulysses, plugin.uninstall_ulysses, [(mha, "ulysses_all_to_all")])
    plugin.install_ulysses()
    try:
        assert mha.ulysses_all_to_all is comm.ulysses_all_to_all and not hasattr(comm.ulysses_all_to_all, "__wrapped__")
    finally:
        plugin.uninstall_ulysses()


def test_install_and_uninstall_fp8_cast(ref):
    fu = importlib.import_module("xtuner.v1.float8.fsdp_utils")
    _cycle(plugin.install_fp8_cast, plugin.uninstall_fp8_cast,
           [(fu, "cast_to_per_block_fp8_with_scales"), (fu, "tensor_to_per_block_fp8_scales")])


def test_install_and_uninstall_lm_head_loss(ref):
    cls = importlib.import_module("xtuner.v1.loss.ce_loss").LMHeadLossContext
    _cycle(plugin.install_lm_head_loss, plugin.uninstall_lm_head_loss, [(cls, "eager_mode"), (cls, "chunk_mode")])


def test_install_and_uninstall_rl_lm_head(ref):
    lp = importlib.import_module("xtuner.v1.loss.rl_loss").LogProbContext
    grpo = importlib.import_module("xtuner.v1.rl.loss.grpo_loss").GRPOLossContext
    _cycle(plugin.install_rl_lm_head, plugin.uninstall_rl_lm_head, [(lp, "loss_fn"), (lp, "chunk_mode"), (grpo, "loss_fn")])


def test_install_and_uninstall_moe_aux_loss(ref):
    cls = importlib.import_module("xtuner.v1.loss.aux_loss").AuxLossContext
    _cycle(plugin.install_moe_aux_loss, plugin.uninstall_moe_aux_loss, [(cls, "accumulate")])


@pytest.mark.parametrize("qk_first", [False, True])
def test_moe_conversion_and_qk_install_are_undone_independently(ref, qk_first):
    """both seams on one model, installed in either order: undoing the one installed first leaves the other in place"""
    model = _model()
    seams = [
        (lambda: plugin.convert_model(model, fused=True, recompute="act"), lambda: plugin.restore_model(model),
         _moe_names(model)),
        (lambda: plugin.install_qk_norm_rope(model), lambda: plugin.uninstall_qk_norm_rope(model), _qk_names(model)),
    ]
    if qk_first:
        seams.reverse()
    (install_a, undo_a, names_a), (install_b, undo_b, names_b) = seams
    before_a, before_b = _snapshot(names_a), _snapshot(names_b)
    install_a()
    install_b()
    _assert_installed(names_a, before_a)
    _assert_installed(names_b, before_b)
    installed_b = _snapshot(names_b)
    undo_a()
    _assert_restored(names_a, before_a)
    _assert_held(names_b, installed_b)
    undo_b()
    _assert_restored(names_b, before_b)
    _assert_restored(names_a, before_a)
