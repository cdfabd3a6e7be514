"""Drop-in conformance (CPU): the host-side mirror must expose the reference's seams with the same names, keyword
arguments and result keys (SURVEY.md §8b).  The reference's side of every comparison was recorded from its own classes
by ``tests/golden/make_reference_api.py`` into ``tests/golden/reference_api.json``."""
import inspect
import json
import os
import sys
import types

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ref():
    with open(os.path.join(HERE, "golden", "reference_api.json")) as f:
        return json.load(f)


def _params(fn):
    return [[n, int(p.kind), p.default is not inspect.Parameter.empty] for n, p in inspect.signature(fn).parameters.items() if n != "self"]


def test_dispatcher_methods_match_generic_dispatcher(ref):
    from xtuner_b200.dispatcher import FusedDispatcher

    abstract = ref["dispatcher_abstract_methods"]
    assert abstract == ["combine", "combine_postprocess", "combine_preprocess", "dispatch", "dispatch_postprocess", "dispatch_preprocess"]
    for name in abstract:
        op, tp = _params(getattr(FusedDispatcher, name)), ref["naive_dispatcher_methods"][name]
        assert [n for n, _, _ in op] == [n for n, _, _ in tp], (name, op, tp)
        assert all(k == inspect.Parameter.KEYWORD_ONLY for _, k, _ in op), f"{name}: keyword-only like the reference"
    # constructor keywords accepted by build_dispatcher (dispatcher/__init__.py:30-96) for the ep=1 case
    ctor = [n for n, _, _ in _params(FusedDispatcher.__init__)]
    for kw in ("n_routed_experts", "process_group", "training_dtype", "generate_dtype"):
        assert kw in ctor


def test_op_protocol_signatures(ref):
    from xtuner_b200 import ops

    def names(fn):
        return [n for n, p in inspect.signature(fn).parameters.items() if n != "self" and p.kind != inspect.Parameter.KEYWORD_ONLY]

    assert names(ops.group_gemm) == ref["op_protocols"]["group_gemm"]
    assert names(ops.permute) == ref["op_protocols"]["permute"]
    assert names(ops.unpermute) == ref["op_protocols"]["unpermute"]


def test_router_results_keys_and_ctor(ref):
    from xtuner_b200.router import GreedyRouter, NoAuxRouter, RouterResults

    assert sorted(RouterResults.__annotations__) == ref["router_results_keys"]
    assert [n for n, _, _ in _params(GreedyRouter.__init__)] == [n for n, _, _ in ref["greedy_router_init"]]
    assert [n for n, _, _ in _params(NoAuxRouter.__init__)] == [n for n, _, _ in ref["noaux_router_init"]]
    assert [n for n, _, _ in _params(GreedyRouter.forward)] == [n for n, _, _ in ref["greedy_router_forward"]]


def test_ulysses_all_to_all_signature(ref):
    from xtuner_b200.comm import ulysses_all_to_all

    assert list(inspect.signature(ulysses_all_to_all).parameters) == ref["ulysses_all_to_all"]


def test_state_dict_keys_match_reference_modules(ref):
    import torch

    from xtuner_b200.moe import MoELayer

    H, I, E, K = 64, 32, 4, 2  # the sizes the reference's MoEGate + MoEBlock were built with for the record
    ref_keys = {k: torch.Size(v) for k, v in ref["moe_layer_state_dict"].items()}
    ours = MoELayer(hidden_size=H, moe_intermediate_size=I, n_routed_experts=E, num_experts_per_tok=K)
    our_keys = {k: v.shape for k, v in ours.state_dict().items()}
    assert our_keys == ref_keys, (our_keys, ref_keys)
    assert all(isinstance(v, torch.Size) for v in our_keys.values())


def test_install_ulysses_rebinds_mha_global(ref, monkeypatch):
    """The reference's mha.py holds ``ulysses_all_to_all`` as a module global imported by value (recorded); the plugin rebinds
    that global and puts it back.  The module here is a stand-in with that one global under the reference module's name."""
    assert ref["mha_imports_ulysses_all_to_all_by_value"]
    mha = types.ModuleType("xtuner.v1.module.attention.mha")
    mha.ulysses_all_to_all = lambda *a, **k: None
    monkeypatch.setitem(sys.modules, mha.__name__, mha)
    from xtuner_b200 import comm, plugin

    orig = mha.ulysses_all_to_all
    plugin.install_ulysses()
    try:
        assert mha.ulysses_all_to_all is comm.ulysses_all_to_all
    finally:
        plugin.uninstall_ulysses()
    assert mha.ulysses_all_to_all is orig


def test_install_fsdp_comm_on_fully_sharded_module():
    """FSDP2 wiring on CPU (gloo, 1 rank): every FSDPModule gets our comm objects through torch's own setters."""
    import torch
    import torch.distributed as dist
    from torch import nn
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.fsdp import fully_shard

    from xtuner_b200 import comm, plugin

    created = False
    if not dist.is_initialized():
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29689", RANK="0", WORLD_SIZE="1", LOCAL_RANK="0")
        dist.init_process_group("gloo", rank=0, world_size=1)
        created = True
    try:
        mesh = init_device_mesh("cpu", (1,))
        model = nn.Sequential(nn.Linear(16, 16), nn.Linear(16, 16))
        for blk in model:
            fully_shard(blk, mesh=mesh)
        fully_shard(model, mesh=mesh)
        n = plugin.install_fsdp_comm(model)
        assert n == 3
        for m in model.modules():
            state = getattr(m, "_get_fsdp_state", None)
            if state is None:
                continue
            pg = m._get_fsdp_state()._fsdp_param_group
            if pg is not None:
                assert isinstance(pg._all_gather_comm, comm.P2PAllGather)
                assert isinstance(pg._reduce_scatter_comm, comm.P2PReduceScatter)
    finally:
        if created:
            dist.destroy_process_group()
