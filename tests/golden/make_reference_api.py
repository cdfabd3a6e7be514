"""Records from the REFERENCE'S OWN classes (imported through ``ref_shim``) what ``tests/test_dropin_conformance.py``
compares our drop-in classes with:  python tests/golden/make_reference_api.py  ->  tests/golden/reference_api.json"""
import inspect
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ref_shim.apply_cpu_patches()
import xtuner.v1.module.attention.mha as mha  # noqa: E402
from xtuner.v1.module.decoder_layer.moe_decoder_layer import MoEActFnConfig, MoEBlock, MoEGate  # noqa: E402
from xtuner.v1.module.dispatcher.base import GenericDispatcher, NaiveDispatcher  # noqa: E402
from xtuner.v1.module.router.greedy import GreedyRouter, GreedyRouterConfig  # noqa: E402
from xtuner.v1.module.router.noaux_router import NoAuxRouter  # noqa: E402
from xtuner.v1.module.router.protocol import RouterResults  # noqa: E402
from xtuner.v1.ops.comm.all_to_all import ulysses_all_to_all  # noqa: E402
from xtuner.v1.ops.moe.protocol import GroupGemmProtocol, MoePermuteProtocol, MoeUnpermuteProtocol  # noqa: E402


def params(fn):  # (name, kind, has default) of every parameter but self
    return [[n, int(p.kind), p.default is not inspect.Parameter.empty] for n, p in inspect.signature(fn).parameters.items() if n != "self"]


def positional(fn):
    return [n for n, k, _ in params(fn) if k != int(inspect.Parameter.KEYWORD_ONLY)]


H, I, E, K = 64, 32, 4, 2
gate = MoEGate(hidden_size=H, n_routed_experts=E, num_experts_per_tok=K,
               router_config=GreedyRouterConfig(scoring_func="softmax", router_scaling_factor=1.0, norm_topk_prob=True))
experts = MoEBlock(hidden_size=H, moe_intermediate_size=I, n_routed_experts=E, moe_act_fn_cfg=MoEActFnConfig())
state = {f"gate.{k}": list(v.shape) for k, v in gate.state_dict().items()}
state.update({f"experts.{k}": list(v.shape) for k, v in experts.state_dict().items()})
abstract = sorted(GenericDispatcher.__abstractmethods__)
api = {
    "dispatcher_abstract_methods": abstract,
    "naive_dispatcher_methods": {n: params(getattr(NaiveDispatcher, n)) for n in abstract},
    "op_protocols": {"group_gemm": positional(GroupGemmProtocol.__call__), "permute": positional(MoePermuteProtocol.__call__),
                     "unpermute": positional(MoeUnpermuteProtocol.__call__)},
    "router_results_keys": sorted(RouterResults.__annotations__),
    "greedy_router_init": params(GreedyRouter.__init__),
    "greedy_router_forward": params(GreedyRouter.forward),
    "noaux_router_init": params(NoAuxRouter.__init__),
    "ulysses_all_to_all": list(inspect.signature(ulysses_all_to_all).parameters),
    "mha_imports_ulysses_all_to_all_by_value": mha.ulysses_all_to_all is ulysses_all_to_all,
    "moe_layer_state_dict": state,  # H, I, E, K = 64, 32, 4, 2
}
with open(os.path.join(HERE, "reference_api.json"), "w") as f:
    f.write(json.dumps(api, sort_keys=True) + "\n")
