"""Routing replay in the reference's own MoE models on an H100 (tests/workers/router_replay_worker.py): with
``seq_ctx.rollout_routed_experts`` set, ``convert_model`` per-op and ``fused=True`` train a step like the reference's own
GPU path — every layer routes exactly the replayed ids (replay removes the near-tie flips the routing comparison of
tests/test_gpu_reference_plugin.py tolerates beyond the first layer), loss within 1e-4 relative, gradients within that
test's bound — and ids offloaded to host memory are moved and give the same step."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HAVE_REF = os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "xtuner", "v1"))


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref absent (oracle/make_ref.py places the reference package there)")
def test_reference_models_replay_rollout_routed_experts_like_the_reference():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "workers", "router_replay_worker.py")], env=env, cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    lines = [l for l in r.stdout.splitlines() if l.startswith("ROUTERREPLAY ")]
    if r.returncode != 0 or not lines:
        err = "\n".join(l for l in r.stderr.splitlines() if "Warning" not in l and l.strip())
        raise AssertionError("router replay worker failed\nSTDOUT:\n" + r.stdout[-2000:] + "\nSTDERR:\n" + err[-6000:])
    d = json.loads(lines[-1][len("ROUTERREPLAY "):])
    for kind, modes in (("greedy", ("per_op", "fused")), ("noaux", ("per_op",))):
        ref = d[kind]["reference"]
        assert all(ref["ids_replayed"]), (kind, ref)
        noise = abs(ref["total"] - ref["rerun_total"]) / abs(ref["total"])
        for mode in modes:
            m = d[kind][mode]
            assert m["layers_converted"] == 2 and m["same_grad_keys"] and m["kernel_launches"] > 0, (kind, mode, m)
            assert all(m["ids_replayed"]), f"{kind}/{mode}: a layer did not route the replayed ids: {m['ids_replayed']}"
            assert m["loss_rel_diff"] <= max(1e-4, 2 * noise), f"{kind}/{mode}: loss differs by {m['loss_rel_diff']:.3e}"
            assert m["worst_grad_rel_to_max"] <= 5e-2, (kind, mode, m["worst_grad"], m["worst_grad_rel_to_max"])
            assert m["offload_same"], f"{kind}/{mode}: ids offloaded to host memory gave a different step"
