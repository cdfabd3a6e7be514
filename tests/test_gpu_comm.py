"""Multi-GPU parity of the peer-memory exchange kernels (needs >= 2 GPUs; skipped otherwise)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_comm_kernels_two_ranks():
    n = min(torch.cuda.device_count(), int(os.environ.get("XTB_TEST_WORLD", "2")))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(ROOT, "tests", "multigpu", "comm_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    if r.returncode != 0 or "COMM_WORKER_OK" not in r.stdout:
        err = "\n".join(l for l in r.stderr.splitlines() if "Warning" not in l and l.strip())
        raise AssertionError("comm worker failed\nSTDOUT:\n" + r.stdout[-2000:] + "\nSTDERR:\n" + err[-6000:])


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_fsdp2_custom_collectives():
    n = min(torch.cuda.device_count(), int(os.environ.get("XTB_TEST_WORLD", "2")))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29534", os.path.join(ROOT, "tests", "multigpu", "fsdp_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    if r.returncode != 0 or "FSDP_WORKER_OK" not in r.stdout:
        err = "\n".join(l for l in r.stderr.splitlines() if "Warning" not in l and l.strip())
        raise AssertionError("fsdp worker failed\nSTDOUT:\n" + r.stdout[-2000:] + "\nSTDERR:\n" + err[-6000:])


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_ep_dispatcher_gpu():
    """ep > 1 dispatchers (NCCL all-to-all and the device-driven peer exchange) against ep = 1, forward and backward, incl.
    async_op=True.  Not run on H100 (needs two GPUs)."""
    n = min(torch.cuda.device_count(), int(os.environ.get("XTB_TEST_WORLD", "2")))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29535", os.path.join(ROOT, "tests", "multigpu", "ep_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    if r.returncode != 0 or "EP_WORKER_OK" not in r.stdout:
        err = "\n".join(l for l in r.stderr.splitlines() if "Warning" not in l and l.strip())
        raise AssertionError("ep worker failed\nSTDOUT:\n" + r.stdout[-2000:] + "\nSTDERR:\n" + err[-6000:])


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_fsdp_expert_shards_step_matches_nccl_reference():
    """The FSDP expert-shard engine inside bench.py (4 layers): the exchange kernels bit-exact against NCCL, the sharded
    step against NCCL-gathered parameters / NCCL reduce-scattered gradients, then a CUDA-graph replay of the step with the
    exchange inside it (bench.fsdp_selfcheck raises on any mismatch)."""
    import json

    n = min(torch.cuda.device_count(), int(os.environ.get("XTB_TEST_WORLD", "2")))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}", "--master-addr", "127.0.0.1",
           "--master-port", "29537", os.path.join(ROOT, "bench.py"), "--gpus", str(n), "--layers", "4", "--steps", "2",
           "--warmup", "1", "--no-cpu-baseline"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        err = "\n".join(l for l in r.stderr.splitlines() if "Warning" not in l and l.strip())
        raise AssertionError("bench --gpus N (fsdp) failed\nSTDOUT:\n" + r.stdout[-2000:] + "\nSTDERR:\n" + err[-6000:])
    d = json.loads(lines[-1])
    assert d["n_gpus"] == n and d["config"]["parallelism"].startswith(f"fsdp={n}")
    assert d["selfcheck"]["all_gather_vs_nccl"] == "bit-exact"
    assert d["selfcheck"]["step_vs_nccl_reference"]["loss_rel_diff"] <= 1e-6
    assert d["roofline_comm"]["all_gather"]["us"] > 0 and d["roofline_comm"]["reduce_scatter"]["us"] > 0
