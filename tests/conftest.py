import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


def pytest_collection_modifyitems(config, items):
    """gpu-marked tests skip (instead of failing with 'Found no NVIDIA driver') when a plain `pytest` runs them on a box
    without CUDA; on a GPU box nothing changes."""
    try:
        import torch

        has_cuda = torch.cuda.is_available()
    except Exception:  # noqa: BLE001
        has_cuda = False
    if has_cuda:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100); run with -m gpu")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def load_golden(name):
    """``<name>.pt``, or for a large fixture ``<name>.part<i>.pt``: lists of (key path, value) merged into one dict."""
    import glob

    import torch

    whole = os.path.join(GOLDEN_DIR, name + ".pt")
    if os.path.exists(whole):
        return torch.load(whole, weights_only=False)
    parts = sorted(glob.glob(os.path.join(GOLDEN_DIR, name + ".part*.pt")))
    if not parts:
        raise FileNotFoundError(whole)
    out = {}
    for part in parts:
        for path, value in torch.load(part, weights_only=False):
            d = out
            for key in path[:-1]:
                d = d.setdefault(key, {})
            d[path[-1]] = value
    return out


@pytest.fixture
def golden():
    return load_golden
