"""CPU-side checks (-m "not gpu"): the C-ABI library builds, loads, exports every symbol the header
declares, and refuses to compute without a GPU (no silent fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g

    g.build()
    from xtuner_b200 import _capi

    return _capi.load()


def test_header_symbols_exported(lib):
    from xtuner_b200 import _capi

    header = open(os.path.join(ROOT, "include", "xtuner_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(xtb_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(_capi.SIGNATURES), (declared ^ set(_capi.SIGNATURES))
    for name in declared:
        assert hasattr(lib, name), f"{name} not exported"


def test_version_and_error_string(lib):
    assert lib.xtb_version() == 100
    assert lib.xtb_launch_count() >= 0


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_no_cpu_fallback(lib):
    from xtuner_b200 import _capi, ops

    assert lib.xtb_init() != 0
    assert b"no CUDA device" in lib.xtb_last_error() or b"failed" in lib.xtb_last_error()
    x = torch.zeros(4, 128, dtype=torch.bfloat16)
    with pytest.raises(_capi.XtbError):
        ops.permute(x, torch.zeros(4, 2, dtype=torch.int32), n_experts=8)
    with pytest.raises(_capi.XtbError):
        ops.group_gemm(x, torch.zeros(2, 128, 128, dtype=torch.bfloat16), torch.tensor([2, 2]))
    with pytest.raises(_capi.XtbError):
        ops.unpermute(x, torch.zeros(4, dtype=torch.int32), None)


def test_argument_validation_is_host_side(lib):
    # invalid shapes are rejected before any CUDA call
    rc = lib.xtb_group_gemm_nt(1, 1, 1, 10, 100, 128, 4, 1, None)
    assert rc == 1 and b"multiples of 128" in lib.xtb_last_error()
    rc = lib.xtb_moe_unpermute(1, 1, None, 4, 2, 7, 1, None)
    assert rc == 1
    assert lib.xtb_moe_permute_workspace_bytes(8192, 2, 8) > 0


def test_swiglu_and_fp8_alignment_and_grid_limits_are_host_side(lib):
    """The SwiGLU kernels move 16-byte vectors, the fp8 tile kernel 8-byte loads and 4-byte stores, and the fp8 block
    kernels put one matrix per grid z index: a pointer or count they cannot take is refused before any CUDA call.  The
    pointer values are never dereferenced."""
    A = 1 << 20  # a 16-byte aligned fake address
    for args in ((A + 8, A), (A, A + 2)):
        assert lib.xtb_swiglu(*args, 4, 64, None) == 1 and b"16-byte aligned" in lib.xtb_last_error()
    for args in ((A + 8, A, A), (A, A + 4, A), (A, A, A + 2)):
        assert lib.xtb_swiglu_bwd(*args, 4, 64, None) == 1 and b"16-byte aligned" in lib.xtb_last_error()
    for args in ((A + 4, A, A), (A, A + 2, A), (A, A, A + 2)):
        assert lib.xtb_fp8_per_tile_quant(*args, 4, 128, None) == 1 and b"aligned" in lib.xtb_last_error()
    assert lib.xtb_fp8_block_scales(A, 1, 65536, 128, 128, A, None) == 1 and b"65535" in lib.xtb_last_error()
    assert lib.xtb_fp8_block_cast(A, 0, 65536, 128, 128, A, A, None) == 1 and b"65535" in lib.xtb_last_error()
    # the widest SwiGLU backward row the 32-bit reciprocal row split takes is I = 8 * 23170
    assert lib.xtb_swiglu_bwd(A, A, A, 4, 8 * 23171, None) == 1 and b"too wide" in lib.xtb_last_error()


def test_every_compute_entry_rejects_null_pointers_on_the_host(lib):
    """Error behaviour of the boundary: a bad call returns XTB_ERR_INVALID (1) with a message naming the entry point —
    before any CUDA call, so it holds without a GPU — instead of crashing."""
    import ctypes

    from xtuner_b200 import _capi

    admin = {"xtb_version", "xtb_last_error", "xtb_init", "xtb_launch_count", "xtb_reset_launch_count"}
    checked = 0
    for name, (_res, args) in _capi.SIGNATURES.items():
        if name in admin or name.endswith("workspace_bytes"):
            continue
        vals = [0.0 if a is ctypes.c_float else (None if a is ctypes.c_void_p else 0) for a in args]
        rc = getattr(lib, name)(*vals)
        msg = lib.xtb_last_error()
        assert rc == 1, (name, rc, msg)
        assert msg.startswith(b"xtb_") and (b"null pointer" in msg or b"required" in msg), (name, msg)
        checked += 1
    assert checked >= 29
