"""tests/gpu_harness.Guarded on CPU tensors, for every output dtype the GPU tests give it.  Each failure must name the
count and the first (row, column).  The modes and the GPU tests that use them:

* every row written (the default): the grouped GEMM, SwiGLU, lm_head, norm/combine and router outputs;
* a row mask: the unpermute backward, whose permuted rows that no entry references must keep the fill;
* nothing written: the entries at T = 0, and g_norm_w when the dispatch backward is not asked for it;
* guards only: the gate backward's grad_x, and the lm_head loss and dW at T = 0."""
import re

import pytest
import torch

from tests.gpu_harness import GUARD, Guarded

DTYPES = [torch.bfloat16, torch.float32, torch.int32, torch.int64]
ROWS, COLS = 5, 7


def _fails(g, what, count, msg, row, col, **kw):
    with pytest.raises(AssertionError, match=re.escape(f"{what}: {count} {msg}; first at row {row}, column {col}")):
        g.check(what, **kw)


@pytest.mark.parametrize("dtype", DTYPES)
def test_fill_and_layout(dtype):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    assert g.v.dtype == dtype and g.v.shape == (ROWS, COLS)
    assert g.buf.shape == (ROWS + 2 * GUARD, COLS) and g.buf.element_size() == dtype.itemsize
    assert GUARD == 16 and g.fill == {2: 0x7FA5, 4: 0x7FC0A5A5, 8: 0x7FA5A5A5A5A5A5A5}[dtype.itemsize]
    assert bool((g.buf == g.fill).all())
    assert g.v.data_ptr() == g.buf[GUARD].data_ptr()


@pytest.mark.parametrize("dtype", DTYPES)
def test_fully_written_passes(dtype):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    g.v.fill_(1)
    assert g.check("out") is g.v
    g.check("out", written=None)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["all", "mask", "none", "guards"])
def test_a_guard_write_fails_in_every_mode(dtype, mode):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    mask = torch.tensor([True, False, True, True, False])
    written = {"all": True, "mask": mask, "none": False, "guards": None}[mode]
    if mode in ("all", "guards"):
        g.v.fill_(1)
    elif mode == "mask":
        g.v[mask] = 1
    g.check("out", written=written)  # the rows in between are as the mode wants them
    g.buf[GUARD - 3, 4] = 0  # row -3
    g.buf[GUARD + ROWS + 2, 1] = 0  # row ROWS + 2
    _fails(g, "out", 2, "guard elements were written", -3, 4, written=written)


@pytest.mark.parametrize("dtype", DTYPES)
def test_one_unwritten_element_fails(dtype):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    g.v.fill_(1)
    g.buf[GUARD + 3, 5] = g.fill
    _fails(g, "out", 1, "output elements were never written", 3, 5)
    mask = torch.tensor([False, False, False, True, False])
    g.buf[GUARD : GUARD + ROWS] = g.fill
    g.v[3].fill_(1)
    g.buf[GUARD + 3, 6] = g.fill
    _fails(g, "masked", 1, "output elements were never written", 3, 6, written=mask)


@pytest.mark.parametrize("dtype", DTYPES)
def test_a_write_outside_the_mask_fails(dtype):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    mask = torch.tensor([True, False, True, False, False])
    g.v[mask] = 1
    assert g.check("masked", written=mask) is g.v
    g.v[3, 2] = 1
    g.v[4, 0] = 1
    _fails(g, "masked", 2, "elements outside the written rows were written", 3, 2, written=mask)


@pytest.mark.parametrize("dtype", DTYPES)
def test_any_write_fails_when_nothing_may_be_written(dtype):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    assert g.check("untouched", written=False) is g.v
    g.v[ROWS - 1, COLS - 1] = 0
    _fails(g, "untouched", 1, "elements outside the written rows were written", ROWS - 1, COLS - 1, written=False)


@pytest.mark.parametrize("dtype", DTYPES)
def test_guards_only_ignores_the_rows_in_between(dtype):
    g = Guarded(ROWS, COLS, dtype, device="cpu")
    g.check("guards", written=None)
    g.v[0, :3] = 1
    g.v[2] = 1
    assert g.check("guards", written=None) is g.v
    with pytest.raises(AssertionError):
        g.check("guards")
    with pytest.raises(AssertionError):
        g.check("guards", written=False)
