"""What the GPU tests that call the C-ABI directly share: the guard-banded output buffer, the worst-ratio reporter,
``XTB_ERR_INVALID`` and ``sm_count()``.  Importing it needs no GPU, so the suite collects on any machine."""
import contextlib

import pytest
import torch

XTB_ERR_INVALID = 1  # include/xtuner_b200.h
GUARD = 16  # rows of fill on each side of a guarded output
FILL16 = 0x7FA5  # a bf16 NaN no kernel produces
FILL32 = 0x7FC0A5A5  # an fp32 NaN no kernel produces; int32 outputs take it too
FILL64 = 0x7FA5A5A5A5A5A5A5
_WORD = {torch.bfloat16: (torch.int16, FILL16), torch.float32: (torch.int32, FILL32),
         torch.int32: (torch.int32, FILL32), torch.int64: (torch.int64, FILL64)}


def sm_count():
    return torch.cuda.get_device_properties().multi_processor_count


class Guarded:
    """A [rows, cols] output of ``dtype``: ``v`` is rows [GUARD, GUARD + rows) of ``buf``, a buffer of fill words."""

    def __init__(self, rows, cols, dtype, device="cuda"):
        word, self.fill = _WORD[dtype]
        self.rows = rows
        self.buf = torch.full((rows + 2 * GUARD, cols), self.fill, dtype=word, device=device)
        self.v = self.buf[GUARD : GUARD + rows].view(dtype)

    def check(self, what, written=True):
        """Asserts that the guard rows kept the fill and, by ``written``, which rows of ``v`` were written: True, all of
        them fully; a bool row mask, the masked rows fully and every other row not at all; False, none at all; None, not
        checked.  A failure gives the count and the first (row, column), rows numbered as in ``v`` (a guard row is
        negative or at least ``rows``).  Returns ``v``."""
        kept = self.buf == self.fill
        row = torch.arange(kept.shape[0], device=kept.device) - GUARD
        guard = ((row < 0) | (row >= self.rows))[:, None]
        _assert_none(~kept & guard, what, "guard elements were written")
        if written is not None:
            want = torch.zeros_like(guard)
            want[GUARD : GUARD + self.rows, 0] = written
            _assert_none(kept & want, what, "output elements were never written")
            _assert_none(~kept & ~want & ~guard, what, "elements outside the written rows were written")
        return self.v


def _assert_none(bad, what, msg):
    if bool(bad.any()):
        r, c = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} {msg}; first at row {r - GUARD}, column {c}")


class Worst(dict):
    """quantity -> the largest |err| / bound noted, printed as ``<tag>: <quantity>: <value:.4g>`` at the end of the
    module that binds ``fixture()``."""

    def __init__(self, tag):
        super().__init__()
        self.tag = tag

    def note(self, name, r):
        self[name] = max(self.get(name, 0.0), float(r))

    def fixture(self, around=contextlib.nullcontext):
        """A module-scoped autouse fixture for the module to bind to a name.  ``around()`` is a context manager entered
        before the module's first test and left after the maxima are printed, for lines of the module's own."""

        @pytest.fixture(scope="module", autouse=True)
        def report():
            with around():
                yield
                for k, v in sorted(self.items()):
                    print(f"{self.tag}: {k}: {v:.4g}")

        return report
