"""Recipe for ``oracle/_ref``: a git-ignored copy of the reference project's pure-Python ``xtuner`` package for the tests
that run the reference's own model code and for the generators under ``tests/golden``.  The reference checkout is looked
for in ``$XTUNER_REFERENCE_SRC``, then as a directory ``reference`` next to this repository, in the home directory or in a
top-level directory; where there is none, nothing is made and those tests skip."""
from __future__ import annotations

import glob
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def find_reference() -> str | None:
    cands = [os.environ.get("XTUNER_REFERENCE_SRC"), os.path.join(os.path.dirname(ROOT), "reference"),
             os.path.join(os.path.expanduser("~"), "reference"), *sorted(glob.glob("/*/reference"))]
    for c in cands:
        if c and os.path.isdir(os.path.join(c, "xtuner", "v1")):
            return c
    return None


def make_ref() -> str | None:
    if os.path.isdir(os.path.join(REF_DIR, "xtuner", "v1")):
        return REF_DIR
    src = find_reference()
    if src is None:
        return None
    tmp = REF_DIR + f".tmp{os.getpid()}"
    try:
        shutil.copytree(os.path.join(src, "xtuner"), os.path.join(tmp, "xtuner"), ignore=shutil.ignore_patterns("__pycache__"))
        os.replace(tmp, REF_DIR)
    except OSError:  # unreadable source, read-only tree, or a copy placed meanwhile
        shutil.rmtree(tmp, ignore_errors=True)
    return REF_DIR if os.path.isdir(os.path.join(REF_DIR, "xtuner", "v1")) else None
