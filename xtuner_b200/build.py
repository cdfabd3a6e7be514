"""Builds the C-ABI CUDA library (``xtuner_b200/lib/libxtuner_b200.so``) for sm_90a with nvcc.

In-tree build: the ``.so`` and the build stamp next to it are git-ignored.  nvcc cross-compiles without a GPU, so this is
also the CPU-side "does it build" check.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libxtuner_b200.so")
OBJ_DIR = os.path.join(PKG_DIR, "build")

SOURCES = ["lib.cu", "route.cu", "gate_mma.cu", "gate_route_replay.cu", "permute.cu", "group_gemm.cu", "comm.cu", "ep.cu", "norm.cu", "fp8.cu", "lm_head_ce.cu",
           "qk_norm_rope.cu", "moe_aux_loss.cu"]

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = [
    *ARCH_FLAGS,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode())  # location-independent: a copied tree keeps its build
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def sources() -> list[str]:
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = sources()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(PKG_DIR), "include", "xtuner_b200.h"))
    stamp = os.path.join(LIB_DIR, ".build_digest")
    digest = _digest(srcs + headers)
    if not force and os.path.exists(LIB_PATH) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: str) -> tuple[str, str]:
        obj = os.path.join(OBJ_DIR, os.path.basename(src).replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr

    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(compile_one, srcs))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            sys.stderr.write(log)
    with open(os.path.join(OBJ_DIR, "ptxas.log"), "w") as f:
        for _, log in results:
            f.write(log)
    # link to a temporary name and rename: a tree snapshot taken mid-build never sees a half-written library
    tmp_lib = LIB_PATH + f".tmp{os.getpid()}"
    link = [nvcc, "-shared", "-o", tmp_lib, *objs, *ARCH_FLAGS, "-cudart", "static"]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if os.path.exists(stamp):
        os.remove(stamp)
    os.replace(tmp_lib, LIB_PATH)
    with open(stamp + ".tmp", "w") as f:
        f.write(digest)
    os.replace(stamp + ".tmp", stamp)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
