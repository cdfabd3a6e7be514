"""Import shim that lets the *reference* (InternLM/xtuner, /root/reference) be imported in the
authoring container, where six of its python dependencies are absent (SURVEY.md Appendix A).

TEST INFRASTRUCTURE ONLY.  Used by ``make_golden.py`` (golden-vector generation) and by the optional
``-m "not gpu"`` cross-check tests that run only when ``/root/reference`` exists.  Nothing in the
product path (``xtuner_b200``) imports this file, and nothing on the GPU box needs it.

The shim installs permissive stand-ins for: mmengine, cyclopts, addict, more_itertools, codetiming, ray.
It also applies the five CPU monkeypatches listed in SURVEY.md Appendix A so that the reference MoE
path (CUDA-only as written) runs on CPU with its *own in-tree torch fallbacks*.
"""
from __future__ import annotations

import importlib.machinery
import importlib.util
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("XTUNER_REFERENCE_ROOT") or os.path.join(
    os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "oracle", "_ref")  # oracle/make_ref.py


def reference_available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "xtuner", "v1"))


class _Anything:
    """Callable / decorator / attribute sink.  Iteration terminates (see SURVEY Appendix A note)."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        # used as decorator with a single callable/class argument -> identity
        if len(a) == 1 and not k and (callable(a[0]) or isinstance(a[0], type)):
            return a[0]
        return _Anything()

    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        return _Anything()

    def __getitem__(self, item):
        if isinstance(item, int):
            raise IndexError(item)
        return _Anything()

    def __iter__(self):
        return iter(())

    def __bool__(self):
        return False

    def __or__(self, other):
        return other

    def __ror__(self, other):
        return other

    def __mro_entries__(self, bases):
        return (object,)


class _StubModule(types.ModuleType):
    def __init__(self, name):
        super().__init__(name)
        self.__path__ = []  # behave like a package so submodules import
        self.__spec__ = importlib.machinery.ModuleSpec(name, None, is_package=True)

    def __getattr__(self, name):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        full = f"{self.__name__}.{name}"
        if full in sys.modules:
            return sys.modules[full]
        return _Anything()


def _mk(name: str, **attrs) -> _StubModule:
    m = _StubModule(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    parent, _, child = name.rpartition(".")
    if parent and parent in sys.modules:
        setattr(sys.modules[parent], child, m)
    return m


class _StubFinder:
    """Resolves any ``ray.*`` / ``cyclopts.*`` / ``mmengine.*`` submodule import to a stub."""

    PREFIXES = ("ray", "cyclopts", "mmengine")

    def find_spec(self, fullname, path=None, target=None):
        root = fullname.split(".")[0]
        if root in self.PREFIXES and fullname not in sys.modules:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        return _StubModule(spec.name)

    def exec_module(self, module):
        pass


def _digit_version(version_str: str, length: int = 4):
    out = []
    for part in version_str.split("+")[0].split(".")[:length]:
        digits = "".join(ch for ch in part if ch.isdigit())
        out.append(int(digits) if digits else 0)
    while len(out) < length:
        out.append(0)
    return tuple(out)


def _is_installed(name: str) -> bool:
    try:
        return importlib.util.find_spec(name) is not None
    except Exception:
        return False


def install_stubs() -> None:
    if getattr(install_stubs, "_done", False):
        return
    install_stubs._done = True

    def _identity_decorator(fn=None, *a, **k):
        return fn if callable(fn) else (lambda f: f)

    mm = _mk(
        "mmengine",
        is_installed=_is_installed,
        digit_version=_digit_version,
        mkdir_or_exist=lambda d, mode=0o777: os.makedirs(d, mode=mode, exist_ok=True),
        load=lambda *a, **k: {},
        list_dir_or_file=lambda *a, **k: iter(()),
    )
    _mk(
        "mmengine.dist",
        get_rank=lambda *a, **k: 0,
        get_world_size=lambda *a, **k: 1,
        barrier=lambda *a, **k: None,
        master_only=_identity_decorator,
        sync_random_seed=lambda *a, **k: 0,
        init_dist=lambda *a, **k: None,
        dist=_Anything(),
    )
    _mk("mmengine.utils", is_installed=_is_installed)
    _mk("mmengine.fileio", list_dir_or_file=lambda *a, **k: iter(()))
    _mk("mmengine.runner", set_random_seed=lambda *a, **k: None)
    del mm

    class Parameter:  # only ever used as Annotated[...] metadata
        def __init__(self, *a, **k):
            pass

    class Group:
        def __init__(self, *a, **k):
            pass

    class App:
        def __init__(self, *a, **k):
            pass

        def default(self, fn=None, *a, **k):
            return fn if callable(fn) else (lambda f: f)

        command = default

        def __call__(self, *a, **k):
            return None

    _mk("cyclopts", Parameter=Parameter, Group=Group, App=App)
    _mk("cyclopts.group", Group=Group)

    class Dict(dict):
        def __getattr__(self, k):
            try:
                return self[k]
            except KeyError as e:
                raise AttributeError(k) from e

        def __setattr__(self, k, v):
            self[k] = v

    _mk("addict", Dict=Dict)

    def consume(iterator, n=None):
        import collections
        import itertools

        if n is None:
            collections.deque(iterator, maxlen=0)
        else:
            next(itertools.islice(iterator, n, n), None)

    _mk("more_itertools", consume=consume)

    class Timer:
        def __init__(self, *a, **k):
            self.last = 0.0

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def start(self):
            pass

        def stop(self):
            return 0.0

    _mk("codetiming", Timer=Timer)
    _mk("ray")
    sys.meta_path.append(_StubFinder())


def import_reference():
    """Put /root/reference on sys.path (after the stubs) and return the ``xtuner.v1`` package."""
    if not reference_available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    import xtuner.v1  # noqa: F401

    return sys.modules["xtuner.v1"]


def apply_cpu_patches() -> None:
    """The five monkeypatches of SURVEY.md Appendix A (CPU execution of the reference MoE path)."""
    import torch

    import_reference()
    if getattr(apply_cpu_patches, "_done", False):
        return
    apply_cpu_patches._done = True

    _orig_histc = torch.histc

    def _histc(input, bins=100, min=0, max=0, **kw):  # 1. int-safe histc (CUDA semantics on CPU)
        if not input.is_floating_point():
            return _orig_histc(input.float(), bins=bins, min=min, max=max, **kw).to(input.dtype)
        return _orig_histc(input, bins=bins, min=min, max=max, **kw)

    torch.histc = _histc

    class _DummyStream:  # 2. MoE.__init__ creates torch.cuda.Stream()
        def __init__(self, *a, **k):
            pass

        def wait_stream(self, *a, **k):
            pass

    if not torch.cuda.is_available():
        torch.cuda.Stream = _DummyStream

    from xtuner.v1.module.dispatcher import base as _disp_base
    from xtuner.v1.module.grouped_linear import moe_group_linear as _mgl
    from xtuner.v1.ops.moe.cuda.permute_unpermute import (
        cuda_token_permute_torch,
        cuda_token_unpermute_torch,
    )

    _disp_base.permute = cuda_token_permute_torch  # 3.
    _disp_base.unpermute = cuda_token_unpermute_torch  # 4.

    def _group_gemm_loop(x, w, tokens_per_expert):  # 5. == tests/ops/test_grouped_gemm_triton.py:6-23
        outs, start = [], 0
        for i, n in enumerate(tokens_per_expert.tolist()):
            outs.append(torch.matmul(x[start : start + n], w[i].T))
            start += n
        return torch.cat(outs)

    _mgl.group_gemm = _group_gemm_loop
