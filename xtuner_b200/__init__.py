"""xtuner_b200 — H100-native (sm_90a) drop-in for XTuner V1's data-parallel MoE training hot path.

Host code is thin Python over a C-ABI CUDA library (``include/xtuner_b200.h``).  Importing this package
does not need a GPU; calling any compute op does (there is no CPU fallback)."""
from . import _capi  # noqa: F401

__version__ = "0.1.0"


def lib_path() -> str:
    return _capi.LIB_PATH
