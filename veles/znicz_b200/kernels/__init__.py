"""sm_90a kernels of znicz_b200 (hand-written CUDA, ahead-of-time compiled, in-tree)."""
from __future__ import annotations

import importlib.util
import os

_ext = None
HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "_znicz_b200_C.so")


def load_extension(required=True):
    """Import the in-tree extension. On a GPU box a missing/unloadable extension is a
    hard error: there is deliberately no eager-PyTorch fallback for the device path."""
    global _ext
    if _ext is not None:
        return _ext
    if not os.path.exists(SO_PATH):
        if required:
            raise RuntimeError(
                "znicz_b200: %s is missing. Build it with "
                "`python -m veles.znicz_b200.kernels.build` (nvcc cross-compiles sm_90a "
                "without a GPU)." % SO_PATH)
        return None
    import torch  # noqa: F401  (libtorch must be loaded first)
    spec = importlib.util.spec_from_file_location("_znicz_b200_C", SO_PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    _ext = mod
    return _ext
