"""Native sm_90a ops for d9d_b200 (hand-written CUDA: wgmma GEMMs fed by TMA, fused elementwise kernels).

``ops.load()`` loads (building first if necessary) the in-tree extension and returns ``torch.ops.d9d_b200``.
On a machine with a GPU the ops are mandatory: callers must not silently fall back to PyTorch.
"""

from __future__ import annotations

import threading

import torch

from . import build as _build

_lock = threading.Lock()
_loaded = False


def is_available() -> bool:
    """True when the native kernels can run (CUDA device present)."""
    return torch.cuda.is_available()


def load():
    """Load the native extension (build on first use). Returns the ``torch.ops.d9d_b200`` namespace."""
    global _loaded
    if _loaded:
        return torch.ops.d9d_b200
    with _lock:
        if not _loaded:
            path = _build.LIB_PATH if _build.is_up_to_date() else _build.build(verbose=True)
            torch.ops.load_library(str(path))
            _loaded = True
    return torch.ops.d9d_b200


def lib_path() -> str:
    return str(_build.LIB_PATH)


__all__ = ["is_available", "lib_path", "load"]
