"""Loader for the in-tree sm_90a extension ``distributed_training_guide_b200/_C*.so``.

The extension is built by ``build.py`` (``__graft_entry__.build()``) with
``nvcc -gencode arch=compute_90a,code=sm_90a``.  On a machine with a CUDA device the
ops *require* it (there is no silent PyTorch fallback on the GPU hot path): a missing
or unloadable extension raises at first use.  On CPU-only machines the pure-PyTorch
reference ops in ``ops/reference.py`` are used.

``DTG_FORCE_REFERENCE=attention,gemm`` is a bring-up/debug switch that routes the named
ops through the reference implementation on GPU; it is never set by the chapter
scripts, the tests or ``bench.py``.
"""
from __future__ import annotations

import importlib
import os
import threading

_lock = threading.Lock()
_C = None
_load_error = None


def load(required: bool = False):
    global _C, _load_error
    if _C is not None:
        return _C
    with _lock:
        if _C is None and _load_error is None:
            try:
                import torch  # noqa: F401  (libtorch symbols must be loaded first)

                _C = importlib.import_module("distributed_training_guide_b200._C")
            except Exception as e:  # pragma: no cover - depends on build state
                _load_error = e
    if _C is None and required:
        raise RuntimeError(
            "the sm_90a extension distributed_training_guide_b200/_C.so is not available "
            f"({_load_error!r}); run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `python -m distributed_training_guide_b200.build`) first"
        )
    return _C


def available() -> bool:
    return load(False) is not None


_forced = {s.strip() for s in os.environ.get("DTG_FORCE_REFERENCE", "").split(",") if s.strip()}


def use_cuda_kernel(op: str, *tensors) -> bool:
    """True when ``op`` must run through the sm_90a extension for these tensors."""
    if not tensors or not all(t.is_cuda for t in tensors if t is not None):
        return False
    if op in _forced or "all" in _forced:
        return False
    load(required=True)
    return True


def launch_count() -> int:
    """Number of kernels launched by this extension since process start (bench.py's gpu_launches)."""
    c = load(False)
    return int(c.launch_count()) if c is not None else 0
