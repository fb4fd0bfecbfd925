"""Loader for the in-tree sm_90a extension ``_colearn_C``.

Policy: on a box with a GPU the extension is *mandatory* — :func:`require` raises if it is
missing rather than silently running a PyTorch fallback.  On a CPU-only box :func:`available` is simply False and the
dispatchers in ``ops/__init__`` use ``ops.reference``.
"""
from __future__ import annotations

import glob
import importlib.util
import os
import threading
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
_lock = threading.Lock()
_mod = None
_err: Optional[Exception] = None
_tried = False


def so_path() -> Optional[str]:
    hits = sorted(glob.glob(os.path.join(_HERE, "_colearn_C*.so")))
    return hits[0] if hits else None


def load(build_if_missing: bool = False):
    """Import the extension (optionally building it first).  Returns the module or None."""
    global _mod, _err, _tried
    with _lock:
        if _mod is not None:
            return _mod
        path = so_path()
        if path is None and build_if_missing:
            from . import build
            path = build.build_all()
        if path is None:
            _tried = True
            _err = FileNotFoundError("_colearn_C*.so not built (run `python -m colearn_federated_learning_b200.ops.build`)")
            return None
        try:
            import torch  # noqa: F401  (libtorch must be loaded first)
            spec = importlib.util.spec_from_file_location("_colearn_C", path)
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)  # type: ignore[union-attr]
            _mod = mod
        except Exception as e:  # noqa: BLE001 - ImportError / OSError (missing libtorch symbols, wrong arch, ...)
            _err = e
        _tried = True
        return _mod


def available() -> bool:
    return load() is not None


def require():
    mod = load()
    if mod is None:
        raise RuntimeError(f"colearn sm_90a extension is required on a CUDA device but could not be loaded: {_err!r}")
    return mod
