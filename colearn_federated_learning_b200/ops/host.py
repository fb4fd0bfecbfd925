"""Native CPU executor of the MLP local fit (``csrc/mlp_host.cpp``) — the worker path of devices without a GPU.

The reference's workers are CPU devices (Raspberry Pi 3B+, 163.7 batch-1 SGD steps/s through PySyft, BASELINE.md);
here a CPU worker — ``remote_worker.py`` on an edge device, the coordinator's VirtualWorker mode on a CPU-only box
(BASELINE config 1), the gloo engine — runs the whole fit as one C++ loop on the flat arena, K clients on K threads.
``ops/reference.py`` stays the definition the executor is tested against and the fallback when the extension has not
been built (``colearn-build-kernels --host``; ``COLEARN_HOST_KERNELS=0`` forces the PyTorch definitions).
"""
from __future__ import annotations

import glob
import importlib.util
import os
import threading
from typing import List, Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_lock = threading.Lock()
_state = {"mod": None, "tried": False, "err": None}
LOSS_CODES = {"bce": 0, "sse": 1, "xent": 2, "mse": 3}


def enabled() -> bool:
    return os.environ.get("COLEARN_HOST_KERNELS", "1") != "0"


def load(build_if_missing: bool = False):
    """The compiled module, or ``None`` (not built / failed to import; the reason is kept in :func:`last_error`)."""
    with _lock:
        if _state["mod"] is not None:
            return _state["mod"]
        if _state["tried"] and not build_if_missing:
            return None                                   # negative result is cached: available() runs once per fit
        hits = sorted(glob.glob(os.path.join(_HERE, "_colearn_host*.so")))
        if not hits and build_if_missing:
            try:
                from . import build
                hits = [build.build_host()]
            except Exception as e:  # noqa: BLE001 - no compiler on the device: stay on the PyTorch definitions
                _state["err"] = e
        if not hits:
            _state["tried"] = True
            return None
        try:
            spec = importlib.util.spec_from_file_location("_colearn_host", hits[0])
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)  # type: ignore[union-attr]
            _state["mod"] = mod
        except Exception as e:  # noqa: BLE001 - ImportError / OSError (ABI mismatch, missing libtorch)
            _state["err"] = e
        _state["tried"] = True
        return _state["mod"]


def last_error() -> Optional[BaseException]:
    return _state["err"]


def available() -> bool:
    return enabled() and load() is not None


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().float()


def mlp_local_sgd_multi(dims: Sequence[int], out_activation: str, thetas: List[torch.Tensor], xs: List[torch.Tensor],
                        ys: List[torch.Tensor], perms: List[Optional[torch.Tensor]], batch_size: int = 1, lr: float = 0.01,
                        epochs: int = 1, max_nr_batches: int = -1, loss: str = "xent", threads: int = 0,
                        class_weights: Optional[Sequence[float]] = None, local_opt=None) -> torch.Tensor:
    """Train K clients concurrently, each in place on its own flat fp32 arena (``thetas[i]`` must be contiguous CPU
    fp32 — a row of a ``[K, P]`` matrix is fine).  Returns ``[K, 2]`` = (last batch loss, mean loss over the steps).
    ``class_weights``: a class-weighted fit (``reference.loss_and_dz``), checked by the caller (``fused_mlp.check_class_weights``).
    ``local_opt``: a ``fl.local_opt.LocalOpt`` other than plain SGD, run by the generic loop (the caller refuses it together
    with class weights)."""
    mod = load()
    if mod is None:
        raise RuntimeError(f"_colearn_host is not built (colearn-build-kernels --host): {last_error()}")
    for t in thetas:
        if t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise ValueError("thetas must be contiguous CPU fp32 tensors (they are updated in place)")
    xs2 = [_f32(x.view(x.shape[0], -1)) for x in xs]
    ys2 = [_f32(y).view(y.shape[0], -1) for y in ys]
    perms2 = [None if p is None else p.detach().to(torch.int32).contiguous().view(-1, x.shape[0]) for p, x in zip(perms, xs2)]
    args = ([int(d) for d in dims], out_activation == "sigmoid", list(thetas), xs2, ys2, perms2, int(batch_size), int(epochs),
            int(max_nr_batches if max_nr_batches is not None else -1), LOSS_CODES[loss], float(lr), int(threads))
    if local_opt is not None and not local_opt.is_plain():
        if class_weights is not None:
            raise ValueError("class weights together with a local optimizer are not supported")
        return mod.mlp_local_sgd_opt(*args, local_opt.launch_args())
    if class_weights is None:
        return mod.mlp_local_sgd(*args)
    return mod.mlp_local_sgd_cw(*args, [float(w) for w in class_weights])


def mlp_forward(flat: torch.Tensor, dims: Sequence[int], x: torch.Tensor, out_activation: str = "none") -> torch.Tensor:
    mod = load()
    if mod is None:
        raise RuntimeError(f"_colearn_host is not built: {last_error()}")
    return mod.mlp_forward([int(d) for d in dims], out_activation == "sigmoid", _f32(flat), _f32(x.view(x.shape[0], -1)))
