"""Model registry + flat parameter arena (un)flatten.

All model state that FedAvg touches lives in ONE contiguous fp32 vector ("arena") in
state-dict order, so "send model" and "average models" are single contiguous messages
(SURVEY §7.0).  ``named_parameters()`` only — buffers are not averaged (reference
``utils.federated_avg`` semantics, SURVEY §2.3 / C16).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from .mlp import FFNN, MLP, Autoencoder, FFNNCategory, MLPNet, MLPSpec, Net, TestingRemote, WideMLP
from .resnet import ResNet18

MODEL_REGISTRY: Dict[str, Callable[[], nn.Module]] = {
    "ffnn": FFNN,
    "testing_remote": TestingRemote,
    "net": Net,
    "mlp": MLP,
    "wide_mlp": WideMLP,
    "resnet18": ResNet18,
    "autoencoder": Autoencoder,
    "ffnn_category": FFNNCategory,
}

DEFAULT_LOSS = {"ffnn": "bce", "testing_remote": "sse", "net": "xent", "mlp": "xent",
                "wide_mlp": "xent", "resnet18": "xent", "autoencoder": "mse",
                "ffnn_category": "xent"}


def register_model(name: str, factory: Callable[..., nn.Module], default_loss: str = "xent", overwrite: bool = False) -> None:
    """Add a user architecture under ``--model NAME`` (the reference asks its users to edit ``client_federated.py`` and
    ``starting_training_local`` instead, README.md:119-169).  ``factory()`` must return a fresh ``nn.Module``; an
    :class:`~colearn_federated_learning_b200.models.mlp.MLPNet` (any layer sizes) trains through the persistent-kernel /
    layer-wise / native host executors, every other module through the autograd path with this repo's flat SGD and
    loss kernels.  Coordinator and workers must register the same name (models travel as flat parameter vectors, never
    as code): load the registering module on both sides with ``--plugin``."""
    if not name or not isinstance(name, str):
        raise ValueError("model name must be a non-empty string")
    if name in MODEL_REGISTRY and not overwrite:
        raise ValueError(f"model {name!r} is already registered (pass overwrite=True to replace it)")
    if default_loss not in ("bce", "sse", "xent", "mse"):
        raise ValueError(f"unknown loss {default_loss!r}")
    if not callable(factory):
        raise TypeError("factory must be callable")
    MODEL_REGISTRY[name] = factory
    DEFAULT_LOSS[name] = default_loss


def load_plugins(specs) -> List[str]:
    """Import user modules that call :func:`register_model` / ``data.register_dataset`` (``--plugin`` on both CLIs).
    A spec is a dotted module name or a path to a ``.py`` file."""
    import importlib
    import importlib.util
    import os

    loaded = []
    for spec in specs or []:
        if spec.endswith(".py") or os.sep in spec:
            path = os.path.abspath(spec)
            name = "colearn_plugin_" + os.path.splitext(os.path.basename(path))[0]
            sp = importlib.util.spec_from_file_location(name, path)
            if sp is None or sp.loader is None:
                raise ImportError(f"cannot load plugin {spec!r}")
            mod = importlib.util.module_from_spec(sp)
            sp.loader.exec_module(mod)
        else:
            mod = importlib.import_module(spec)
        loaded.append(mod.__name__)
    return loaded


def build_model(name: str, **kwargs) -> nn.Module:
    try:
        return MODEL_REGISTRY[name](**kwargs)
    except KeyError:
        raise ValueError(f"unknown model {name!r}; choose from {sorted(MODEL_REGISTRY)}") from None


def model_spec(model: nn.Module) -> Optional[MLPSpec]:
    return model.spec if isinstance(model, MLPNet) else None


def param_layout(model: nn.Module) -> List[Tuple[str, torch.Size, int, int]]:
    """[(name, shape, offset, numel)] for ``named_parameters()`` in order."""
    out, off = [], 0
    for name, p in model.named_parameters():
        out.append((name, p.shape, off, p.numel()))
        off += p.numel()
    return out


def num_params(model: nn.Module) -> int:
    return sum(p.numel() for p in model.parameters())


@torch.no_grad()
def flatten_params(model: nn.Module, out: Optional[torch.Tensor] = None,
                   dtype: torch.dtype = torch.float32) -> torch.Tensor:
    n = num_params(model)
    if out is None:
        dev = next(model.parameters()).device
        out = torch.empty(n, dtype=dtype, device=dev)
    off = 0
    for p in model.parameters():
        k = p.numel()
        out[off:off + k].copy_(p.detach().reshape(-1))
        off += k
    return out


@torch.no_grad()
def unflatten_params(model: nn.Module, flat: torch.Tensor) -> nn.Module:
    off = 0
    for p in model.parameters():
        k = p.numel()
        p.copy_(flat[off:off + k].view_as(p))
        off += k
    return model


def alias_params_to_arena(model: nn.Module, flat: torch.Tensor) -> nn.Module:
    """Re-point every parameter's storage into ``flat`` (zero-copy).  After this, the kernels
    that update ``flat`` (broadcast, SGD, FedAvg apply) update the module in place — the
    arena-era equivalent of PySyft's in-place ``model.send()/get()`` (SURVEY §2.3)."""
    off = 0
    with torch.no_grad():
        for p in model.parameters():
            k = p.numel()
            view = flat[off:off + k].view(p.shape)
            view.copy_(p.detach())
            p.data = view
            off += k
    return model


def state_dict_from_flat(model: nn.Module, flat: torch.Tensor) -> "OrderedDict[str, torch.Tensor]":
    """CPU fp32 state_dict (params from ``flat``, buffers from the module)."""
    sd = OrderedDict((k, v.detach().cpu().clone()) for k, v in model.state_dict().items())
    off = 0
    for name, p in model.named_parameters():
        k = p.numel()
        sd[name] = flat[off:off + k].detach().float().cpu().view(p.shape).clone()
        off += k
    return sd
