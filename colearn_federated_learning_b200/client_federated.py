"""Reference-shaped API surface (``client_federated.py`` of CoLearn) on top of the GPU engine.

Keeps the names a CoLearn user knows — ``Net``, ``TestingRemote``, ``FFNN``, ``loss_fn``,
``train_local``, ``encrypted_training``, ``train_remote``, ``evaluate``,
``get_private_data_loaders`` — with the reference's signatures where they make sense without
PySyft objects.  Each docstring cites the reference lines it mirrors.
"""
from __future__ import annotations

import asyncio
from typing import Any, Optional, Tuple

import torch
import torch.nn.functional as F

from .control.workers import RemoteWorkerClient
from .data import FederatedDataLoader
from .fl.encrypted import encrypted_training as _encrypted_training
from .fl.encrypted import get_private_data_loaders as _get_private_data_loaders
from .fl.evaluate import evaluate as _evaluate
from .fl.trainer import FitConfig, local_fit
from .models import FFNN, Net, TestingRemote, flatten_params, unflatten_params  # noqa: F401
from .smpc import CryptoProvider


def loss_fn(target: torch.Tensor, pred: torch.Tensor) -> torch.Tensor:
    """``F.binary_cross_entropy(input=pred, target=target)`` (reference cf.py:76-79).  On the device
    path this is the fused ``ops.sigmoid_bce`` / the BCE branch inside the persistent kernel."""
    return F.binary_cross_entropy(input=pred, target=target)


def train_local(worker: str, model, opt: Optional[Any], epochs: int, federated_train_loader: FederatedDataLoader,
                args) -> Tuple[Any, torch.Tensor]:
    """Fit ``model`` on the batches that live on ``worker`` (reference cf.py:82-127: sum-squared-error
    loss, SGD).  Returns ``(model, last_loss)``.  Unlike the reference the fit runs as one fused
    call on the worker's shard; the caller must pass each worker its *own replica* (true FedAvg)."""
    shard = federated_train_loader.fed[worker]
    lr = opt.param_groups[0]["lr"] if opt is not None else args.lr
    cfg = FitConfig(model=getattr(args, "model", "ffnn"), loss="sse", batch_size=args.batch_size, epochs=epochs,
                    max_nr_batches=getattr(args, "federate_after_n_batches", -1), lr=lr, seed=args.seed)
    dev = shard.x.device
    flat = flatten_params(model).to(dev)
    model.to(dev)
    last, _ = local_fit(flat, model, shard.x, shard.y, cfg)
    unflatten_params(model, flat)
    return model, last


def encrypted_training(args, model, private_train_loader, optimizer=None, epoch: int = 0):
    """One epoch of SMPC training on secret-shared batches (reference cf.py:130-170)."""
    return _encrypted_training(model, private_train_loader, args.lr, epoch, args.log_interval, args.batch_size)


async def train_remote(worker: RemoteWorkerClient, traced_model, batch_size: int, optimizer: str, max_nr_batches: int,
                       epochs: int, lr: float, model_name: str = "ffnn", loss: str = "bce"):
    """Send the model to ``worker``, fit remotely, get it back (reference cf.py:175-213: TrainConfig.send →
    async_fit → model_ptr.get).  Returns ``(worker.id, model, loss)``; one RPC carries all three legs."""
    cfg = FitConfig(model=model_name, loss=loss, batch_size=batch_size, epochs=epochs, max_nr_batches=max_nr_batches,
                    lr=lr, optimizer=optimizer)
    flat = flatten_params(traced_model).cpu()
    loop = asyncio.get_running_loop()
    new_flat, last, _n = await loop.run_in_executor(None, lambda: worker.fit(flat, cfg))
    unflatten_params(traced_model, new_flat)
    return worker.id, traced_model, torch.tensor(last)


def evaluate(model, test_loader, device):
    """Local evaluation of the global model (reference cf.py:217-253): average BCE + accuracy."""
    xs, ys = zip(*[(d, t) for d, t in test_loader])
    x = torch.cat([d.reshape(-1, d.shape[-1]) for d in xs]).to(device)
    y = torch.cat([t.reshape(-1, 1) for t in ys]).to(device)
    print("Local evaluation start...")
    return _evaluate(model.to(device), x, y)


def get_private_data_loaders(workers, args, n_train_items, precision_fractional=3, crypto_provider=None, dataset=None):
    """Secret-shared ``(data, target)`` batches (reference cf.py:257-277)."""
    from .data import NetworkTrafficDataset
    provider = crypto_provider or CryptoProvider(seed=args.seed)
    ds = dataset if dataset is not None else NetworkTrafficDataset(args.test_path)
    return _get_private_data_loaders(ds, provider, n_train_items, args.batch_size, precision_fractional, args.seed)
