"""Synthetic UNSW-2018 IoT-Botnet-shaped data (there is no network for the real dataset).

``BASELINE.json``: "synthetic UNSW-IoT-shaped data / random-init weights".  The generator
produces the 10 model features already MinMax-scaled to [0, 1] with a binary ``attack`` label
that is a noisy function of a few features (so that loss-decrease tests are meaningful), and can
also write a CSV with the exact Bot-IoT "10-best" 19-column header so the whole CSV → dataset →
training path is exercised (reference example file: ``dataset_example/*.csv``).
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from .datasets import CATEGORIES, CSV_HEADER, FEATURE_COLUMNS


def synthetic_unsw(n: int, seed: int = 0, n_features: int = 10, noise: float = 0.05,
                   device: Optional[torch.device] = None,
                   label_dtype: torch.dtype = torch.float32) -> Tuple[torch.Tensor, torch.Tensor]:
    """Returns ``(X[n, n_features] in [0,1], y[n,1] in {0,1})``; deterministic in ``seed``."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, n_features, generator=g)
    w = torch.linspace(-1.5, 1.5, n_features)
    logit = (x - 0.5) @ w * 4.0 + noise * torch.randn(n, generator=g)
    y = (logit > 0).to(label_dtype).view(n, 1)
    if device is not None:
        x, y = x.to(device), y.to(device)
    return x, y


def synthetic_anomaly(n: int, seed: int = 0, attack_fraction: float = 0.1,
                      device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Traffic for the anomaly detector (``--model autoencoder``): ``(X[n, 10] in [0, 1], y[n, 1])``, deterministic in
    ``seed``.  A benign row (y = 0) lies near a 3-dimensional manifold: the sigmoid of a standard-normal latent through a
    fixed 10 x 3 map (the same for every seed), plus N(0, 0.01^2) noise.  An attack row (y = 1, each row with probability
    ``attack_fraction``) is uniform in [0, 1]^10, off the manifold almost surely."""
    if not 0.0 <= attack_fraction <= 1.0:
        raise ValueError(f"attack_fraction must be in [0, 1], not {attack_fraction}")
    fixed = torch.Generator().manual_seed(20190718)
    w = torch.randn(10, 3, generator=fixed) * 1.5
    b = torch.randn(10, generator=fixed) * 0.5
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(n, 3, generator=g)
    benign = (torch.sigmoid(z @ w.t() + b) + 0.01 * torch.randn(n, 10, generator=g)).clamp(0.0, 1.0)
    attack = torch.rand(n, 10, generator=g)
    y = (torch.rand(n, generator=g) < attack_fraction).view(n, 1)
    x = torch.where(y, attack, benign)
    y = y.float()
    if device is not None:
        x, y = x.to(device), y.to(device)
    return x, y


def synthetic_category(n: int, seed: int = 0, device: Optional[torch.device] = None,
                       probs: Optional[Sequence[float]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Traffic for the attack classifier (``--model ffnn_category``): ``(X[n, 10] in [0, 1], y[n, 1])`` with ``y`` the class
    index into CATEGORIES, deterministic in ``seed``.  Each class is a Gaussian blob (sd 0.08) around its own fixed centre in
    [0.2, 0.8]^10 (the same for every seed), clipped to [0, 1]; the classes are drawn with probabilities ``probs`` (one per
    class, in CATEGORIES order), by default 40 / 20 / 20 / 10 / 10 %, so Normal is the majority class at 40 %."""
    fixed = torch.Generator().manual_seed(20181105)
    centres = 0.2 + 0.6 * torch.rand(len(CATEGORIES), 10, generator=fixed)
    g = torch.Generator().manual_seed(seed)
    probs = torch.tensor([0.4, 0.2, 0.2, 0.1, 0.1] if probs is None else [float(p) for p in probs])
    y = torch.multinomial(probs, n, replacement=True, generator=g) if n > 0 else torch.zeros(0, dtype=torch.long)
    x = (centres[y] + 0.08 * torch.randn(n, 10, generator=g)).clamp(0.0, 1.0)
    y = y.float().view(n, 1)
    if device is not None:
        x, y = x.to(device), y.to(device)
    return x, y


def synthetic_images(n: int, seed: int = 0, size: int = 32, classes: int = 10,
                     device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Synthetic ``[n,3,size,size]`` images with class-dependent mean (BASELINE config 4)."""
    g = torch.Generator().manual_seed(seed)
    y = torch.randint(0, classes, (n,), generator=g)
    x = torch.randn(n, 3, size, size, generator=g) * 0.5
    x += (y.float().view(n, 1, 1, 1) / classes - 0.5)
    if device is not None:
        x, y = x.to(device), y.to(device)
    return x, y


def synthetic_for_model(model: str, n: int, seed: int = 0,
                        device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Synthetic data of the shape ``model`` consumes (``--synthetic N`` on the CLIs): 32x32 images with 10 classes
    for ``resnet18``, 28x28 single-channel digits-shaped inputs for ``net`` (784-128-64-10), two XOR-like features
    for ``testing_remote``, benign rows on a manifold with 10 % attacks off it for ``autoencoder``, five attack categories for
    ``ffnn_category``, the ten UNSW-IoT features otherwise.  Labels are ``[n, 1]`` floats (class index for the
    cross-entropy models), which is what every fit executor accepts."""
    if model == "resnet18":
        x, y = synthetic_images(n, seed=seed)
        y = y.float().view(n, 1)
    elif model == "net":
        x, y = synthetic_images(n, seed=seed, size=28)
        x, y = x[:, :1].contiguous(), y.float().view(n, 1)
    elif model == "testing_remote":
        x, y = synthetic_unsw(n, seed=seed, n_features=2)
    elif model == "autoencoder":
        x, y = synthetic_anomaly(n, seed=seed)
    elif model == "ffnn_category":
        x, y = synthetic_category(n, seed=seed)
    else:
        x, y = synthetic_unsw(n, seed=seed)
    if device is not None:
        x, y = x.to(device), y.to(device)
    return x, y


def write_synthetic_csv(path: str, n: int, seed: int = 0, attack_fraction: Optional[float] = None) -> str:
    """Write a Bot-IoT-shaped CSV (19 columns, header identical to the reference example)."""
    import pandas as pd

    rng = np.random.default_rng(seed)
    x, y = synthetic_unsw(n, seed)
    x, y = x.numpy(), y.numpy().reshape(-1).astype(int)
    if attack_fraction is not None:
        y = (rng.random(n) < attack_fraction).astype(int)
    scale = {"seq": 262212, "stddev": 2.5, "N_IN_Conn_P_SrcIP": 100, "min": 5.0, "state_number": 11,
             "mean": 5.0, "N_IN_Conn_P_DstIP": 100, "drate": 60.0, "srate": 1000.0, "max": 5.0}
    df = pd.DataFrame({c: x[:, i] * scale[c] for i, c in enumerate(FEATURE_COLUMNS)})
    for c in ("seq", "N_IN_Conn_P_SrcIP", "state_number", "N_IN_Conn_P_DstIP"):
        df[c] = df[c].round().astype(int)
    df["pkSeqID"] = np.arange(1, n + 1)
    df["proto"] = rng.choice(["tcp", "udp"], n)
    df["saddr"] = [f"192.168.100.{rng.integers(1, 254)}" for _ in range(n)]
    df["sport"] = rng.integers(1024, 65535, n)
    df["daddr"] = [f"192.168.100.{rng.integers(1, 10)}" for _ in range(n)]
    df["dport"] = rng.choice([80, 53, 443, 8080], n)
    df["attack"] = y
    df["category"] = np.where(y == 1, rng.choice(["DDoS", "DoS", "Reconnaissance"], n), "Normal")
    df["subcategory"] = np.where(y == 1, rng.choice(["TCP", "UDP", "HTTP"], n), "Normal")
    df[CSV_HEADER].to_csv(path, index=False, float_format="%.6f")
    return path
