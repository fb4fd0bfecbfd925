"""Datasets and transforms.

Parity: ``NetworkTrafficDataset`` (reference ``datasets.py:17-58``) reads a Bot-IoT "10-best"
CSV, keeps ``attack`` (label) + the 10 model features in the reference's column order
(``datasets.py:29``), MinMax-scales the features over the *local* file (``:31-32``) and yields
``(float32[10], float32[1])``.  Transforms ``ToTensor`` / ``Normalize`` / ``ToTensorLong``
mirror ``datasets.py:60-89``.

GPU-first difference: in addition to the per-sample ``__getitem__`` protocol the dataset
exposes :meth:`tensors` — the whole shard as two dense tensors — because the training kernels
consume a device-resident ``[N, F]`` matrix and a permutation, never a Python-level DataLoader.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import numpy as np
import torch
from torch.utils.data import Dataset

FEATURE_COLUMNS = ["seq", "stddev", "N_IN_Conn_P_SrcIP", "min", "state_number", "mean",
                   "N_IN_Conn_P_DstIP", "drate", "srate", "max"]
LABEL_COLUMN = "attack"
CATEGORY_COLUMN = "category"
# The attack categories of Bot-IoT, in class-index order.  Index 0 is Normal, so "any attack" is class != 0.
CATEGORIES = ("Normal", "DDoS", "DoS", "Reconnaissance", "Theft")
CSV_HEADER = ["pkSeqID", "proto", "saddr", "sport", "daddr", "dport", "seq", "stddev",
              "N_IN_Conn_P_SrcIP", "min", "state_number", "mean", "N_IN_Conn_P_DstIP", "drate",
              "srate", "max", "attack", "category", "subcategory"]

_device = torch.device("cuda" if torch.cuda.is_available() else "cpu")


def minmax_scale(x: np.ndarray) -> np.ndarray:
    """Column-wise scale to [0, 1]; constant columns map to 0 (sklearn ``MinMaxScaler``
    semantics, which the reference uses at ``datasets.py:31-32``)."""
    x = np.asarray(x, dtype=np.float64)
    lo = x.min(axis=0)
    rng = x.max(axis=0) - lo
    rng[rng == 0] = 1.0
    return (x - lo) / rng


class ToTensor:
    """ndarray → float32 tensor on the default device (reference ``datasets.py:60-69``)."""

    def __init__(self, device: Optional[torch.device] = None) -> None:
        self.device = device

    def __call__(self, sample: np.ndarray) -> torch.Tensor:
        x = torch.from_numpy(np.asarray(sample))
        return x.to(self.device or _device).float()


class ToTensorLong:
    """ndarray → int64 tensor (reference ``datasets.py:82-89``)."""

    def __init__(self, device: Optional[torch.device] = None) -> None:
        self.device = device

    def __call__(self, sample: np.ndarray) -> torch.Tensor:
        return torch.from_numpy(np.asarray(sample)).long().to(self.device or _device)


class Normalize:
    """``(x - (max+min)/2) / ((max+min)/2)`` over the whole tensor (reference ``datasets.py:71-80``)."""

    def __call__(self, sample: torch.Tensor) -> torch.Tensor:
        x_max, x_min = torch.max(sample), torch.min(sample)
        mid = (x_max + x_min) / 2
        return (sample - mid) / mid


class NetworkTrafficDataset(Dataset):
    def __init__(self, csv_file: str, transform: Optional[Callable] = None) -> None:
        import pandas as pd

        df = pd.read_csv(csv_file)
        self.df = df[[LABEL_COLUMN] + FEATURE_COLUMNS]
        self.data = minmax_scale(self.df.values[:, 1:])
        self.targets = self.df.iloc[:, 0]
        self.transform = transform
        # class index (CATEGORIES) of every row, None for a CSV without the column
        self.categories = _category_codes(df, csv_file) if CATEGORY_COLUMN in df.columns else None

    def __len__(self) -> int:
        return len(self.df)

    def __getitem__(self, idx):
        if torch.is_tensor(idx):
            idx = idx.tolist()
        data = np.array(self.data[idx])
        tgt = np.asarray(self.targets)
        label = tgt[idx].reshape(-1, 1) if isinstance(idx, list) else np.array([tgt[idx]])
        if self.transform:
            data, label = self.transform(data), self.transform(label)
        return data, label

    def tensors(self, device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        x = torch.from_numpy(np.ascontiguousarray(self.data)).float()
        y = torch.from_numpy(np.asarray(self.targets, dtype=np.float32)).view(-1, 1)
        if device is not None:
            x, y = x.to(device), y.to(device)
        return x, y


def _category_codes(df, csv_file: str) -> np.ndarray:
    """int64 [N] class indices of the ``category`` column.  ValueError naming the CSV line (header = line 1) and the value
    for a category outside CATEGORIES, or for a row whose ``attack`` disagrees with it (attack == 0 exactly when Normal)."""
    index = {name: i for i, name in enumerate(CATEGORIES)}
    names = df[CATEGORY_COLUMN].astype(str).str.strip()
    codes = names.map(index)
    bad = codes.isna().to_numpy()
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError(f"{csv_file}:{i + 2}: category {df[CATEGORY_COLUMN].iloc[i]!r} is not one of {', '.join(CATEGORIES)}")
    codes = codes.to_numpy(dtype=np.int64)
    attack = df[LABEL_COLUMN].to_numpy()
    bad = (attack == 0) != (codes == 0)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise ValueError(f"{csv_file}:{i + 2}: attack {attack[i].item()!r} disagrees with category {names.iloc[i]!r} "
                         "(attack is 0 exactly for Normal rows)")
    return codes


def category_tensors(ds, device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(X[N, F], class index[N, 1] float)`` of a dataset that carries attack categories (``ds.categories``).  ValueError for
    one that does not (a CSV without the column, a plugin dataset, the XOR toy)."""
    codes = getattr(ds, "categories", None)
    if codes is None:
        raise ValueError(f"the {type(ds).__name__} has no attack categories (a '{CATEGORY_COLUMN}' column)")
    x = dataset_tensors(ds, device)[0]
    y = torch.from_numpy(np.array(codes, dtype=np.float32)).view(-1, 1).to(x.device)
    return x, y


class BaseDataset(Dataset):
    """In-memory ``(data, targets)`` dataset (the PySyft ``sy.BaseDataset`` used at rw.py:80)."""

    def __init__(self, data: torch.Tensor, targets: torch.Tensor) -> None:
        assert len(data) == len(targets)
        self.data, self.targets = data, targets

    def __len__(self) -> int:
        return len(self.data)

    def __getitem__(self, idx):
        return self.data[idx], self.targets[idx]

    def tensors(self, device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        x, y = self.data.detach().float(), self.targets.detach().float()
        if y.dim() == 1:
            y = y.view(-1, 1)
        if device is not None:
            x, y = x.to(device), y.to(device)
        return x, y


def category_dataset(x: torch.Tensor, codes: torch.Tensor) -> BaseDataset:
    """Rows whose attack categories are known (class indices into CATEGORIES, e.g. ``synthetic_category``'s labels) as a
    dataset shaped like the CSV adapter's: the binary ``attack`` label (category != Normal) as targets, the class indices as
    ``categories``"""
    codes = codes.reshape(-1).long()
    ds = BaseDataset(x, (codes != 0).float().view(-1, 1))
    ds.categories = codes.cpu().numpy()
    return ds


def xor_toy_dataset() -> BaseDataset:
    """The worker's default toy data when ``--training`` is omitted (reference rw.py:75-80)."""
    data = torch.tensor([[0.0, 1.0], [1.0, 0.0], [1.0, 1.0], [0.0, 0.0]])
    target = torch.tensor([[1.0], [1.0], [0.0], [0.0]])
    return BaseDataset(data, target)


def dataset_tensors(ds, device: Optional[torch.device] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Dense ``(X[N,F], y[N,1])`` view of any supported dataset."""
    if hasattr(ds, "tensors") and callable(ds.tensors):
        return ds.tensors(device)
    xs, ys = zip(*[ds[i] for i in range(len(ds))])
    x = torch.stack([torch.as_tensor(v).float().reshape(-1) for v in xs])
    y = torch.stack([torch.as_tensor(v).float().reshape(-1) for v in ys])
    if device is not None:
        x, y = x.to(device), y.to(device)
    return x, y


# ------------------------------------------------------------------------------------------------------------------
# dataset registry: what ``--dataset NAME`` resolves to on both CLIs (the reference tells its users to write their own
# ``datasets.py`` and edit ``remote_worker.py`` / ``starting_training_local``, README.md:119-169)
# ------------------------------------------------------------------------------------------------------------------
DATASET_REGISTRY = {"unsw": NetworkTrafficDataset}


def register_dataset(name: str, factory, overwrite: bool = False) -> None:
    """``factory(path) -> dataset`` with ``.data`` / ``.targets`` (array-likes or tensors, one row per sample), e.g. a
    :class:`BaseDataset`.  Selected with ``--dataset NAME`` together with ``-dt/--training`` (worker) or ``--test-path``
    (coordinator, local / encrypted mode and evaluation)."""
    if not name or not isinstance(name, str):
        raise ValueError("dataset name must be a non-empty string")
    if name in DATASET_REGISTRY and not overwrite:
        raise ValueError(f"dataset {name!r} is already registered (pass overwrite=True to replace it)")
    if not callable(factory):
        raise TypeError("factory must be callable")
    DATASET_REGISTRY[name] = factory


def load_dataset(name: str, path: str):
    try:
        factory = DATASET_REGISTRY[name]
    except KeyError:
        raise ValueError(f"unknown dataset {name!r}; choose from {sorted(DATASET_REGISTRY)} or register one (--plugin)") from None
    return factory(path)
