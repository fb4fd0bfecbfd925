"""Fully-connected model family.

Parity (reference ``client_federated.py``): ``FFNN`` 10-50-30-10-1 + sigmoid (``:50-69``, the
production model, 2 401 params), ``TestingRemote`` 2-50-10-1 (``:37-48``, 671 params),
``Net`` 784-128-64-10 (``:22-34``, 109 386 params).  BASELINE.json adds ``MLP`` 10-64-64-2 and
``WideMLP`` 10-4096x4-2 (50 397 186 params).  State-dict keys are ``fc1.weight, fc1.bias, ...``
exactly like the reference so ``test.pth`` files are interchangeable (SURVEY §2.7).

Every model carries an :class:`MLPSpec` describing its layer dims, output activation and
default loss.  The sm_90a kernels (``ops/``) consume the spec + a flat fp32 parameter arena
instead of the ``nn.Module``; the module form exists for CPU execution, checkpoints and as the
numerics oracle in tests.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass(frozen=True)
class MLPSpec:
    dims: Tuple[int, ...]          # (in, h1, ..., out)
    out_activation: str = "none"   # none | sigmoid
    default_loss: str = "xent"     # bce | sse | xent | mse
    flatten_input: bool = False
    target: str = "label"          # label: trained on the dataset's labels; input: trained to reconstruct its input (fl/anomaly.py);
                                   # category: trained on the attack category of every row (data.CATEGORIES, fl/category.py)

    @property
    def n_layers(self) -> int:
        return len(self.dims) - 1

    @property
    def n_params(self) -> int:
        return sum(self.dims[i] * self.dims[i + 1] + self.dims[i + 1] for i in range(self.n_layers))

    def offsets(self) -> List[Tuple[int, int]]:
        """(weight_offset, bias_offset) of each layer inside the flat arena (state-dict order:
        fc1.weight, fc1.bias, fc2.weight, ...; weights row-major ``[out, in]``)."""
        out, off = [], 0
        for i in range(self.n_layers):
            w = off
            off += self.dims[i] * self.dims[i + 1]
            b = off
            off += self.dims[i + 1]
            out.append((w, b))
        return out


class MLPNet(nn.Module):
    """ReLU MLP with ``fc{i}`` naming; output activation per spec."""

    spec: MLPSpec

    def __init__(self, spec: MLPSpec) -> None:
        super().__init__()
        self.spec = spec
        for i in range(spec.n_layers):
            setattr(self, f"fc{i + 1}", nn.Linear(spec.dims[i], spec.dims[i + 1]))

    def layers(self) -> List[nn.Linear]:
        return [getattr(self, f"fc{i + 1}") for i in range(self.spec.n_layers)]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.spec.flatten_input:
            x = x.view(-1, self.spec.dims[0])
        ls = self.layers()
        for layer in ls[:-1]:
            x = F.relu(layer(x))
        x = ls[-1](x)
        if self.spec.out_activation == "sigmoid":
            x = torch.sigmoid(x)
        return x

    def get_traced_model(self):
        """Reference API (``client_federated.py:68-69``).  The engine never ships TorchScript —
        the flat arena is the wire format — but the traced module is still offered."""
        return torch.jit.trace(self, torch.zeros(self.spec.dims[0]))


FFNN_SPEC = MLPSpec((10, 50, 30, 10, 1), "sigmoid", "bce")
TESTING_REMOTE_SPEC = MLPSpec((2, 50, 10, 1), "none", "sse")
NET_SPEC = MLPSpec((784, 128, 64, 10), "none", "xent", flatten_input=True)
MLP_SPEC = MLPSpec((10, 64, 64, 2), "none", "xent")
WIDE_MLP_SPEC = MLPSpec((10, 4096, 4096, 4096, 4096, 2), "none", "xent")
AE_SPEC = MLPSpec((10, 32, 4, 32, 10), "none", "mse", target="input")
FFNN_CAT_SPEC = MLPSpec((10, 50, 30, 10, 5), "none", "xent", target="category")


class FFNN(MLPNet):
    """Simple binary feed-forward network (reference ``client_federated.py:50-69``)."""

    spec = FFNN_SPEC                # on the class too: the CLI tells whether it has class-weighted kernels without building it

    def __init__(self) -> None:
        super().__init__(FFNN_SPEC)


class TestingRemote(MLPNet):
    """XOR-toy / inference model (reference ``client_federated.py:37-48``)."""

    __test__ = False  # not a pytest class

    def __init__(self) -> None:
        super().__init__(TESTING_REMOTE_SPEC)


class Net(MLPNet):
    """MNIST MLP (reference ``client_federated.py:22-34``; unused there, kept for parity)."""

    def __init__(self) -> None:
        super().__init__(NET_SPEC)


class MLP(MLPNet):
    """BASELINE configs 2/3: 10-64-64-2 on UNSW-IoT features, softmax cross-entropy."""

    def __init__(self) -> None:
        super().__init__(MLP_SPEC)


class Autoencoder(MLPNet):
    """Anomaly detector: 10-32-4-32-10 trained on benign rows to reconstruct its input (974 params); a row whose
    reconstruction error passes the federated alarm threshold is an alarm (fl/anomaly.py)."""

    spec = AE_SPEC                  # on the class too: the CLI tells an autoencoder from its registry entry without building it

    def __init__(self) -> None:
        super().__init__(AE_SPEC)


class FFNNCategory(MLPNet):
    """Attack classifier: the FFNN's 10-50-30-10 body with a 5-way head (2 445 params), trained with softmax cross-entropy on
    the ``category`` column (Normal, DDoS, DoS, Reconnaissance, Theft; data.CATEGORIES)."""

    spec = FFNN_CAT_SPEC            # on the class too: the CLI tells a category model from its registry entry without building it

    def __init__(self) -> None:
        super().__init__(FFNN_CAT_SPEC)


class WideMLP(MLPNet):
    """BASELINE config 5: 10-4096x4-2 (bandwidth sweep model, 201.6 MB fp32)."""

    def __init__(self, width: int = 4096, depth: int = 4) -> None:
        super().__init__(MLPSpec((10,) + (width,) * depth + (2,), "none", "xent"))
