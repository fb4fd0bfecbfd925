"""Server optimizers of the FedOpt family on top of the FedAvg average.

Plain FedAvg with a server learning rate is ``theta += lr * (a - theta)`` with ``a = sum_k w_k theta_k``.  Treating
``d = a - theta`` as a pseudo-gradient gives server momentum (FedAvgM, Hsu et al. 2019) and the adaptive server optimizers
of Reddi et al., *Adaptive Federated Optimization* (ICLR 2021), Alg. 2:

=========  ==========================================================  ================================
kind       state update                                                 model update
=========  ==========================================================  ================================
sgd        --                                                           theta += lr d   (plain FedAvg)
avgm       m = b1 m + d                                                 theta += lr m
adagrad    m = b1 m + (1 - b1) d ;  v = v + d^2                         theta += lr m / (sqrt(v) + tau)
adam       m = b1 m + (1 - b1) d ;  v = b2 v + (1 - b2) d^2             same
yogi       m = b1 m + (1 - b1) d ;  v = v - (1 - b2) d^2 sign(v - d^2)  same
=========  ==========================================================  ================================

``m`` starts at 0 and ``v`` at ``tau^2``; there is no bias correction.  A round in which no client model arrived leaves
``theta``, ``m`` and ``v`` as they are.  The step runs fused into the FedAvg kernels (``ops/csrc/server_opt.cuh``);
``ops.reference.server_opt_step`` is its PyTorch definition.

The moments live in memory only: a checkpoint holds the model, and a restart begins with ``m = 0``, ``v = tau^2``.
"""
from __future__ import annotations

import logging
import math
from dataclasses import dataclass
from typing import List, Optional

import torch

log = logging.getLogger(__name__)

KINDS = {"sgd": 0, "avgm": 1, "adagrad": 2, "adam": 3, "yogi": 4}   # codes of ServerOptKind (server_opt.cuh)
ADAPTIVE = ("adagrad", "adam", "yogi")


def default_server_lr(kind: str) -> float:
    """1.0 for ``sgd`` / ``avgm`` (plain FedAvg step), 0.01 for the adaptive kinds (their step is ~lr per element)."""
    return 0.01 if kind in ADAPTIVE else 1.0


@dataclass
class ServerOpt:
    """Server optimizer settings.  ``lr=None`` takes :func:`default_server_lr` of the kind."""
    kind: str = "sgd"
    lr: Optional[float] = None
    beta1: float = 0.9
    beta2: float = 0.99
    tau: float = 1e-3

    def __post_init__(self) -> None:
        if self.kind not in KINDS:
            raise ValueError(f"unknown server optimizer {self.kind!r}; expected one of {', '.join(KINDS)}")
        if self.lr is None:
            self.lr = default_server_lr(self.kind)
        self.lr = float(self.lr)
        for name in ("beta1", "beta2"):
            b = float(getattr(self, name))
            if not 0.0 <= b < 1.0:
                raise ValueError(f"server optimizer {name} must lie in [0, 1), got {b}")
            setattr(self, name, b)
        self.tau = float(self.tau)
        if not (self.tau > 0.0 and math.isfinite(self.tau)):
            raise ValueError(f"server optimizer tau must be > 0, got {self.tau}")
        if not math.isfinite(self.lr):
            raise ValueError(f"server learning rate must be finite, got {self.lr}")

    @property
    def code(self) -> int:
        return KINDS[self.kind]

    @property
    def has_v(self) -> bool:
        return self.kind in ADAPTIVE

    @property
    def hyper(self) -> List[float]:
        """``[beta1, beta2, tau]`` in the order the kernel bindings take them."""
        return [self.beta1, self.beta2, self.tau]

    def init_state(self, n: int, device=None) -> "ServerOptState":
        """Fresh moments for ``n`` parameters: ``m = 0`` (every kind but sgd), ``v = tau^2`` (adaptive kinds)."""
        m = torch.zeros(n, dtype=torch.float32, device=device) if self.kind != "sgd" else None
        v = torch.full((n,), self.tau * self.tau, dtype=torch.float32, device=device) if self.has_v else None
        return ServerOptState(self, m, v)


@dataclass
class ServerOptState:
    """A :class:`ServerOpt` together with its moment buffers (``None`` where the kind has none); what
    ``ops.fedavg_apply(..., opt=state)`` takes and updates in place."""
    opt: ServerOpt
    m: Optional[torch.Tensor]
    v: Optional[torch.Tensor]

    @property
    def kind(self) -> str:
        return self.opt.kind

    @property
    def code(self) -> int:
        return self.opt.code

    @property
    def lr(self) -> float:
        return self.opt.lr

    @property
    def hyper(self) -> List[float]:
        return self.opt.hyper

    @property
    def numel(self) -> int:
        return int(self.m.numel()) if self.m is not None else 0


def resolve_server_opt(server_opt: Optional[ServerOpt], server_lr: float) -> ServerOpt:
    """The optimizer an engine / coordinator runs: ``server_opt`` itself, or plain FedAvg with ``server_lr``.  A
    ``ServerOpt`` carries its own learning rate, so passing ``server_lr != 1`` next to it is refused instead of guessed."""
    if server_opt is None:
        return ServerOpt("sgd", lr=server_lr)
    if float(server_lr) != 1.0:
        raise ValueError(f"server_lr={server_lr} given next to server_opt={server_opt.kind!r}, which carries its own lr "
                         f"({server_opt.lr}); set ServerOpt(lr=...) only")
    return server_opt


def server_opt_state(state: Optional[ServerOptState], opt: ServerOpt, theta: torch.Tensor) -> ServerOptState:
    """The state ``opt`` steps ``theta`` with from one round to the next: ``state`` when it belongs to ``opt`` and to a model
    of theta's size, its moments moved to theta's device; otherwise fresh moments (a changed model size is logged)."""
    if state is None or state.opt != opt or state.numel != theta.numel():
        if state is not None and state.numel != theta.numel():
            log.info("Server optimizer state reset: the model has %d parameters, the state %d", theta.numel(), state.numel)
        return opt.init_state(theta.numel(), theta.device)
    if state.m.device != theta.device:
        state.m = state.m.to(theta.device)
        state.v = state.v.to(theta.device) if state.v is not None else None
    return state
