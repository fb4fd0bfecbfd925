"""Asynchronous buffered aggregation (FedBuff, Nguyen et al., AISTATS 2022; staleness weighting as in FedAsync, Xie et al. 2019).

Remote mode's synchronous rounds last as long as the slowest device.  With ``--async-buffer K`` every device trains whenever it
is free, from whatever global version is current, and the server steps once ``K`` replies are buffered:

* **Versions.**  The global model has a version ``v`` (0 at the start, +1 per server step).  A fit request carries the version
  of the theta it sends, and the coordinator records which version it sent to which device (``base``); a version a device
  echoes is never trusted.
* **Staleness.**  ``tau_k = v - base_k`` when the step is taken; the reply's weight is scaled by ``s(tau) = (1 + tau)^-a``
  (``--staleness-exponent a``, 0.5 = FedBuff's ``1 / sqrt(1 + tau)``).  A reply with ``tau > --max-staleness S`` is dropped.
* **Step.**  ``alpha`` are the usual FedAvg weights of the kept replies (uniform, or ``n_k``-weighted with ``--weighted``,
  normalised to 1) and the step target is ``a = theta + sum_k alpha_k s(tau_k) d_k``, ``d_k`` the device's delta to its own
  base (``x_k - theta_{base_k}`` for fp32 replies, read from the version ring by ``ops.fedavg_apply_based``; the decoded delta
  for int8 / int4 / top-k replies, already taken against the model the device received).  The weights are not renormalised
  over ``s``: stale buffers make shorter steps.  With every ``tau = 0`` this is the synchronous FedAvg target.
* **Aggregators.**  The coordinate-wise median / trimmed mean run over the deltas and stay unweighted, so staleness does not
  enter them; the distance-based kinds take ``alpha_k s(tau_k)`` as their alpha and start from 0.
* **Order.**  The kept replies are sorted by ``(base, device id)`` before the apply: a step depends on which replies made it
  up, not on the order they arrived in.

The fp32 version ring holds ``S + 2`` versions (slot ``version mod (S + 2)``): the ``S + 1`` a step may read as bases
(``v - S .. v``) and the one it writes, so the slot the apply stores the new theta into is never a base of the same step.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .fedavg import normalized_weights

DEFAULT_MAX_STALENESS = 4
DEFAULT_STALENESS_EXPONENT = 0.5


@dataclass(frozen=True)
class AsyncSettings:
    buffer: int                                   # K: replies per server step (>= 1)
    concurrency: int = 0                          # fits in flight; 0 = one per selected device
    max_staleness: int = DEFAULT_MAX_STALENESS    # S: replies older than this many versions are dropped
    exponent: float = DEFAULT_STALENESS_EXPONENT  # a of s(tau) = (1 + tau)^-a

    def __post_init__(self) -> None:
        if self.buffer < 1:
            raise ValueError(f"--async-buffer must be >= 1 to turn asynchronous aggregation on, not {self.buffer}")
        if self.concurrency < 0:
            raise ValueError(f"--async-concurrency must be >= 1 (0 = one fit per device), not {self.concurrency}")
        if self.max_staleness < 0:
            raise ValueError(f"--max-staleness must be >= 0, not {self.max_staleness}")
        if not (np.isfinite(self.exponent) and self.exponent >= 0):
            raise ValueError(f"--staleness-exponent must be finite and >= 0, not {self.exponent}")

    @property
    def ring_slots(self) -> int:
        """versions the fp32 ring keeps: the S + 1 a step may read and the one it writes"""
        return self.max_staleness + 2

    def slot(self, version: int) -> int:
        return version % self.ring_slots


def staleness_weight(tau: int, exponent: float) -> float:
    """``s(tau) = (1 + tau)^-a``"""
    return float((1.0 + tau) ** -exponent)


@dataclass
class Reply:
    """One checked fit reply in the buffer: ``update`` is the fp32 model or the codec's wire fields, ``base`` the version the
    coordinator sent the device."""
    device: str
    base: int
    update: Any
    n: int
    loss: float


@dataclass
class StepPlan:
    kept: List[Reply]          # sorted by (base, device)
    weights: List[float]       # float32 values: alpha_k s(tau_k), in the order of kept
    stale_dropped: List[str]   # devices whose reply was older than S versions
    record: List[list]         # [[device, base, staleness, weight], ...] in the order of kept


def plan_step(buffer: Sequence[Reply], version: int, settings: AsyncSettings, weighted: bool) -> StepPlan:
    """What one server step at global version ``version`` does with the buffered replies: drop the stale ones, sort the rest by
    ``(base, device)`` and weigh each by ``alpha_k s(tau_k)``."""
    stale = [r for r in buffer if version - r.base > settings.max_staleness]
    kept = sorted((r for r in buffer if version - r.base <= settings.max_staleness), key=lambda r: (r.base, r.device))
    if not kept:
        return StepPlan([], [], [r.device for r in stale], [])
    alpha = normalized_weights([r.n for r in kept] if weighted else None, len(kept), dtype=torch.float64).tolist()
    w = [float(np.float32(a * staleness_weight(version - r.base, settings.exponent))) for a, r in zip(alpha, kept)]
    rec = [[r.device, r.base, version - r.base, wk] for r, wk in zip(kept, w)]
    return StepPlan(kept, w, [r.device for r in stale], rec)


def ring_init(theta: torch.Tensor, settings: AsyncSettings) -> torch.Tensor:
    """The fp32 version ring ``[S + 2, P]`` on theta's device, version 0 in its slot"""
    ring = torch.zeros(settings.ring_slots, theta.numel(), dtype=torch.float32, device=theta.device)
    ring[settings.slot(0)].copy_(theta.reshape(-1))
    return ring


def replay(theta0: torch.Tensor, steps: Sequence[Tuple[Sequence[torch.Tensor], Sequence[int], Sequence[float]]], settings: AsyncSettings,
           server_lr: float = 1.0, aggregator=None) -> List[torch.Tensor]:
    """Every fp32 global version ``[theta_0, theta_1, ...]`` of the given steps, each ``(models, bases, weights)`` in the order
    the step applied them, through ``ops.reference.fedavg_apply_based`` on the CPU (an independent replay of a run's records)."""
    from ..ops import reference
    theta = theta0.detach().to("cpu", torch.float32).reshape(-1).clone()
    ring = ring_init(theta, settings)
    versions = [theta.clone()]
    for v, (models, bases, weights) in enumerate(steps):
        if len(models):
            reference.fedavg_apply_based(theta, torch.stack([m.reshape(-1).float().cpu() for m in models]), ring,
                                         [settings.slot(b) for b in bases], torch.tensor(weights, dtype=torch.float32),
                                         settings.slot(v + 1), server_lr, aggregator=aggregator)
        else:
            ring[settings.slot(v + 1)].copy_(theta)
        versions.append(theta.clone())
    return versions


def optional_settings(buffer: int, concurrency: int, max_staleness: int, exponent: float) -> Optional[AsyncSettings]:
    """The settings of the ``--async-*`` flags, None when ``--async-buffer`` is 0 (synchronous rounds)"""
    if buffer == 0:
        if concurrency or max_staleness != DEFAULT_MAX_STALENESS or exponent != DEFAULT_STALENESS_EXPONENT:
            raise ValueError("--async-concurrency / --max-staleness / --staleness-exponent need --async-buffer K > 0")
        return None
    return AsyncSettings(buffer, concurrency, max_staleness, exponent)
