"""Byzantine-robust aggregation of the client models: coordinate-wise (Yin et al., *Byzantine-Robust Distributed Learning:
Towards Optimal Statistical Rates*, ICML 2018) and distance-based (the geometric median of RFA, Pillutla et al., IEEE TSP 2022;
the norm-bounded mean of Sun et al., *Can You Really Backdoor Federated Learning?*, 2019).

The FedAvg average ``a = sum_k w_k theta_k`` follows any single client wherever it goes.  The coordinate-wise median and
trimmed mean survive a minority of bad clients: per parameter, the ``n`` contributing values are ordered and ``b`` of them
are dropped at each end before the rest is averaged.

============  =====================================  ==========================================================
kind          values dropped at each end ``b``       result
============  =====================================  ==========================================================
mean          --                                     the weighted FedAvg average (default)
median        ``floor((n - 1) / 2)``                 the middle value (odd n), the mean of the middle two (even n)
trimmed_mean  ``min(floor(beta n), floor((n-1)/2))``  the mean of the values left, ``beta = trim_fraction``
============  =====================================  ==========================================================

The order is the IEEE total order of the float32 values (``-NaN < -Inf < ... < -0 < +0 < ... < +Inf < +NaN``), ties
broken by client slot, so a minority that sends NaN or Inf is trimmed like any other outlier.  ``beta n`` is formed in
float32.  The robust kinds are unweighted: the sample counts ``n_k`` do not enter.  The result is the ``a`` the server step
(``theta += lr (a - theta)``, or a :class:`fl.server_opt.ServerOpt` step) moves towards.  The kernels fuse it into the
FedAvg kernels (``ops/csrc/robust_agg.cuh``); ``ops.reference.robust_aggregate`` is its PyTorch definition.

The distance-based kinds are weighted (``--weighted`` ``n_k`` weights, or uniform) and bound how far one client moves the
model.  Each reweights client ``k`` by its L2 distance ``d_k`` from a centre and takes the weighted mean:

==========  ======================================  ================================================================
kind        centre                                  weight of client k
==========  ======================================  ================================================================
geomed      smoothed Weiszfeld iterate (``iters``)  ``alpha_k / max(eps, d_k)``, normalised
norm_clip   the round's start point                 ``alpha_k min(1, clip_norm / d_k)``, not normalised
==========  ======================================  ================================================================

A client whose distance is not finite (a NaN / Inf model) gets weight 0 and ``alpha`` is renormalised over the others; with
none left the model does not move.  ``ops/csrc/distance_agg.cuh`` defines the arithmetic, ``ops.reference.distance_aggregate``
transcribes it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np

# codes of AggKind (robust_agg.cuh) and DistAggKind (distance_agg.cuh)
KINDS = {"mean": 0, "median": 1, "trimmed_mean": 2, "geomed": 3, "norm_clip": 4}
COORDINATE_WISE = ("median", "trimmed_mean")
DISTANCE_BASED = ("geomed", "norm_clip")
GEOMED_MAX_ITERS = 16


@dataclass(frozen=True)
class Aggregator:
    """How the client models are combined into the average.  ``trim_fraction`` (``beta`` in [0, 0.5)) is used by
    ``trimmed_mean`` only; ``iters`` (1..16) and ``eps`` (finite, > 0) by ``geomed``; ``clip_norm`` (finite, > 0, no
    default) by ``norm_clip``, which requires it."""
    kind: str = "mean"
    trim_fraction: float = 0.1
    iters: int = 3
    eps: float = 1e-6
    clip_norm: Optional[float] = None

    def __post_init__(self) -> None:
        if self.kind not in KINDS:
            raise ValueError(f"unknown aggregator {self.kind!r}; expected one of {', '.join(KINDS)}")
        beta = float(self.trim_fraction)
        if not (math.isfinite(beta) and 0.0 <= beta < 0.5):
            raise ValueError(f"trim fraction must lie in [0, 0.5), got {self.trim_fraction}")
        object.__setattr__(self, "trim_fraction", beta)
        if int(self.iters) != self.iters or not 1 <= int(self.iters) <= GEOMED_MAX_ITERS:
            raise ValueError(f"geomed iterations must be an integer in 1..{GEOMED_MAX_ITERS}, got {self.iters}")
        object.__setattr__(self, "iters", int(self.iters))
        # the kernels take eps and the clip as float32: both must stay finite and > 0 there
        eps = float(self.eps)
        if not (math.isfinite(eps) and eps > 0.0 and math.isfinite(float(np.float32(eps))) and float(np.float32(eps)) > 0.0):
            raise ValueError(f"geomed eps must be finite and > 0, got {self.eps}")
        object.__setattr__(self, "eps", eps)
        if self.clip_norm is not None:
            tau = float(self.clip_norm)
            if not (math.isfinite(tau) and tau > 0.0 and math.isfinite(float(np.float32(tau))) and float(np.float32(tau)) > 0.0):
                raise ValueError(f"clip norm must be finite and > 0, got {self.clip_norm}")
            object.__setattr__(self, "clip_norm", tau)
        elif self.kind == "norm_clip":
            raise ValueError("aggregator 'norm_clip' needs a clip norm (--clip-norm): it has no default")

    @property
    def code(self) -> int:
        return KINDS[self.kind]

    @property
    def robust(self) -> bool:
        """Any kind but the plain mean."""
        return self.kind != "mean"

    @property
    def coordinate_wise(self) -> bool:
        """``median`` / ``trimmed_mean``: per parameter, unweighted."""
        return self.kind in COORDINATE_WISE

    @property
    def distance_based(self) -> bool:
        """``geomed`` / ``norm_clip``: per client, from its L2 distance; weighted."""
        return self.kind in DISTANCE_BASED

    @property
    def weighted(self) -> bool:
        """Whether the FedAvg weights ``alpha_k`` enter the aggregate (the mean and the distance-based kinds)."""
        return not self.coordinate_wise

    @property
    def clip(self) -> float:
        """The clip norm the kernels take (0 unless ``norm_clip``)."""
        return float(self.clip_norm) if self.kind == "norm_clip" else 0.0

    @property
    def trim(self) -> float:
        """The trim fraction the kernels take (0 unless ``trimmed_mean``)."""
        return self.trim_fraction if self.kind == "trimmed_mean" else 0.0
