"""Byzantine-robust aggregation of the client models (Yin et al., *Byzantine-Robust Distributed Learning: Towards Optimal
Statistical Rates*, ICML 2018).

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
"""
from __future__ import annotations

import math
from dataclasses import dataclass

KINDS = {"mean": 0, "median": 1, "trimmed_mean": 2}   # codes of AggKind (robust_agg.cuh)


@dataclass(frozen=True)
class Aggregator:
    """How the client models are combined into the average.  ``trim_fraction`` (``beta`` in [0, 0.5)) is used by
    ``trimmed_mean`` only."""
    kind: str = "mean"
    trim_fraction: float = 0.1

    def __post_init__(self) -> None:
        if self.kind not in KINDS:
            raise ValueError(f"unknown aggregator {self.kind!r}; expected one of {', '.join(KINDS)}")
        beta = float(self.trim_fraction)
        if not (math.isfinite(beta) and 0.0 <= beta < 0.5):
            raise ValueError(f"trim fraction must lie in [0, 0.5), got {self.trim_fraction}")
        object.__setattr__(self, "trim_fraction", beta)

    @property
    def code(self) -> int:
        return KINDS[self.kind]

    @property
    def robust(self) -> bool:
        return self.kind != "mean"

    @property
    def trim(self) -> float:
        """The trim fraction the kernels take (0 unless ``trimmed_mean``)."""
        return self.trim_fraction if self.kind == "trimmed_mean" else 0.0
