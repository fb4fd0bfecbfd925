"""Local optimizers of a device's fit: SGD with momentum / nesterov / weight decay, and Adam.

Every fit request names its optimizer the way ``torch.optim`` and PySyft's ``TrainConfig`` spell it (``FitConfig.optimizer``,
``"SGD"`` or ``"Adam"``) and may carry its arguments (``FitConfig.optimizer_args``).  This module is the only place that knows
those names, their arguments, their ranges and their wire form.

The state lives for one fit, as PySyft builds a fresh optimizer per ``TrainConfig``: the moments start at 0 and Adam's step
count at 1 at the beginning of every fit, and the step count counts optimizer steps (batches) across all epochs of that fit.
Nothing is carried between rounds.  Each step follows ``torch.optim``'s single-tensor SGD and Adam in float32, on the batch
gradient ``g`` the kernels form (the mean over the batch; a sum for ``sse``)::

    g <- g + wd * theta                                  (wd != 0)
    SGD   b <- g (first step), b <- mu * b + g;  d <- g + mu * b (nesterov) or b (mu = 0: d = g);  theta <- theta - lr * d
    Adam  m <- b1 * m + (1 - b1) * g;  v <- b2 * v + (1 - b2) * g^2;  p1 <- p1 * b1, p2 <- p2 * b2 (from 1, in float32)
          theta <- theta - ((lr / (1 - p1)) * m) / (sqrt(v) / sqrt(1 - p2) + eps)

``ops/csrc/local_opt.cuh`` writes that operation order down for the kernels and the host executor, and
``ops.reference.local_opt_step`` for PyTorch.  Plain SGD (no momentum, no weight decay) is today's fit and runs the kernels it
always ran; any other optimizer trains on the persistent kernel's optimizer instances (``ops.mlp_local_sgd(local_opt=...)``), or on
the layer-wise wgmma trainer's optimizer epilogue (``fl/layerwise.py``) for the MLPs that have no persistent kernel.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Mapping, Optional, Tuple

KINDS = {"SGD": 1, "Adam": 2}          # LocalOptKind of local_opt.cuh
ARGS = {"SGD": ("momentum", "nesterov", "weight_decay", "dampening", "maximize"),
        "Adam": ("betas", "eps", "weight_decay", "amsgrad", "maximize")}


def _finite(name: str, v: Any) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise ValueError(f"local optimizer: {name} must be a number, got {v!r}")
    f = float(v)
    if not math.isfinite(f):
        raise ValueError(f"local optimizer: {name} must be finite, got {f}")
    return f


@dataclass(frozen=True)
class LocalOpt:
    """One fit's optimizer.  ``kind`` is ``"SGD"`` (reads ``momentum``, ``nesterov``, ``weight_decay``) or ``"Adam"`` (reads
    ``betas``, ``eps``, ``weight_decay``); the constructor refuses what the kernels cannot run, with the reason."""
    kind: str = "SGD"
    momentum: float = 0.0
    nesterov: bool = False
    weight_decay: float = 0.0
    betas: Tuple[float, float] = (0.9, 0.999)
    eps: float = 1e-8

    def __post_init__(self) -> None:
        if not isinstance(self.kind, str) or self.kind not in KINDS:
            raise ValueError(f"unknown local optimizer {self.kind!r}; expected one of {', '.join(KINDS)}")
        mu = _finite("momentum", self.momentum)
        if not 0.0 <= mu < 1.0:
            raise ValueError(f"local optimizer: momentum must lie in [0, 1), got {mu}")
        if not isinstance(self.nesterov, bool):
            raise ValueError(f"local optimizer: nesterov must be true or false, got {self.nesterov!r}")
        if self.nesterov and mu == 0.0:
            raise ValueError("local optimizer: nesterov needs momentum > 0")
        wd = _finite("weight_decay", self.weight_decay)
        if wd < 0.0:
            raise ValueError(f"local optimizer: weight_decay must be >= 0, got {wd}")
        betas = tuple(self.betas) if isinstance(self.betas, (list, tuple)) else None
        if betas is None or len(betas) != 2:
            raise ValueError(f"local optimizer: betas must be two numbers, got {self.betas!r}")
        betas = tuple(_finite("betas", b) for b in betas)
        for b in betas:
            if not 0.0 <= b < 1.0:
                raise ValueError(f"local optimizer: betas must lie in [0, 1), got {betas}")
        eps = _finite("eps", self.eps)
        if not eps > 0.0:
            raise ValueError(f"local optimizer: eps must be > 0, got {eps}")
        if self.kind == "Adam" and (mu != 0.0 or self.nesterov):
            raise ValueError("local optimizer: Adam takes no momentum or nesterov (use betas)")
        object.__setattr__(self, "momentum", mu)
        object.__setattr__(self, "weight_decay", wd)
        object.__setattr__(self, "betas", betas)
        object.__setattr__(self, "eps", eps)

    def is_plain(self) -> bool:
        """SGD with no momentum and no weight decay: the fit the register-resident kernels have always run"""
        return self.kind == "SGD" and self.momentum == 0.0 and self.weight_decay == 0.0

    @property
    def code(self) -> int:
        return KINDS[self.kind]

    def launch_args(self) -> List[float]:
        """``[kind, nesterov, momentum, weight_decay, beta1, beta2, eps]``: the ``LocalOptArgs`` the bindings take"""
        return [float(self.code), float(self.nesterov), self.momentum, self.weight_decay, self.betas[0], self.betas[1], self.eps]

    def args(self) -> Dict[str, Any]:
        """The arguments of this kind, as ``torch.optim`` names them (``optimizer_args`` on the wire)"""
        if self.kind == "SGD":
            return {"momentum": self.momentum, "nesterov": self.nesterov, "weight_decay": self.weight_decay}
        return {"betas": list(self.betas), "eps": self.eps, "weight_decay": self.weight_decay}

    def record(self) -> Dict[str, Any]:
        """What a round record and a training result carry: ``{kind, ...its arguments}``"""
        return {"kind": self.kind, **self.args()}

    def torch_optimizer(self, params, lr: float):
        """The ``torch.optim`` optimizer this stands for (user-registered modules train through autograd)"""
        import torch
        if self.kind == "SGD":
            return torch.optim.SGD(params, lr=lr, momentum=self.momentum, nesterov=self.nesterov, weight_decay=self.weight_decay)
        return torch.optim.Adam(params, lr=lr, betas=self.betas, eps=self.eps, weight_decay=self.weight_decay)


PLAIN = LocalOpt()


def from_request(name: Optional[str], args: Optional[Mapping[str, Any]] = None) -> LocalOpt:
    """The optimizer a fit request names (``FitConfig.optimizer`` / ``optimizer_args``), or ValueError with the reason.
    Unknown names and arguments are refused; ``dampening != 0``, ``amsgrad`` and ``maximize`` are refused rather than
    ignored."""
    kind = "SGD" if name is None else name
    if not isinstance(kind, str) or kind not in KINDS:
        raise ValueError(f"unknown local optimizer {kind!r}; expected one of {', '.join(KINDS)}")
    args = {} if args is None else args
    if not isinstance(args, Mapping):
        raise ValueError(f"local optimizer arguments must be a mapping, got {type(args).__name__}")
    kw: Dict[str, Any] = {}
    for key, v in args.items():
        if key not in ARGS[kind]:
            raise ValueError(f"local optimizer {kind}: unknown argument {key!r} (accepted: {', '.join(ARGS[kind])})")
        if key == "dampening":
            if _finite("dampening", v) != 0.0:
                raise ValueError("local optimizer SGD: dampening != 0 is not supported")
        elif key in ("amsgrad", "maximize"):
            if v is not False:
                raise ValueError(f"local optimizer {kind}: {key}={v!r} is not supported")
        else:
            kw[key] = v
    return LocalOpt(kind, **kw)


def resolve(local_opt: Optional[LocalOpt]) -> Optional[LocalOpt]:
    """None for plain SGD (the call of before optimizers existed), the optimizer otherwise"""
    return None if local_opt is None or local_opt.is_plain() else local_opt


def wire(local_opt: Optional[LocalOpt]) -> Tuple[str, Optional[Dict[str, Any]]]:
    """``(FitConfig.optimizer, FitConfig.optimizer_args)``: ``("SGD", None)`` for plain SGD, so that a default request is
    byte for byte the one it was before optimizers existed"""
    lo = resolve(local_opt)
    return ("SGD", None) if lo is None else (lo.kind, lo.args())


def refuse_non_plain(local_opt: Optional[LocalOpt], what: str) -> None:
    """ValueError when a trainer without optimizer instances is asked for anything but plain SGD"""
    if resolve(local_opt) is not None:
        raise ValueError(f"local optimizer {local_opt.kind} {local_opt.args()}: {what} trains with plain SGD only "
                         "(momentum, weight decay and Adam run on the persistent-kernel MLPs and the layer-wise MLP trainer)")
