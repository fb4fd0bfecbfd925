"""Class-weighted training: how the per-class loss weights of a training are chosen, checked and recorded.

A class-weighted fit multiplies row i's loss term and gradient by ``w[c_i]``, the weight of its class (the 0 / 1 label of the
binary FFNN, the attack category of ``ffnn_category``), while the batch reductions stay as they are (``ops/reference.py::
loss_and_dz``; the kernels: ``ops/csrc/mlp_persistent_cw.cu``).  The weights are one vector per training, the same on every
device:

* ``--class-weight w0,w1,...``: given by the user (``mode: "given"``);
* ``--class-weight balanced``: ``w_c = min(cap, N / (C * N_c))`` from the class counts ``N_c`` of every device's training rows
  (``N = sum N_c``; a class no device holds gets 1), the usual balanced weighting, federated: local mode counts its virtual
  workers' shards, remote mode asks each device for its counts once per training (the ``class_counts`` request).

This module is the only one that computes or checks weights; the control plane asks it and ships the vector in the fit
config (``FitConfig.class_weights``).  How many classes a model has is its target's answer (``fl/targets.py``).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import torch

DEFAULT_CAP = 10.0
_MAX_COUNT = 2 ** 53          # a count reply above this is not an exact float64 integer


@dataclass(frozen=True)
class Setting:
    """What ``--class-weight`` asks for: ``balanced`` (weights from the federated counts, capped at ``cap``) or ``given``"""

    mode: str
    classes: int
    cap: float = DEFAULT_CAP
    given: Optional[List[float]] = None


def setting(args, classes: Optional[int], box: bool = False, encryption: bool = False) -> Optional[Setting]:
    """The :class:`Setting` of ``args.class_weight`` / ``args.class_weight_max`` for a model of ``classes`` classes (None: the
    model has no class-weighted kernel), None without ``--class-weight``; ValueError with the reason for a setting that cannot
    train"""
    spec = getattr(args, "class_weight", None)
    cap = float(getattr(args, "class_weight_max", DEFAULT_CAP))
    if spec is None:
        if cap != DEFAULT_CAP:
            raise ValueError("--class-weight-max applies to --class-weight balanced, which is not set")
        return None
    if box:
        raise ValueError("--class-weight does not run in box mode (--box): the star / engine path launches the unweighted kernels")
    if encryption:
        raise ValueError("--class-weight does not run with -e: the secret-shared trainer launches the unweighted kernels")
    if classes is None:
        raise ValueError(f"--class-weight does not apply to --model {args.model}: only the binary FFNN (ffnn) and ffnn_category "
                         "have class-weighted kernels")
    if not (math.isfinite(cap) and cap > 0):
        raise ValueError(f"--class-weight-max must be a finite number > 0, not {cap}")
    text = str(spec).strip()
    if text == "balanced":
        if getattr(args, "secure_agg", False):
            raise ValueError("--class-weight balanced does not combine with --secure-agg: every device's class counts would reveal "
                             "the label mix of its data, which secure aggregation hides (give the weights as a list instead)")
        return Setting("balanced", classes, cap)
    if cap != DEFAULT_CAP:
        raise ValueError("--class-weight-max applies to --class-weight balanced only")
    try:
        given = [float(v) for v in text.split(",")]
    except ValueError:
        raise ValueError(f"--class-weight takes 'balanced' or {classes} comma-separated numbers >= 0, not {text!r}") from None
    return Setting("given", classes, cap, check_weights(given, classes, "--class-weight"))


def check_weights(w: Any, classes: int, what: str = "class weights") -> List[float]:
    """``w`` as a list of floats, or ValueError: exactly ``classes`` finite numbers >= 0 (untrusted input: a fit request)"""
    if not isinstance(w, (list, tuple)) or len(w) != classes:
        raise ValueError(f"{what}: {classes} weights expected, one per class, not {w!r}")
    out = []
    for c, v in enumerate(w):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
            raise ValueError(f"{what}: weight {v!r} of class {c} is not a finite number >= 0")
        out.append(float(v))
    return out


def count(y: torch.Tensor, classes: int) -> List[int]:
    """The class counts of a fit's training rows ``y`` (their first column: the 0 / 1 label or the class index); ValueError for
    a label that is not a class index"""
    v = y.detach().reshape(y.shape[0], -1)[:, 0].double().cpu() if y.numel() else torch.zeros(0, dtype=torch.float64)
    if bool(((v != v.floor()) | (v < 0) | (v >= classes)).any()):
        raise ValueError(f"a training label is not a class index in [0, {classes})")
    return [int(n) for n in torch.bincount(v.long(), minlength=classes).tolist()]


def balanced(counts: Sequence[int], cap: float = DEFAULT_CAP) -> List[float]:
    """``w_c = min(cap, N / (C * N_c))`` in float64 (``N = sum counts``, ``C = len(counts)``), 1 for a class without rows, cast
    once to float32 (the values the kernels multiply with)"""
    n, c = float(sum(counts)), len(counts)
    w = np.array([min(cap, n / (c * float(k))) if k > 0 else 1.0 for k in counts], dtype=np.float64)
    return [float(v) for v in w.astype(np.float32)]


def check_counts(reply: Dict[str, Any], classes: int) -> List[int]:
    """The counts of a device's ``class_counts`` reply, or ValueError: ``ok`` and a list of exactly ``classes`` non-negative
    Python ints (not bools) below 2^53"""
    if not isinstance(reply, dict) or not reply.get("ok"):
        raise ValueError(str(reply.get("error") if isinstance(reply, dict) else reply))
    got = reply.get("counts")
    if not isinstance(got, list) or len(got) != classes:
        raise ValueError(f"counts must be a list of {classes} integers, not {got!r}")
    for v in got:
        if isinstance(v, bool) or not isinstance(v, int) or v < 0 or v >= _MAX_COUNT:
            raise ValueError(f"count {v!r} is not an integer in [0, 2^53)")
    return list(got)


def record(st: Setting, weights: Sequence[float], counts: Optional[Sequence[int]] = None,
           excluded: Sequence[str] = ()) -> Dict[str, Any]:
    """The ``class_weights`` block of the training result and of the training's first round record"""
    return {"mode": st.mode, "counts": None if counts is None else [int(v) for v in counts], "weights": [float(v) for v in weights],
            "excluded": list(excluded)}


class NoCounts(ValueError):
    """No device answered usable class counts: the training cannot form its weights"""


def weights_from(st: Setting, per_device: Dict[str, Any]) -> Dict[str, Any]:
    """The record of a training from the devices' ``class_counts`` replies (``per_device``: id -> reply); ``balanced`` only.  A
    device whose reply fails :func:`check_counts` is listed under ``excluded``; :class:`NoCounts` when every device is."""
    total, excluded = [0] * st.classes, []
    for wid, reply in per_device.items():
        try:
            got = check_counts(reply, st.classes)
        except (ValueError, AttributeError):
            excluded.append(wid)
            continue
        total = [a + b for a, b in zip(total, got)]
    if len(excluded) == len(per_device):
        raise NoCounts(f"no device answered usable class counts (excluded: {', '.join(excluded) or 'none'})")
    return record(st, balanced(total, st.cap), total, excluded)


def local(st: Setting, labels: Sequence[torch.Tensor]) -> Dict[str, Any]:
    """The record of a local-mode training from its virtual workers' training labels"""
    if st.mode == "given":
        return record(st, st.given)
    total = [0] * st.classes
    for y in labels:
        total = [a + b for a, b in zip(total, count(y, st.classes))]
    return record(st, balanced(total, st.cap), total)
