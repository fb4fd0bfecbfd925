"""Attack categorisation: a model of the target :data:`fl.targets.CATEGORY` (``ffnn_category``) is trained and evaluated on
the attack category of every row (``data.CATEGORIES``: Normal, DDoS, DoS, Reconnaissance, Theft) instead of the binary
``attack`` label; :mod:`fl.targets` picks those labels (``data.category_tensors``: the dataset's category codes; a dataset
without them is refused).  This module holds what its federated-evaluation record adds to the usual per-class and macro
metrics (:func:`record`): the class names and the binary detection view of the same summed summary, so that its numbers
compare line for line with the binary FFNN's.
"""
from __future__ import annotations

from typing import Any, Dict, Optional, Sequence

from ..data.datasets import CATEGORIES
from . import fedeval
from .fedeval import _auc_ap, _div


def attack_view(s: fedeval.Summary) -> Dict[str, Any]:
    """Normal vs any attack from a category model's summary.  The counts collapse the C x C confusion matrix (true x predicted)
    to class 0 vs the rest, attack positive; ROC-AUC and AP come from the class-0 histogram pair, which ranks the rows by the
    probability of Normal: read from the highest bin down for Normal, so from the lowest bin up for attacks."""
    conf = s.confusion
    tn, fp = int(conf[0, 0]), int(conf[0, 1:].sum())
    fn, tp = int(conf[1:, 0].sum()), int(conf[1:, 1:].sum())
    recall = _div(tp, tp + fn)
    auc, ap = _auc_ap(s.hist[0, 1][::-1], s.hist[0, 0][::-1])
    return {"tp": tp, "fp": fp, "tn": tn, "fn": fn, "detection_rate": recall, "fpr": _div(fp, fp + tn),
            "precision": _div(tp, tp + fp), "f1": _div(2 * tp, 2 * tp + fp + fn), "auc": auc, "ap": ap}


def record(summaries: Dict[str, Optional[fedeval.Summary]], excluded: Sequence[str] = (),
           missing: Sequence[str] = ()) -> Dict[str, Any]:
    """``fedeval.record`` plus ``classes`` (the names) and ``attack`` (:func:`attack_view` of the summed summary, None
    without one)"""
    rec = fedeval.record(summaries, excluded, missing)
    tot = fedeval.add([v for v in summaries.values() if v is not None])
    rec["classes"] = list(CATEGORIES)
    rec["attack"] = attack_view(tot) if tot is not None else None
    return rec
