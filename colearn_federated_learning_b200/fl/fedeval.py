"""Federated evaluation: every device scores the global model on rows it keeps out of training and returns only additive
counts; the coordinator sums them and derives the detection metrics.  The union of the devices' data is never gathered.

This is the only module that knows the summary format (``ops/csrc/eval_summary.cuh``): per device ``n``, ``n_invalid``, a
float64 ``loss_sum`` and the counts — the ``C' x C'`` confusion matrix (true class x predicted class, ``C' = 2`` for a
one-column sigmoid head) followed by ``C`` score histograms of ``2 x bins`` bins (row 0: rows of the other classes, row 1:
rows of the histogram's class; C = 1: the histogram of p, row 1 = label 1).  On the wire the counts travel as little-endian
uint32 words.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import ops


@dataclass
class Summary:
    classes: int            # C, the model's output columns
    bins: int
    n: int
    n_invalid: int
    loss_sum: float
    counts: np.ndarray      # int64 [C'^2 + C 2 bins]

    @property
    def labels(self) -> int:
        return 2 if self.classes == 1 else self.classes

    @property
    def confusion(self) -> np.ndarray:
        k = self.labels
        return self.counts[:k * k].reshape(k, k)

    @property
    def hist(self) -> np.ndarray:
        k = self.labels
        return self.counts[k * k:].reshape(self.classes, 2, self.bins)


def count_words(classes: int, bins: int) -> int:
    k = 2 if classes == 1 else classes
    return k * k + classes * 2 * bins


def split_eval(x: torch.Tensor, y: torch.Tensor, fraction: float, seed: int):
    """``(x_train, y_train, x_eval, y_eval)``: the first ``floor(fraction n)`` indices of ``randperm(n)`` (generator seeded with
    ``seed``) are held out for evaluation, the training rows keep their original order (a dataset ordered by category, as
    the Bot-IoT CSV is, would give a biased contiguous tail)."""
    if not 0.0 <= fraction < 1.0:
        raise ValueError(f"the evaluation fraction must be in [0, 1), not {fraction}")
    n = int(x.shape[0])
    k = int(math.floor(fraction * n))
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(int(seed)))
    held = perm[:k]
    keep = torch.ones(n, dtype=torch.bool)
    keep[held] = False
    held, keep = held.to(x.device), keep.to(x.device)
    return x[keep], y[keep], x[held], y[held]


def check_model(model) -> int:
    """The number of output columns C the summary of ``model`` has (ValueError for a model it cannot score).  A one-column
    model must end in a sigmoid: its output is then a score in [0, 1] (``testing_remote`` regresses).  C is the width of the
    last layer: ``spec.dims[-1]`` of an MLP, otherwise the ``out_features`` of the module's last ``nn.Linear``."""
    spec = getattr(model, "spec", None)
    if spec is not None:
        if spec.dims[-1] == 1 and spec.out_activation != "sigmoid":
            raise ValueError("federated evaluation needs a classifier: a one-column model without a sigmoid head has no score")
        return int(spec.dims[-1])
    linears = [m for m in model.modules() if isinstance(m, torch.nn.Linear)]
    if not linears:
        raise ValueError(f"federated evaluation cannot tell the output width of {type(model).__name__} (no nn.Linear head)")
    return int(linears[-1].out_features)


@torch.no_grad()
def summarize(model, flat: Optional[torch.Tensor], x: torch.Tensor, y: torch.Tensor, bins: int = 256, threshold: float = 0.5,
              segments: Optional[Sequence[int]] = None) -> List[Summary]:
    """One :class:`Summary` per segment of consecutive rows of ``x`` / ``y`` (all rows when ``segments`` is None) of the model
    whose parameters are ``flat``: one forward through ``forward_flat`` (persistent, layer-wise or conv-net inference), one
    ``ops.eval_summary`` launch.  ``flat`` is loaded into ``model`` first: the paths of ``forward_flat`` that run the module
    itself (a model that is not an MLP on the CPU, an MLP no persistent kernel covers on a GPU) would otherwise score whatever
    parameters it holds, e.g. the last local fit's."""
    from .evaluate import forward_flat
    from ..models import unflatten_params
    classes = check_model(model)
    if flat is not None:
        unflatten_params(model, flat)
    out = forward_flat(model, flat, x)
    out = out.view(-1, 1) if out.dim() == 1 else out
    if out.shape[1] != classes:
        raise ValueError(f"the model gave {out.shape[1]} output columns, its last layer has {classes}")
    counts, loss = ops.eval_summary(out.float(), y.reshape(-1).to(out.device).float(), bins, threshold, segments)
    counts, loss = counts.cpu().numpy(), loss.cpu().tolist()
    return [Summary(out.shape[1], int(bins), int(c[0]), int(c[1]), float(l), c[2:].copy()) for c, l in zip(counts, loss)]


def add(summaries: Sequence[Summary]) -> Optional[Summary]:
    """The sum of summaries of one shape (None for none)."""
    if not summaries:
        return None
    first = summaries[0]
    for s in summaries[1:]:
        if (s.classes, s.bins) != (first.classes, first.bins):
            raise ValueError("summaries of different shapes cannot be added")
    return Summary(first.classes, first.bins, sum(s.n for s in summaries), sum(s.n_invalid for s in summaries),
                   float(sum(s.loss_sum for s in summaries)), np.sum([s.counts for s in summaries], axis=0).astype(np.int64))


def check(s: Summary) -> Summary:
    """A device's summary is untrusted input: exact lengths, non-negative counts, ``sum(confusion) == n - n_invalid``, every
    histogram's class totals equal to the confusion row sums, a finite ``loss_sum >= 0``.  ValueError with the reason."""
    if s.counts.shape != (count_words(s.classes, s.bins),):
        raise ValueError(f"{s.counts.shape[0] if s.counts.ndim == 1 else s.counts.shape} count words, expected {count_words(s.classes, s.bins)}")
    if s.n < 0 or s.n_invalid < 0 or s.n_invalid > s.n or bool((s.counts < 0).any()):
        raise ValueError("negative counts")
    conf = s.confusion
    valid = s.n - s.n_invalid
    if int(conf.sum()) != valid:
        raise ValueError(f"confusion matrix sums to {int(conf.sum())}, {valid} valid rows reported")
    rows = conf.sum(1)
    h = s.hist.sum(2)
    pos = np.array([rows[1]]) if s.classes == 1 else rows
    if not (np.array_equal(h[:, 1], pos) and np.array_equal(h[:, 0], valid - pos)):
        raise ValueError("histogram class totals differ from the confusion matrix")
    if not (math.isfinite(s.loss_sum) and s.loss_sum >= 0.0):
        raise ValueError(f"loss_sum {s.loss_sum!r} is not a finite value >= 0")
    return s


def to_wire(s: Summary) -> Dict[str, Any]:
    if s.n >= 1 << 32:
        raise ValueError("more than 2^32 - 1 evaluation rows do not fit the uint32 counts")
    return {"classes": s.classes, "bins": s.bins, "n": s.n, "n_invalid": s.n_invalid, "loss_sum": s.loss_sum,
            "counts": s.counts.astype("<u4").tobytes()}


def from_wire(reply: Dict[str, Any], classes: int, bins: int) -> Summary:
    """The :class:`Summary` of an ``evaluate`` reply after :func:`check` (ValueError for a malformed one)."""
    raw = reply.get("counts")
    if not isinstance(raw, (bytes, bytearray)) or len(raw) != 4 * count_words(classes, bins):
        raise ValueError(f"counts of {len(raw) if isinstance(raw, (bytes, bytearray)) else type(raw).__name__} bytes, "
                         f"expected {4 * count_words(classes, bins)}")
    n, bad, loss = reply.get("n"), reply.get("n_invalid"), reply.get("loss_sum")
    if not all(isinstance(v, int) and not isinstance(v, bool) for v in (n, bad)) or not isinstance(loss, (int, float)) or isinstance(loss, bool):
        raise ValueError("n / n_invalid must be integers and loss_sum a number")
    counts = np.frombuffer(bytes(raw), dtype="<u4").astype(np.int64)
    return check(Summary(int(classes), int(bins), n, bad, float(loss), counts))


def _div(a, b) -> Optional[float]:
    return float(a) / float(b) if b else None


def _auc_ap(neg: np.ndarray, pos: np.ndarray) -> Tuple[Optional[float], Optional[float]]:
    """ROC-AUC (Mann-Whitney on the bin indices, ties counted 1/2) and average precision (sklearn's step sum over the bin
    thresholds, highest first) of one histogram pair; None without positives or negatives."""
    neg, pos = [int(v) for v in neg], [int(v) for v in pos]
    P, N = sum(pos), sum(neg)
    auc = None
    if P and N:
        above, num = 0, 0
        for b in range(len(pos) - 1, -1, -1):
            num += neg[b] * (2 * above + pos[b])
            above += pos[b]
        auc = num / (2 * P * N)
    ap = None
    if P:
        tp = fp = 0
        ap = 0.0
        for b in range(len(pos) - 1, -1, -1):
            if pos[b] == 0 and neg[b] == 0:
                continue
            tp += pos[b]
            fp += neg[b]
            ap += (pos[b] / P) * (tp / (tp + fp))
    return auc, ap


def _mean(vals) -> Optional[float]:
    v = [x for x in vals if x is not None]
    return sum(v) / len(v) if v else None


def metrics(s: Summary) -> Dict[str, Any]:
    """The detection metrics of a summary; an undefined value (no positives, no valid rows, ...) is None, never NaN.
    ``auc`` / ``ap`` / ``f1`` are the binary ones for a two-class model (class 1 positive) and the macro means otherwise."""
    conf = s.confusion
    valid = s.n - s.n_invalid
    out: Dict[str, Any] = {"n": s.n, "n_invalid": s.n_invalid, "loss": _div(s.loss_sum, valid),
                           "accuracy": _div(int(np.trace(conf)), s.n)}
    hist = s.hist
    if s.labels == 2:
        tn, fp, fn, tp = (int(v) for v in conf.reshape(-1))
        recall, fpr = _div(tp, tp + fn), _div(fp, fp + tn)
        auc, ap = _auc_ap(hist[-1, 0], hist[-1, 1])
        out.update(tp=tp, fp=fp, tn=tn, fn=fn, precision=_div(tp, tp + fp), recall=recall, detection_rate=recall, fpr=fpr,
                   f1=_div(2 * tp, 2 * tp + fp + fn),
                   balanced_accuracy=(recall + 1.0 - fpr) / 2 if recall is not None and fpr is not None else None, auc=auc, ap=ap)
    if s.classes >= 2:
        rows, cols = conf.sum(1), conf.sum(0)
        per = []
        for c in range(s.classes):
            d = int(conf[c, c])
            auc, ap = _auc_ap(hist[c, 0], hist[c, 1])
            per.append({"precision": _div(d, int(cols[c])), "recall": _div(d, int(rows[c])), "f1": _div(2 * d, int(rows[c] + cols[c])),
                        "auc": auc, "ap": ap})
        out["per_class"] = per
        out["macro_f1"] = _mean(p["f1"] for p in per)
        out["macro_auc"] = _mean(p["auc"] for p in per)
        out["macro_ap"] = _mean(p["ap"] for p in per)
        if s.labels != 2:
            out.update(f1=out["macro_f1"], auc=out["macro_auc"], ap=out["macro_ap"], detection_rate=None, fpr=None)
    return out


def record(summaries: Dict[str, Optional[Summary]], excluded: Sequence[str] = (), missing: Sequence[str] = ()) -> Dict[str, Any]:
    """The ``fed_eval`` field of a round record: per-device metrics of the summaries that passed the checks, the metrics of
    their sum, the devices whose reply failed the checks (``eval_excluded``) and those without evaluation data
    (``eval_missing``)."""
    good = {k: v for k, v in summaries.items() if v is not None}
    tot = add(list(good.values()))
    return {"devices": {k: metrics(v) for k, v in good.items()}, "total": metrics(tot) if tot is not None else None,
            "eval_excluded": list(excluded), "eval_missing": list(missing)}


def summary_line(m: Optional[Dict[str, Any]]) -> str:
    """loss, accuracy, detection rate, false-alarm rate and ROC-AUC of a metrics dict as one log line ('-': undefined)"""
    m = m or {}
    f = lambda k: "-" if m.get(k) is None else f"{m[k]:.6g}"  # noqa: E731
    return (f"loss {f('loss')} accuracy {f('accuracy')} detection rate {f('detection_rate')} false-alarm rate {f('fpr')} "
            f"auc {f('auc')}")
