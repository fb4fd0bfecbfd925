"""Federated anomaly detection: an autoencoder (a model whose ``spec.target`` is ``"input"``) is trained on every device's
benign rows to reconstruct them; a row whose reconstruction error lies at or above the federated alarm threshold is an
alarm.  The devices agree on the threshold without pooling their data: each returns an additive summary of its held-out
rows, and the coordinator picks the threshold from the sum.

This is the only module that knows these rules:

* **Training rows.**  A device trains on its rows labelled 0 (benign), with the input itself as the target: the kernel's
  ``y`` is the shard's ``x`` (``y_dim`` = D), so nothing is copied twice.  ``n_k`` of ``--weighted`` is the benign count.
  The labels of held-out rows are used only to score.
* **Error and bins** (``ops/csrc/recon_summary.cuh``): ``e = sum_c (xhat_c - x_c)^2`` in float64 from fp32 differences; the
  bin of ``e`` comes from the bits of ``(float)e``: 32 octaves ``[2^-24, 2^8)`` of ``bins / 32`` sub-bins each, below them
  bin 0, above them bin ``bins - 1``.  A summary holds ``n``, ``n_invalid``, the error histograms of label 0 and label 1 and
  the float64 error sum; on the wire the histograms travel as little-endian uint32 words.
* **Threshold.**  With ``H0`` the benign histogram of the sum and ``N0`` its total, the alarm bin is
  ``j* = min j in [0, bins]`` with ``sum_{b >= j} H0[b] <= floor(fpr N0)``, None when ``N0 = 0``.  A row is an alarm iff
  ``bin(e) >= j*``; the threshold reported is the lower edge of bin ``j*`` (``inf`` for ``j* = bins``: no alarm).  On the
  held-out benign rows the false-alarm rate is ``<= fpr`` by construction.
* **Metrics** from the two histograms: mean error, false-alarm and detection rate, precision, F1 at ``j*``, and ROC-AUC and
  AP by the formulas of :mod:`fl.fedeval`.
* **Replies**: exact word counts, non-negative counts, ``sum(hist) == n - n_invalid``, a finite error sum ``>= 0``.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import ops
from .fedeval import _auc_ap, _div

MIN_BINS = 32


def is_autoencoder(model) -> bool:
    """True for a model trained to reconstruct its input (``MLPSpec.target == "input"``)"""
    spec = getattr(model, "spec", None)
    return spec is not None and getattr(spec, "target", "label") == "input"


def training_rows(x: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(x_benign, x_benign)``: the rows labelled 0 as input and target (one tensor, passed twice)"""
    xb = x[y.reshape(-1) == 0].contiguous()
    return xb, xb


@dataclass
class ReconSummary:
    bins: int
    n: int
    n_invalid: int
    err_sum: float
    hist: np.ndarray        # int64 [2, bins]: label 0, label 1


def _summaries(counts: torch.Tensor, total: torch.Tensor, bins: int) -> List[ReconSummary]:
    counts, total = counts.cpu().numpy(), total.cpu().tolist()
    return [ReconSummary(int(bins), int(c[0]), int(c[1]), float(t), c[2:].reshape(2, bins).copy()) for c, t in zip(counts, total)]


@torch.no_grad()
def summarize(model, flat: torch.Tensor, x: torch.Tensor, y: Optional[torch.Tensor], bins: int,
              segments: Optional[Sequence[int]] = None) -> List[ReconSummary]:
    """One :class:`ReconSummary` per segment of consecutive rows of ``x`` (all rows when ``segments`` is None) of the
    autoencoder whose parameters are ``flat``: one forward (``ops.mlp_forward``), one ``ops.recon_summary`` launch."""
    from .evaluate import forward_flat
    if not is_autoencoder(model):
        raise ValueError("the reconstruction summary needs an autoencoder (a model trained on its input)")
    x = x.to(flat.device).float()
    xhat = forward_flat(model, flat, x)
    counts, total, _, _ = ops.recon_summary(xhat, x, None if y is None else y.reshape(-1).to(x.device).float(), bins, segments)
    return _summaries(counts, total, bins)


@torch.no_grad()
def predict(model, flat: torch.Tensor, x: torch.Tensor, alarm_bin: int, bins: int) -> torch.Tensor:
    """Per-row alarms (uint8 0 / 1) of the autoencoder ``flat`` at ``alarm_bin``; a row with a non-finite value is an alarm"""
    from .evaluate import forward_flat
    x = x.to(flat.device).float()
    xhat = forward_flat(model, flat, x)
    return ops.recon_summary(xhat, x, None, bins, None, int(alarm_bin))[3]


def add(summaries: Sequence[ReconSummary]) -> Optional[ReconSummary]:
    if not summaries:
        return None
    bins = summaries[0].bins
    if any(s.bins != bins for s in summaries):
        raise ValueError("summaries of different bin counts cannot be added")
    return ReconSummary(bins, sum(s.n for s in summaries), sum(s.n_invalid for s in summaries), float(sum(s.err_sum for s in summaries)),
                        np.sum([s.hist for s in summaries], axis=0).astype(np.int64))


def check(s: ReconSummary) -> ReconSummary:
    """A device's summary is untrusted input (ValueError with the reason)"""
    if s.hist.shape != (2, s.bins):
        raise ValueError(f"histogram of shape {s.hist.shape}, expected (2, {s.bins})")
    if s.n < 0 or s.n_invalid < 0 or s.n_invalid > s.n or bool((s.hist < 0).any()):
        raise ValueError("negative counts")
    if int(s.hist.sum()) != s.n - s.n_invalid:
        raise ValueError(f"histograms sum to {int(s.hist.sum())}, {s.n - s.n_invalid} valid rows reported")
    if not (math.isfinite(s.err_sum) and s.err_sum >= 0.0):
        raise ValueError(f"err_sum {s.err_sum!r} is not a finite value >= 0")
    return s


def to_wire(s: ReconSummary) -> Dict[str, Any]:
    if s.n >= 1 << 32:
        raise ValueError("more than 2^32 - 1 evaluation rows do not fit the uint32 counts")
    return {"bins": s.bins, "n": s.n, "n_invalid": s.n_invalid, "err_sum": s.err_sum, "counts": s.hist.reshape(-1).astype("<u4").tobytes()}


def from_wire(reply: Dict[str, Any], bins: int) -> ReconSummary:
    """The :class:`ReconSummary` of an ``evaluate`` reply after :func:`check`, for the ``bins`` the coordinator asked for"""
    raw = reply.get("counts")
    if not isinstance(raw, (bytes, bytearray)) or len(raw) != 8 * bins:
        raise ValueError(f"counts of {len(raw) if isinstance(raw, (bytes, bytearray)) else type(raw).__name__} bytes, expected {8 * bins}")
    n, bad, err = reply.get("n"), reply.get("n_invalid"), reply.get("err_sum")
    if not all(isinstance(v, int) and not isinstance(v, bool) for v in (n, bad)) or not isinstance(err, (int, float)) or isinstance(err, bool):
        raise ValueError("n / n_invalid must be integers and err_sum a number")
    hist = np.frombuffer(bytes(raw), dtype="<u4").astype(np.int64).reshape(2, bins)
    return check(ReconSummary(int(bins), n, bad, float(err), hist))


def alarm_bin(h0: np.ndarray, fpr: float) -> Optional[int]:
    """``j* = min j in [0, B]`` with ``sum_{b >= j} h0[b] <= floor(fpr N0)``; None when ``N0 = 0``"""
    n0 = int(np.sum(h0))
    if n0 == 0:
        return None
    budget = math.floor(fpr * n0)
    tail = 0
    for j in range(len(h0) - 1, -1, -1):
        tail += int(h0[j])
        if tail > budget:
            return j + 1
    return 0


def bin_edge(j: int, bins: int) -> float:
    """The lower edge of bin ``j`` (exact): 0 for bin 0, ``inf`` for ``j = bins`` (no row reaches it)"""
    if j == 0:
        return 0.0
    if j >= bins:
        return math.inf
    sub = bins // MIN_BINS
    return math.ldexp(sub + j % sub, j // sub - 24 - (sub.bit_length() - 1))


def metrics(s: ReconSummary, j: Optional[int]) -> Dict[str, Any]:
    """The detection metrics of a summary at alarm bin ``j``; an undefined value is None, never NaN"""
    valid = s.n - s.n_invalid
    h0, h1 = s.hist[0], s.hist[1]
    mean = _div(s.err_sum, valid)
    out: Dict[str, Any] = {"n": s.n, "n_invalid": s.n_invalid, "mean_error": mean, "loss": mean}
    auc, ap = _auc_ap(h0, h1)
    n0, n1 = int(h0.sum()), int(h1.sum())
    if j is None:
        out.update(tp=None, fp=None, tn=None, fn=None, accuracy=None, precision=None, recall=None, detection_rate=None, fpr=None,
                   f1=None, auc=auc, ap=ap)
        return out
    fp, tp = int(h0[j:].sum()), int(h1[j:].sum())
    tn, fn = n0 - fp, n1 - tp
    recall = _div(tp, n1)
    out.update(tp=tp, fp=fp, tn=tn, fn=fn, accuracy=_div(tp + tn, s.n), precision=_div(tp, tp + fp), recall=recall, detection_rate=recall,
               fpr=_div(fp, n0), f1=_div(2 * tp, 2 * tp + fp + fn), auc=auc, ap=ap)
    return out


def record(summaries: Dict[str, ReconSummary], fpr: float, bins: int, excluded: Sequence[str] = (),
           missing: Sequence[str] = ()) -> Dict[str, Any]:
    """The ``fed_eval`` field of a round record: the alarm bin and threshold chosen from the sum of the summaries that passed
    the checks, the metrics of every device and of the sum at that bin, and the devices left out (as in fl/fedeval.py)"""
    tot = add(list(summaries.values()))
    j = alarm_bin(tot.hist[0], fpr) if tot is not None else None
    return {"devices": {k: metrics(v, j) for k, v in summaries.items()}, "total": metrics(tot, j) if tot is not None else None,
            "eval_excluded": list(excluded), "eval_missing": list(missing), "alarm_bin": j,
            "threshold": bin_edge(j, bins) if j is not None else None, "bins": int(bins), "fpr": float(fpr)}


def checkpoint_meta(rec: Optional[Dict[str, Any]]) -> Dict[str, Any]:
    """The ``anomaly`` entry of a checkpoint's JSON sidecar from the last ``fed_eval`` record (no threshold without one)"""
    rec = rec or {}
    return {k: rec.get(k) for k in ("alarm_bin", "bins", "threshold", "fpr")}


def check_settings(args, box: bool = False, encryption: bool = False) -> None:
    """The settings an autoencoder needs (ValueError with the reason): a threshold is only chosen by federated evaluation,
    with at least 32 bins and no classifier threshold; box mode all-gathers classifier summaries and -e exchanges shares"""
    if box:
        raise ValueError("--model autoencoder does not run in box mode (--box): its federated evaluation all-gathers classifier summaries")
    if encryption:
        raise ValueError("--model autoencoder does not run with -e: the encrypted fit trains classifiers on secret shares")
    if args.fed_eval_every < 1:
        raise ValueError("--model autoencoder needs --fed-eval-every N >= 1: the alarm threshold is chosen by federated evaluation, "
                         "and a model saved without one cannot flag anything")
    if args.eval_threshold != 0.5:
        raise ValueError("--eval-threshold applies to classifiers: the autoencoder's threshold follows from --alarm-fpr")
    if args.eval_bins < MIN_BINS:
        raise ValueError(f"--model autoencoder needs --eval-bins >= {MIN_BINS} (32 octaves of reconstruction error), not {args.eval_bins}")
    if not 0.0 < args.alarm_fpr < 1.0:
        raise ValueError(f"--alarm-fpr must be in (0, 1), not {args.alarm_fpr}")
