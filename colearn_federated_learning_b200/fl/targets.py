"""What a model trains and is scored on: the only reader of ``MLPSpec.target``.

* :data:`LABEL` (``"label"``, and every model without a ``spec``): the dataset's labels, scored by :mod:`fl.fedeval`;
* :data:`INPUT` (``"input"``, the autoencoder): the benign rows, reconstructed; scored by the reconstruction-error summary and
  the federated alarm threshold of :mod:`fl.anomaly`;
* :data:`CATEGORY` (``"category"``, ``ffnn_category``): the rows' attack categories, with the record fields of
  :mod:`fl.category`.

:func:`of` finds a model's target, and the control plane makes one call to it wherever the targets differ.  The rules live
in the modules named above; the targets only pick among them.
"""
from __future__ import annotations

import logging
import os
from typing import Any, Dict, Optional, Sequence, Tuple

import torch

from ..data.datasets import CATEGORIES, BaseDataset, category_dataset, category_tensors
from ..data.synthetic import synthetic_for_model
from ..models import MODEL_REGISTRY
from ..ops.fused_mlp import NET_FFNN, net_kind_for
from . import anomaly, category, classweight, fedeval
from .evaluate import predict as classify

log = logging.getLogger(__name__)


class Target:
    """The dataset's labels (:data:`LABEL`); :data:`INPUT` and :data:`CATEGORY` override what differs for them"""

    def check_settings(self, args, box: bool = False, encryption: bool = False) -> None:
        """ValueError with the reason when the settings cannot train a model of this target"""
        classweight.setting(args, self.classes(args.model), box, encryption)

    def classes(self, model) -> Optional[int]:
        """How many classes a class-weighted fit of ``model`` (a built model, a model class or a registry name) weighs, None when
        it cannot be class-weighted: 2 (the 0 / 1 label) for the sigmoid FFNN, the one net of this target with class-weighted
        kernels"""
        if isinstance(model, str):
            model = MODEL_REGISTRY.get(model)
        spec = getattr(model, "spec", None)
        return 2 if spec is not None and net_kind_for(spec.dims, spec.out_activation) == NET_FFNN else None

    def dataset(self, ds):
        """The dataset the coordinator trains on, from the loaded CSV or synthetic dataset"""
        return ds

    def device_rows(self, model, key: str, x: torch.Tensor, y: torch.Tensor,
                    codes: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """``(x, labels)`` a device trains and scores ``model`` on, from its ``key`` rows and their attack categories ``codes``
        (None when it has none); ValueError with the reason when they cannot serve"""
        return x, y

    def training_rows(self, x: torch.Tensor, y: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """The rows a fit takes from a shard (``n_k`` counts them)"""
        return x, y

    def summarize(self, model, flat: torch.Tensor, x: torch.Tensor, y: torch.Tensor, bins: int, threshold: float,
                  segments: Optional[Sequence[int]] = None) -> list:
        return fedeval.summarize(model, flat, x, y, bins, threshold, segments)

    def to_wire(self, s) -> Dict[str, Any]:
        return fedeval.to_wire(s)

    def from_wire(self, reply: Dict[str, Any], classes: int, bins: int):
        return fedeval.from_wire(reply, classes, bins)

    def record(self, summaries: Dict[str, Any], args, excluded: Sequence[str] = (), missing: Sequence[str] = ()) -> Dict[str, Any]:
        """The ``fed_eval`` field of a round record"""
        return fedeval.record(summaries, excluded, missing)

    def checkpoint_meta(self, rec: Optional[Dict[str, Any]]) -> Dict[str, Any]:
        """What a checkpoint's JSON sidecar carries, from the last ``fed_eval`` record"""
        return {}

    def predict(self, model, flat: torch.Tensor, x: torch.Tensor, req: Dict[str, Any]) -> torch.Tensor:
        """A device's predictions for a ``predict`` request; ValueError with the reply's error for a refused one"""
        return classify(model, x, flat)

    def inference_alarm(self, path: str) -> Optional[Dict[str, Any]]:
        """What an INFERENCE request needs from the checkpoint at ``path``; ValueError with the reason the checkpoint cannot
        serve"""
        return None

    def log_predictions(self, pred) -> None:
        pass


class _Input(Target):
    def check_settings(self, args, box: bool = False, encryption: bool = False) -> None:
        anomaly.check_settings(args, box, encryption)
        super().check_settings(args, box, encryption)

    def classes(self, model) -> Optional[int]:
        return None                 # trained on its input: no classes

    def training_rows(self, x, y):
        return anomaly.training_rows(x, y)

    def summarize(self, model, flat, x, y, bins, threshold, segments=None):
        return anomaly.summarize(model, flat, x, y, bins, segments)

    def to_wire(self, s):
        return anomaly.to_wire(s)

    def from_wire(self, reply, classes, bins):
        return anomaly.from_wire(reply, bins)

    def record(self, summaries, args, excluded=(), missing=()):
        return anomaly.record(summaries, args.alarm_fpr, args.eval_bins, excluded, missing)

    def checkpoint_meta(self, rec):
        return {"anomaly": anomaly.checkpoint_meta(rec)}

    def predict(self, model, flat, x, req):
        # per-row alarms at the federated threshold the request carries ("alarm_bin" of "bins" error bins)
        j, bins = req.get("alarm_bin"), req.get("bins")
        if not isinstance(j, int) or not isinstance(bins, int) or isinstance(j, bool) or isinstance(bins, bool):
            raise ValueError(f"{req['model']} predicts alarms: the request needs an integer alarm_bin and bins")
        try:
            return anomaly.predict(model, flat, x, j, bins)
        except ValueError as e:
            raise ValueError(f"prediction refused: {e}") from None

    def inference_alarm(self, path):
        # the alarm threshold travels with the checkpoint (its JSON sidecar); without one an autoencoder flags nothing
        from ..utils.checkpoint import load_meta
        alarm = (load_meta(path).get("anomaly") or {}) if os.path.exists(path) else {}
        if alarm.get("alarm_bin") is None or alarm.get("bins") is None:
            raise ValueError(f"the autoencoder checkpoint at {path} has no alarm threshold (train it with --fed-eval-every)")
        return alarm


class _Category(Target):
    def check_settings(self, args, box: bool = False, encryption: bool = False) -> None:
        if box:
            raise ValueError(f"--model {args.model} does not run in box mode (--box): box mode trains on the binary attack label")
        if encryption:
            raise ValueError(f"--model {args.model} does not run with -e: the secret-shared training takes the binary attack label")
        super().check_settings(args, box, encryption)

    def classes(self, model) -> Optional[int]:
        return len(CATEGORIES)

    def dataset(self, ds):
        return BaseDataset(*category_tensors(ds))     # the rows' attack categories are the labels

    def device_rows(self, model, key, x, y, codes):
        if codes is None:
            raise ValueError(f"{model.__class__.__name__} trains on attack categories: this device's {key} data has none")
        return x, codes

    def record(self, summaries, args, excluded=(), missing=()):
        return category.record(summaries, excluded, missing)

    def checkpoint_meta(self, rec):
        return {"classes": list(CATEGORIES)}

    def log_predictions(self, pred) -> None:
        log.info("attack categories: %s", [CATEGORIES[i] if 0 <= i < len(CATEGORIES) else i for i in pred])


LABEL, INPUT, CATEGORY = Target(), _Input(), _Category()
_BY_NAME = {"input": INPUT, "category": CATEGORY}


def of(model) -> Target:
    """The target of a built model, a model class or a registry name: :data:`LABEL` for one without a ``spec`` (a conv net, a
    plugin factory, an unknown name) and for any ``target`` other than ``"input"`` and ``"category"``"""
    if isinstance(model, str):
        model = MODEL_REGISTRY.get(model)
    return _BY_NAME.get(getattr(getattr(model, "spec", None), "target", None), LABEL)


def synthetic_dataset(name: str, n: int, seed: int = 0):
    """``n`` rows of ``synthetic_for_model`` for the model ``name`` as a dataset shaped like the CSV adapter's: a category
    model's rows carry the binary attack label as targets and their class indices as ``categories``"""
    x, y = synthetic_for_model(name, n, seed=seed)
    return category_dataset(x, y) if of(name) is CATEGORY else BaseDataset(x, y)
