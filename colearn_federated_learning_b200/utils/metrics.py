"""Round metrics: structured JSONL + the reference's human-readable round log.

The reference's experiment logs (``data/*/coordinator/round_testing*.txt``) have the shape
``Testing round on: <max_batches>`` / ``Loss for worker id: <id> tensor(...)`` /
``Time round <r> : <sec>`` / ``Total training time: <sec>`` /
``Loss evaluation global model after training: <x>`` (SURVEY §2.7) — but the code that wrote
them is not in the reference tree (SURVEY §2.8-4).  :class:`RoundLogger` writes exactly that
format plus one JSON object per round for machines.
"""
from __future__ import annotations

import json
import logging
import os
import threading
import time
from typing import Any, Dict, List, Optional

log = logging.getLogger(__name__)


class PrometheusExporter:
    """Optional ``/metrics`` endpoint (``--metrics-port``): the round quantities of :class:`RoundLogger` as Prometheus
    series, for deployments that scrape instead of tailing log files (the reference's observability is the psutil /
    temperature scripts under ``data/`` attached by hand to the PID it logs at start-up, SURVEY §5)."""

    def __init__(self, port: int, addr: str = "127.0.0.1") -> None:
        from prometheus_client import CollectorRegistry, Counter, Gauge, Histogram, start_http_server

        self.registry = CollectorRegistry()
        mk = dict(registry=self.registry)
        self.trainings = Counter("colearn_trainings_total", "training windows that ran to completion", **mk)
        self.rounds = Counter("colearn_rounds_total", "federated rounds completed", **mk)
        self.round_seconds = Histogram("colearn_round_seconds", "wall time of one federated round",
                                       buckets=(1e-3, 3e-3, 1e-2, 3e-2, 0.1, 0.3, 1, 3, 10, 30, 100), **mk)
        self.bytes_out = Counter("colearn_bytes_to_workers_total", "application bytes shipped to the devices (model + fit config)", **mk)
        self.bytes_in = Counter("colearn_bytes_from_workers_total", "application bytes received from the devices (trained model + loss)", **mk)
        self.selected = Gauge("colearn_round_selected_workers", "devices that contributed to the last round", **mk)
        self.worker_loss = Gauge("colearn_worker_last_loss", "last local loss reported by a device", ["worker"], **mk)
        self.training_seconds = Gauge("colearn_last_training_seconds", "total time of the last training", **mk)
        # federated evaluation (--fed-eval-every): the total over the devices of the last evaluated round
        self.eval_loss = Gauge("colearn_eval_loss", "federated evaluation: mean loss of the global model on the devices' held-out rows", **mk)
        self.eval_accuracy = Gauge("colearn_eval_accuracy", "federated evaluation: accuracy of the global model", **mk)
        self.eval_auc = Gauge("colearn_eval_auc", "federated evaluation: ROC-AUC (macro one-vs-rest for multi-class models)", **mk)
        self.eval_f1 = Gauge("colearn_eval_f1", "federated evaluation: F1 (macro for multi-class models)", **mk)
        self.server, self.thread = start_http_server(port, addr=addr, registry=self.registry)
        self.port = self.server.server_port

    def close(self) -> None:
        self.server.shutdown()
        self.server.server_close()


class RoundLogger:
    def __init__(self, jsonl_path: Optional[str] = None, text_path: Optional[str] = None,
                 exporter: Optional[PrometheusExporter] = None) -> None:
        self.jsonl_path, self.text_path = jsonl_path, text_path
        self.exporter = exporter
        self._lock = threading.Lock()
        self.records: List[Dict[str, Any]] = []
        self._t_start: Optional[float] = None
        for p in (jsonl_path, text_path):
            if p:
                os.makedirs(os.path.dirname(os.path.abspath(p)), exist_ok=True)

    def _text(self, line: str) -> None:
        log.info(line)
        if self.text_path:
            with open(self.text_path, "a") as f:
                f.write(line + "\n")

    def start_training(self, max_batches: int) -> None:
        self._t_start = time.time()
        self._text(f"Testing round on: {max_batches}")

    def worker_loss(self, worker_id: str, loss: float) -> None:
        self._text(f"Loss for worker id: {worker_id} tensor({loss:.4f}, requires_grad=True)")
        if self.exporter is not None:
            self.exporter.worker_loss.labels(worker=str(worker_id)).set(float(loss))

    def end_round(self, round_idx: int, seconds: float, **fields: Any) -> Dict[str, Any]:
        self._text(f"Time round {round_idx} : {seconds}")
        fed_eval = fields.get("fed_eval")
        if fed_eval is not None:
            from ..fl.fedeval import summary_line
            total = fed_eval.get("total") or {}
            self._text(f"Federated evaluation round {round_idx}: {summary_line(total)}")
            if self.exporter is not None:
                for gauge, key in ((self.exporter.eval_loss, "loss"), (self.exporter.eval_accuracy, "accuracy"),
                                   (self.exporter.eval_auc, "auc"), (self.exporter.eval_f1, "f1")):
                    if total.get(key) is not None:
                        gauge.set(float(total[key]))
        rec = {"round": round_idx, "t_round_s": seconds, "ts": time.time(), **fields}
        if self.exporter is not None:
            self.exporter.rounds.inc()
            self.exporter.round_seconds.observe(float(seconds))
            self.exporter.bytes_out.inc(float(fields.get("bytes_out", 0) or 0))
            self.exporter.bytes_in.inc(float(fields.get("bytes_in", 0) or 0))
            if "selected" in fields and fields["selected"] is not None:
                self.exporter.selected.set(len(fields["selected"]))
        with self._lock:
            self.records.append(rec)
            if self.jsonl_path:
                with open(self.jsonl_path, "a") as f:
                    f.write(json.dumps(rec, default=float) + "\n")
        return rec

    def end_training(self, eval_loss: Optional[float] = None) -> float:
        total = time.time() - (self._t_start or time.time())
        self._text(f"Total training time: {total}")
        if self.exporter is not None:
            self.exporter.trainings.inc()
            self.exporter.training_seconds.set(total)
        if eval_loss is not None:
            self._text(f"Loss evaluation global model after training: {eval_loss}")
        return total
