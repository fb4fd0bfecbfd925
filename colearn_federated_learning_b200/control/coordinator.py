"""The Coordinator: pub/sub subscriber + temporal-window scheduler + round loops.

Parity map (reference ``federated_coordinator.py``):
  ``Coordinator.__init__``  :93-124   bounds 1/2/100/2, ``./test.pth``, ``Arguments()``
  ``on_connect/on_publish`` :128-129, :291-292
  ``on_message``            :131-289  parse → worker handle → TRAINING / INFERENCE / NOT_READY
  ``run``                   :294-313  connect, subscribe qos 0, loop_forever, Ctrl-C cleanup
  ``starting_training_local`` :318-392, ``starting_training_enc`` :394-472,
  ``training_remote``       :475-597

Differences that are deliberate (SURVEY §2.8): the registry is locked; local mode is *true*
FedAvg (every worker starts the round from the same global θ) instead of averaging K aliases of
one module; INFERENCE uses the trained architecture; encrypted mode saves its model; Ctrl-C never
``KeyError``s; a failing/slow remote worker is dropped from the round instead of hanging it
(``fit_timeout``); selection at the upper bound is implemented, not just logged.
"""
from __future__ import annotations

import asyncio
import logging
import os
import secrets
import time
import zlib
from collections import OrderedDict
from functools import partial
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from .. import ops, settings
from ..data import federate, synthetic_for_model, BaseDataset
from ..fl.fedavg import normalized_weights
from ..fl.trainer import FitConfig, local_fit, make_perm, resolve_loss
from ..fl import anomaly, asyncagg, category, fedeval, uplink
from ..fl.evaluate import evaluate
from ..fl.secagg import check_masked_reply, check_unmask_reply, correction_streams, frac_bits, pk_from_bytes, pk_to_bytes
from ..fl.server_opt import server_opt_state
# the reply checks live next to the codec (the workers run them on the downlink wire too) and are exported from here as before
from ..fl.uplink import UplinkCodec, check_quantized_reply, check_topk_reply, downlink_key, uplink_key  # noqa: F401
from ..models import MODEL_REGISTRY, MLPNet, build_model, flatten_params, unflatten_params
from ..utils.checkpoint import DEFAULT_PATH, checkpoint_compatible, load_or_init, save_model
from ..utils.metrics import RoundLogger
from .arguments import Arguments, ROUND_MODE_BATCHES
from .bus import BusClient, InProcessBroker, Message
from .event_parser import EventParser
from .selection import (LOWER_BOUND, LOWER_BOUND_ENC, UPPER_BOUND, UPPER_BOUND_ENC, SelectionPolicy)
from .window import TemporalWindow
from .workers import RemoteWorkerClient, VirtualWorker, replica_crc

log = logging.getLogger(__name__)


def default_device() -> torch.device:
    return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def traffic(handle) -> tuple:
    """(bytes sent, bytes received) so far over a device handle (0 for handles that do not count)"""
    return getattr(handle, "bytes_sent", 0), getattr(handle, "bytes_received", 0)


class Coordinator(BusClient):
    def __init__(self, window: float, remote: bool, federated_round: int, encryption: bool,
                 iot_validation: bool, args: Optional[Arguments] = None, broker: Optional[InProcessBroker] = None,
                 transport: str = "inproc", timer_factory=None, path: str = DEFAULT_PATH,
                 strict_events: bool = False, device: Optional[torch.device] = None,
                 select_k: Optional[int] = None, selection: str = "all", fit_timeout: Optional[float] = None,
                 filter_file: Optional[str] = None, metrics: Optional[RoundLogger] = None,
                 rearm_if_pending: bool = False, evaluate_after: bool = False, worker_ssl_context=None) -> None:
        super().__init__(client_id="coordinator", broker=broker, transport=transport)
        self.worker_ssl_context = worker_ssl_context     # TLS towards the devices' RPC servers (control/tls.py)
        self.registry = settings.init()

        # Command parameters (fc.py:105-109)
        self.window = window
        self.remote = remote
        self.enabled_round = max(1, int(federated_round))
        self.encryption = encryption
        self.iot_validation = iot_validation

        # Other useful parameters (fc.py:112-124)
        kwargs = {"filter_file": filter_file} if filter_file else {}
        self.event_parser = EventParser(self.iot_validation, strict=strict_events, **kwargs)
        self.training_lower_bound = LOWER_BOUND
        self.training_lower_bound_enc = LOWER_BOUND_ENC
        self.training_upper_bound = UPPER_BOUND
        self.training_upper_bound_enc = UPPER_BOUND_ENC
        self.known_workers: Dict[str, Any] = {}   # the reference's ``server._known_workers``
        self.path = path
        self.args = args or Arguments()
        self.device = device or (torch.device("cpu") if self.args.no_cuda else default_device())
        self.select_k = select_k
        self.selection = selection
        self.fit_timeout = fit_timeout
        self.metrics = metrics or RoundLogger()
        self.evaluate_after = evaluate_after
        self.last_predictions: Optional[List[int]] = None
        self.trainings_done = 0
        self._in_flight: Dict[str, Any] = {}      # id -> handle of the devices a running training is using
        self._withdrawn: set = set()              # ids that sent NOT_READY while their fit was in flight
        # server optimizer moments (--server-opt other than sgd): carried from round to round and from window to window for the
        # Coordinator's lifetime, reset when the model's parameter count changes; never written to the checkpoint
        self._server_opt_state = None

        self.windower = TemporalWindow(self.registry, window, self._start_training, timer_factory,
                                       lower_bound=0, rearm_if_pending=rearm_if_pending)

    # ------------------------------------------------------------------ paho-style callbacks
    def on_connect(self, mqttc, obj, flags, rc) -> None:
        log.info("Connected!")

    def on_publish(self, mqttc, obj, mid) -> None:
        log.info("mid: " + str(mid))

    def on_message(self, mqttc, obj, msg: Message) -> None:
        """One bus event (fc.py:131-289): decode it, build the device handle its state needs, run the state's handler
        from ``_STATE_HANDLERS``.  Malformed payloads, filtered addresses and unknown states end in one log line."""
        log.info("%s %s %s", msg.topic, msg.qos, msg.payload)
        event = self._decode_event(msg.payload)
        if event is None:
            log.info("Event ignored: payload is not a valid '(ip[, port], STATE)' tuple for this mode")
            return
        handler = self._STATE_HANDLERS[event["state"]]
        handle = None
        if event["state"] != "NOT_READY":
            handle = self._open_handle(event)
            if handle is None:
                return
        getattr(self, handler)(event, handle)
        log.info("ONMESSAGE: Training devices: " + str(self.registry))
        log.info("ONMESSAGE: All known workers: " + str(list(self.known_workers)))

    _STATE_HANDLERS = {"TRAINING": "_on_training", "INFERENCE": "_on_inference", "NOT_READY": "_on_not_ready"}

    def _decode_event(self, payload) -> Optional[Dict[str, Any]]:
        """``{ip, port, state, id}`` of a payload, or None.  Local events are ``(ip, STATE)``, remote ones
        ``(ip, port, STATE)``; the device id is ``ip`` / ``ip:port`` (fc.py:149,162)."""
        ev = self.event_parser.parse(payload, remote=self.remote)
        if ev is None:
            return None
        ident = f"{ev.ip}:{ev.port}" if self.remote else ev.ip
        return {"ip": ev.ip, "port": ev.port, "state": ev.state, "id": ident}

    def _open_handle(self, event: Dict[str, Any]):
        """The object a TRAINING / INFERENCE event registers: an in-process VirtualWorker, or a connection to the
        device's RPC server.  A device that cannot be reached is skipped (fc.py:166-170)."""
        if not self.remote:
            log.info("Local testing")
            return VirtualWorker(event["id"], self.device)
        log.info("Remote execution, worker id %s", event["id"])
        try:
            return RemoteWorkerClient(event["id"], event["ip"], event["port"], verbose=True, ssl_context=self.worker_ssl_context)
        except OSError as e:
            log.info("Device %s unreachable, skipped: %r", event["id"], e)
            return None

    def _on_training(self, event: Dict[str, Any], worker) -> None:
        # a device that announces twice (duplicate delivery, reconnect) replaces its handle; the old connection is closed
        # unless a training in flight is still using it (that one closes it itself)
        old = self.known_workers.get(worker.id)
        if old is not None and old is not worker and worker.id not in self._in_flight:
            self._close_quietly(old)
        self.known_workers[worker.id] = worker
        armed = self.windower.on_training(worker.id, worker)
        log.info(worker)
        if armed:
            log.info("Timer starting")

    def _on_inference(self, event: Dict[str, Any], worker) -> None:
        if self.remote:
            self._inference(worker)
        else:
            log.info("Inference is a remote-mode feature (local mode only tests the plumbing)")

    def _on_not_ready(self, event: Dict[str, Any], _worker) -> None:
        ident = event["id"]
        log.info("%s withdrew (NOT_READY): removing it from the known lists", ident)
        removed = self.windower.on_not_ready(ident)
        if removed is not None:
            if self._in_flight.get(ident) is removed:
                # its fit RPC is running and holds the connection's lock: closing here would block the bus thread until the
                # fit returns (forever for a hung device).  The training that uses the handle closes it when it finishes.
                self._withdrawn.add(ident)
                log.info("Worker %s is training right now; its connection is closed by that training", ident)
            else:
                self._close_quietly(removed)
        self.known_workers.pop(ident, None)

    @staticmethod
    def _close_quietly(handle) -> None:
        try:
            handle.close()
        except Exception:  # noqa: BLE001 - a dead socket must not take the bus thread down
            pass

    # ------------------------------------------------------------------ lifecycle
    def run(self, host: str, port: int, topic: str, forever: bool = True) -> None:
        self.connect(host, port)
        self.subscribe(topic, 0)
        log.info("Coordinator started. Press CTRL-C to stop")
        if not forever:
            self.loop_start()
            return
        try:
            self.loop_forever()
        except KeyboardInterrupt:
            self.shutdown()

    def shutdown(self) -> None:
        log.info("Coordinator stopped.")
        if self.windower.cancel():
            log.info("Cancelling the timer..")
        for key, worker in list(self.known_workers.items()):
            log.info("Closing socket for worker " + str(worker))
            try:
                worker.close()
            except Exception:  # noqa: BLE001
                pass
        self.loop_stop()
        log.info("Done")

    # ------------------------------------------------------------------ training dispatch
    def _start_training(self, snapshot: "OrderedDict[str, Any]") -> Any:
        from ..models.registry import num_params
        from ..utils.threads import small_model_threads
        self._in_flight = dict(snapshot)
        sizes = self.__dict__.setdefault("_param_counts", {})
        if self.args.model not in sizes:
            try:
                sizes[self.args.model] = num_params(build_model(self.args.model))
            except Exception:  # noqa: BLE001 - an unknown model fails later, with the proper message
                sizes[self.args.model] = 0
        try:
            # small models on the CPU: one intra-op thread (utils/threads.py: OpenMP fork/join costs more than the ops)
            with small_model_threads(sizes[self.args.model], self.device):
                return self._dispatch_training(snapshot)
        finally:
            self._in_flight = {}

    def _dispatch_training(self, snapshot: "OrderedDict[str, Any]") -> Any:
        if self.remote:
            loop = asyncio.new_event_loop()  # fresh loop inside the timer thread (fc.py:194-203)
            try:
                return loop.run_until_complete(self.training_remote(snapshot))
            finally:
                loop.close()
        if self.encryption:
            return self.starting_training_enc(snapshot)
        return self.starting_training_local(snapshot)

    def _policy(self, lower: int, upper: int, policy: Optional[str] = None) -> SelectionPolicy:
        return SelectionPolicy(lower_bound=lower, upper_bound=upper, policy=policy or self.selection,
                               select_k=self.select_k, seed=self.args.seed)

    def _load_model(self, name: Optional[str] = None):
        model = build_model(name or self.args.model)
        log.info("Loading model procedure started...")
        if os.path.exists(self.path) and not checkpoint_compatible(model, self.path):
            log.info("Checkpoint at %s does not match model %s; starting from a fresh model", self.path, name or self.args.model)
        else:
            load_or_init(model, self.path)
        log.info("Done")
        return model

    def _dataset(self):
        if self.args.synthetic and self.args.synthetic > 0:
            x, y = synthetic_for_model(self.args.model, self.args.synthetic, seed=self.args.seed)
            return BaseDataset(x, y)
        from ..data import load_dataset
        ds = load_dataset(getattr(self.args, "dataset", "unsw"), self.args.test_path)
        if category.is_category(MODEL_REGISTRY.get(self.args.model)):
            return BaseDataset(*category.labels(ds))     # the rows' attack categories are the labels
        return ds

    def _fit_config(self, mode: str) -> FitConfig:
        loss = self.args.loss
        if loss in ("auto", "", None):
            # reference: local mode trains with sum-squared-error (cf.py:112), remote with BCE (cf.py:79)
            loss = "sse" if (mode == "local" and self.args.model in ("ffnn", "testing_remote")) else resolve_loss(self.args.model, "auto")
        return FitConfig(model=self.args.model, loss=loss, batch_size=self.args.batch_size, epochs=self.args.epochs,
                         max_nr_batches=self.args.federate_after_n_batches, lr=self.args.lr, shuffle=True,
                         seed=self.args.seed)

    def _maybe_checkpoint(self, model, theta: torch.Tensor, round_idx: int, meta: Dict[str, Any]) -> None:
        """``--save-every N``: durable progress inside a long training (the reference only saves after the last
        round, fc.py:381,585).  Atomic like every checkpoint write; the final save still happens."""
        n = getattr(self.args, "save_every", 0)
        if n and (round_idx + 1) % n == 0 and round_idx + 1 < self.enabled_round:
            from ..models import state_dict_from_flat
            from ..utils.checkpoint import save_state_dict
            save_state_dict(state_dict_from_flat(model, theta), self.path, meta={**meta, "model": self.args.model, "rounds": round_idx + 1, "partial": True})
            log.info("checkpoint after round %d written to %s", round_idx + 1, self.path)

    def _deregister(self, trained) -> None:
        """Forget the devices that just trained (fc.py:376-379, 571-577) — unless the device re-announced itself
        while its training was running: that newer registration is a late joiner and rides the next window."""
        for wid in trained:
            used = self._in_flight.get(wid)
            current = self.registry.get(wid)
            if used is not None and current is not None and current is not used:
                log.info("Keeping " + str(wid) + ": it registered again during the training")
                continue
            log.info("Removing: " + str(wid) + " from training devices")
            self.registry.remove(wid)
            self.known_workers.pop(wid, None)

    # ------------------------------------------------------------------ local (VirtualWorker) mode
    def starting_training_local(self, snapshot: "OrderedDict[str, Any]") -> Optional[Dict[str, Any]]:
        to_train = self._policy(self.training_lower_bound, self.training_upper_bound).select(snapshot)
        if not to_train:
            log.info("No behaviour defined for the number of devices achieved")
            return None
        if self.args.async_buffer:
            raise ValueError("--async-buffer applies to remote mode only: local mode trains its virtual workers in lockstep launches")
        model = self._load_model()
        cfg = self._fit_config("local")
        ae = anomaly.is_autoencoder(model)
        if ae:
            anomaly.check_settings(self.args)

        log.info("Distribution data among the virtual workers")
        fed = federate(self._dataset(), list(to_train.keys()), self.device)
        log.info("Done")
        held = self._hold_out_local(model, fed, cfg.seed)
        if ae:
            from ..data.federate import Shard
            for wid in fed.workers:
                fed.shards[wid] = Shard(wid, *anomaly.training_rows(fed[wid].x, fed[wid].y))

        theta = flatten_params(model).to(self.device)
        model.to(self.device)
        log.info("Start training")
        self.metrics.start_training(cfg.max_nr_batches)
        result: Dict[str, Any] = {"workers": list(to_train.keys()), "losses": {}, "rounds": self.enabled_round}
        codec = self.args.uplink_codec()
        result["uplink"] = codec.kind
        # topk: every device's error-feedback residual, zero at the start of the training (memory only, not checkpointed)
        residual = torch.zeros(len(fed.workers), theta.numel(), device=self.device) if codec.sparse else None
        # compressed downlink: the workers train from the replica (theta at round 0, then advanced by one encode per round)
        # and their deltas are taken against it; theta stays the true global model
        down = self.args.downlink_codec()
        result["downlink"] = down.kind
        replica = theta.clone() if down.kind != "fp32" else theta
        for r in range(self.enabled_round):
            t0 = time.time()
            if r > 0 and down.kind != "fp32":
                ops.encode_downlink(theta, replica, down, downlink_key(cfg.seed + r))
            flats, losses, counts = train_virtual_workers(replica, model, fed, cfg, r)
            live = [i for i, c in enumerate(counts) if c > 0]
            agg_w = None
            if live:
                w = normalized_weights([counts[i] for i in live] if self.args.weighted else None, len(live), device=self.device)
                # every live worker's update through the uplink codec (one batched encode), as a device would send it; topk: a
                # worker that did not train this round keeps its residual
                res = residual if residual is None or len(live) == len(fed.workers) else residual[live]
                wire = uplink.encode(codec, flats[live], replica, [uplink_key(fed.workers[i], cfg.seed + r) for i in live], res)
                if res is not residual:
                    residual[live] = res
                agg_w = self._server_update(theta, partial(uplink.server_apply, theta, wire, w, codec), len(live))
            for wid, l in zip(fed.workers, losses):
                self.metrics.worker_loss(wid, l)
                result["losses"][wid] = l
            rec = {}
            if agg_w is not None:
                # distance-based aggregator: the final weight of every worker in the order of `selected` (0: excluded or not trained)
                rec["agg_weights"] = [0.0] * len(fed.workers)
                for j, i in enumerate(live):
                    rec["agg_weights"][i] = agg_w[j]
            if held is not None and self._fed_eval_round(r):
                ex, ey, sizes = held
                if ae:
                    rec["fed_eval"] = result["fed_eval"] = anomaly.record(
                        dict(zip(fed.workers, anomaly.summarize(model, theta, ex, ey, self.args.eval_bins, sizes))), self.args.alarm_fpr,
                        self.args.eval_bins)
                else:
                    make = category.record if category.is_category(model) else fedeval.record
                    rec["fed_eval"] = result["fed_eval"] = make(
                        dict(zip(fed.workers, fedeval.summarize(model, theta, ex, ey, self.args.eval_bins, self.args.eval_threshold, sizes))))
            self.metrics.end_round(r, time.time() - t0, selected=fed.workers, n_k=counts, loss_k=losses, **rec)
            self._maybe_checkpoint(model, theta, r, {"workers": fed.workers, "mode": "local", **self._model_meta(model, result)})
        log.info("End training")
        unflatten_params(model, theta)
        save_model(model.cpu(), self.path, meta={"model": self.args.model, "rounds": self.enabled_round, "workers": fed.workers, "mode": "local",
                                                 **self._model_meta(model, result)})
        self._deregister(to_train.keys())
        self.metrics.end_training()
        self.trainings_done += 1
        log.info("End training local")
        return result

    @staticmethod
    def _model_meta(model, result: Dict[str, Any]) -> Dict[str, Any]:
        """An autoencoder's checkpoint sidecar carries the alarm threshold of its last federated evaluation, a category
        model's the names of its classes"""
        if anomaly.is_autoencoder(model):
            return {"anomaly": anomaly.checkpoint_meta(result.get("fed_eval"))}
        return {"classes": list(category.CATEGORIES)} if category.is_category(model) else {}

    def _fed_eval_round(self, r: int) -> bool:
        """``--fed-eval-every N``: the global model is evaluated after every N-th round and after the last one"""
        n = self.args.fed_eval_every
        return n > 0 and ((r + 1) % n == 0 or r + 1 == self.enabled_round)

    def _hold_out_local(self, model, fed, seed: int):
        """``--fed-eval-every`` in local mode: every virtual worker's shard loses its ``--eval-fraction`` held-out rows
        (``fedeval.split_eval``, keyed by the worker's position); returns ``(x, y, rows per worker)`` of the held-out rows
        in worker order, or None without federated evaluation (the shards are left as they are)."""
        if self.args.fed_eval_every <= 0:
            return None
        self.args.fed_eval_settings()
        fedeval.check_model(model)
        if not self.args.eval_fraction > 0:
            raise ValueError("--fed-eval-every in local mode needs --eval-fraction > 0")
        from ..data.federate import Shard
        xs, ys, sizes = [], [], []
        for i, wid in enumerate(fed.workers):
            sh = fed[wid]
            xt, yt, xe, ye = fedeval.split_eval(sh.x, sh.y, self.args.eval_fraction, seed + i)
            fed.shards[wid] = Shard(wid, xt, yt)
            xs.append(xe)
            ys.append(ye)
            sizes.append(int(xe.shape[0]))
        return torch.cat(xs), torch.cat(ys), sizes

    # ------------------------------------------------------------------ encrypted (SMPC) mode
    def starting_training_enc(self, snapshot: "OrderedDict[str, Any]") -> Optional[Dict[str, Any]]:
        from ..fl.encrypted import train_encrypted

        to_train = self._policy(self.training_lower_bound_enc, self.training_upper_bound_enc, "first").select(snapshot)
        if not to_train:
            log.info("No behaviour defined for a number of workers less than " + str(self.training_lower_bound_enc))
            return None
        model = self._load_model()
        log.info("Distribute the data among the virtual workers...")
        result = train_encrypted(model, self._dataset(), list(to_train.keys()), self.args)
        save_model(model, self.path, meta={"model": self.args.model, "mode": "encrypted", "workers": list(to_train.keys())})
        self._deregister(to_train.keys())
        self.trainings_done += 1
        log.info("End encryption")
        return result

    # ------------------------------------------------------------------ remote mode
    async def training_remote(self, snapshot: "OrderedDict[str, Any]") -> Optional[Dict[str, Any]]:
        to_train = self._policy(self.training_lower_bound, self.training_upper_bound).select(snapshot)
        if not to_train:
            log.info("No behaviour defined for the number of devices achieved")
            return None
        model = self._load_model()
        if self.enabled_round > 1 and self.args.federate_after_n_batches < 0:
            log.info("Round activated!")
            self.args.set_federated_batches(ROUND_MODE_BATCHES)  # fc.py:533-535
        log.info("Federated batches: " + str(self.args.federate_after_n_batches))
        cfg = self._fit_config("remote")
        if self.args.fed_eval_every > 0:
            self.args.fed_eval_settings()
        if anomaly.is_autoencoder(model):
            anomaly.check_settings(self.args)
        theta = flatten_params(model).cpu()
        loop = asyncio.get_running_loop()
        # one thread per selected device: every fit RPC of a round is in flight at the same time (the default
        # executor would cap the fan-out at min(32, cpu_count + 4) and serialise a 100-device round)
        from concurrent.futures import ThreadPoolExecutor
        pool = ThreadPoolExecutor(max_workers=max(1, len(to_train)), thread_name_prefix="fit-rpc")
        self.metrics.start_training(cfg.max_nr_batches)
        result: Dict[str, Any] = {"workers": list(to_train.keys()), "losses": {}, "rounds": self.enabled_round, "dropped": []}
        alive = OrderedDict(to_train)
        run = self._remote_async if self.args.async_settings() is not None else self._remote_rounds
        try:
            theta = await run(alive, to_train, theta, cfg, loop, pool, model, result)
        finally:
            # whatever happened above, the devices' sockets are closed and they leave the registry (fc.py:573-580, 595-597)
            pool.shutdown(wait=False)
            for wid, worker in to_train.items():
                log.info("Closing socket for " + str(wid))
                self._close_quietly(worker)
            self._withdrawn.difference_update(to_train.keys())
            self._deregister(to_train.keys())
        unflatten_params(model, theta)
        save_model(model, self.path, meta={"model": self.args.model, "rounds": self.enabled_round, "workers": list(to_train.keys()), "mode": "remote",
                                           **self._model_meta(model, result)})
        eval_loss = None
        if self.evaluate_after:
            ds = self._dataset()
            from ..data import dataset_tensors
            x, y = dataset_tensors(ds, self.device)
            eval_loss = evaluate(model.to(self.device), x, y, verbose=False)["loss"]
            result["eval_loss"] = eval_loss
        self.metrics.end_training(eval_loss)
        self.trainings_done += 1
        return result

    async def _fit(self, loop, pool, wid: str, worker, flat: torch.Tensor, rcfg: FitConfig, codec: UplinkCodec, *, ef_reset: bool = False,
                   secagg: Optional[Dict[str, Any]] = None, downlink: Optional[Dict[str, Any]] = None, version: Optional[int] = None,
                   crc: Optional[int] = None):
        """One device's fit RPC, run in ``pool`` (the fields as in :meth:`RemoteWorkerClient.fit_update`): ``(checked update,
        loss, n)``, or ``(None, None, 0)`` when the RPC failed or the reply failed the checks of its format, or did not echo
        the replica crc ``crc``.  A device's reply is untrusted input: a malformed update would poison (or abort) the whole
        average, so such a device counts as failed."""
        try:
            if codec.kind == "fp32" and secagg is None:
                # the fp32 model (never with a compressed downlink): `fit` is every handle's verb for it
                kw = {} if version is None else {"version": version}
                got, loss, n = await loop.run_in_executor(pool, lambda: worker.fit(flat, rcfg, timeout=self.fit_timeout, **kw))
                update = {"params": got}
            else:
                update, loss, n = await loop.run_in_executor(pool, lambda: worker.fit_update(
                    flat, rcfg, codec, ef_reset=ef_reset, secagg=secagg, downlink=downlink, version=version, timeout=self.fit_timeout))
            if crc is not None and update.get("replica_crc") != crc:
                raise ValueError(f"replica crc {update.get('replica_crc')!r} returned, the coordinator's is {crc}")
            if secagg is not None:
                return check_masked_reply(update, flat.numel()), loss, n
            return uplink.check_reply(update, codec, flat.numel()), loss, n
        except Exception as e:  # noqa: BLE001 - a failing device must not sink the round or the training
            log.info("Worker %s failed its fit: %r", wid, e)
            return None, None, 0

    async def _remote_rounds(self, alive, to_train, theta, cfg, loop, pool, model, result) -> torch.Tensor:
        """The round loop of ``training_remote`` (fc.py:540-568): fan the fit RPC out to every live device, FedAvg what came
        back, repeat.  Returns the final global parameters.  With a quantized ``--uplink-codec`` the devices send their deltas
        (fl/uplink.py), each reply is checked by :func:`check_quantized_reply` and the decode runs inside the FedAvg kernel;
        with ``topk`` they send sparse deltas with error feedback (the first round resets their residuals), checked by
        :func:`check_topk_reply`.  With a compressed ``--downlink-codec`` the rounds after the first send the devices a wire
        to the replica they keep instead of the model (:meth:`_downlink_fields`), and a device whose replica's crc differs
        from the coordinator's is dropped."""
        codec = self.args.uplink_codec()
        down = self.args.downlink_codec()
        result["uplink"], result["downlink"] = codec.kind, down.kind
        eval_classes = fedeval.check_model(model) if self.args.fed_eval_every > 0 else None
        # the replica of the model the devices hold, tagged "<nonce>:<round>" (a fresh nonce per training: a device cannot
        # mistake an earlier training's replica for this one's); memory only
        replica = theta.to(self.device).clone() if down.kind != "fp32" else None
        nonce = secrets.token_hex(8)
        sa = None
        if self.args.secure_agg:
            # secure aggregation (fl/secagg.py): key agreement once per training, tagged with its nonce; fewer than two
            # devices left after it cannot hide one update in a sum
            sa = await self._secagg_setup(alive, nonce, loop, pool, result)
            if sa is None:
                return theta
        for r in range(self.enabled_round):
            log.info("\n\n#### ROUND {} #####".format(r))
            t0 = time.time()
            rcfg = cfg.with_seed(cfg.seed + r)
            downlink = self._downlink_fields(down, theta, replica, nonce, r, rcfg.seed) if replica is not None else None
            crc = replica_crc(replica) if replica is not None else None
            u1 = list(alive)                                          # secure aggregation: this round's participants
            fields = None if sa is None else {"tag": sa["tag"], "t": r, "u1": u1, "clip": sa["clip"], "frac_bits": sa["frac_bits"]}
            sent0 = {wid: traffic(w) for wid, w in alive.items()}
            results = await asyncio.gather(*[self._fit(loop, pool, wid, w, theta, rcfg, codec, ef_reset=r == 0, secagg=fields,
                                                       downlink=downlink, crc=crc) for wid, w in alive.items()])
            flats, counts, ids = [], [], []
            for wid, (flat, loss, n) in zip(u1, results):
                if flat is not None:
                    flats.append(flat)
                    counts.append(n)
                    ids.append(wid)
                    self.metrics.worker_loss(wid, loss)
                    result["losses"][wid] = loss
                else:
                    result["dropped"].append(wid)
                    alive.pop(wid, None)
            secagg_rec = {}
            agg_rec = {}
            if sa is not None:
                theta, secagg_rec = await self._secagg_round(theta, r, u1, ids, flats, alive, sa, loop, pool, result)
            elif flats:
                w = normalized_weights(counts if self.args.weighted else None, len(flats), device=self.device)
                th = theta.to(self.device)
                wire = uplink.stack(flats, codec, self.device)
                agg_w = self._server_update(th, partial(uplink.server_apply, th, wire, w, codec), len(flats))
                if agg_w is not None:
                    agg_rec["agg_weights"] = agg_w       # the final weight of every device in `ids` (distance-based aggregator)
                theta = th.cpu()
                self._average_buffers(model, [getattr(alive.get(wid), "last_buffers", None) for wid in ids], w.cpu())
            # traffic of this round: model + fit config towards the devices, trained model + loss back (paper §4.3), and the
            # unmask exchange of secure aggregation
            bytes_out = sum(traffic(w)[0] - sent0[wid][0] for wid, w in to_train.items() if wid in sent0)
            bytes_in = sum(traffic(w)[1] - sent0[wid][1] for wid, w in to_train.items() if wid in sent0)
            if self._fed_eval_round(r):
                agg_rec["fed_eval"] = result["fed_eval"] = await self._remote_fed_eval(alive, theta, eval_classes, loop, pool, ae=anomaly.is_autoencoder(model))
            self.metrics.end_round(r, time.time() - t0, selected=ids, n_k=counts, bytes_out=bytes_out, bytes_in=bytes_in, **secagg_rec,
                                   **agg_rec)
            result["bytes_out"] = result.get("bytes_out", 0) + bytes_out
            result["bytes_in"] = result.get("bytes_in", 0) + bytes_in
            self._maybe_checkpoint(model, theta, r, {"workers": list(to_train.keys()), "mode": "remote", **self._model_meta(model, result)})
            if not alive:
                break
        return theta

    async def _remote_async(self, alive, to_train, theta, cfg, loop, pool, model, result) -> torch.Tensor:
        """Asynchronous buffered aggregation (``--async-buffer K``, :mod:`fl.asyncagg`): up to ``C`` fits in flight, each from
        the global version current when it was sent; a freed device gets the current theta at once, every reply passes the
        reply checks of its uplink codec and goes into the buffer (a failing device is dropped as in :meth:`_remote_rounds`),
        and every ``K`` buffered replies make one server step (``-f`` of them).  fp32 replies are applied as deltas to their
        base through the version ring (``ops.fedavg_apply_based``), codec replies are deltas already and keep their apply with
        the staleness-scaled weights.  A ``--fed-eval-every`` step stops dispatching, drains the fits in flight into the buffer
        and evaluates theta before it resumes.  After the last step nothing is dispatched and the fits still in flight are
        awaited (up to ``fit_timeout``) and discarded."""
        st = self.args.async_settings()
        codec = self.args.uplink_codec()
        result["uplink"], result["downlink"] = codec.kind, "fp32"
        if any(b.is_floating_point() for b in model.buffers()):
            raise ValueError(f"--async-buffer does not apply to {self.args.model}: averaging BatchNorm statistics across model versions "
                             "is not defined")
        eval_classes = fedeval.check_model(model) if self.args.fed_eval_every > 0 else None
        th = theta.to(self.device).clone()
        ring = asyncagg.ring_init(th, st) if codec.kind == "fp32" else None
        # what a fit request sends: a snapshot of theta at `version`.  A request is serialised later, in the executor thread, and
        # the steps update th in place (th.cpu() is th itself on a CPU coordinator), so every version gets its own copy
        current = th.detach().to("cpu", copy=True)
        version, steps, dispatched = 0, 0, 0
        buffer: List[asyncagg.Reply] = []
        in_flight: Dict[Any, Any] = {}                             # task -> (device, base version)
        idle = list(alive)
        fitted: set = set()                                        # top-k: a device's first fit resets its residual
        concurrency = st.concurrency or len(alive)
        result["async_discarded"] = 0

        def dispatch() -> None:
            nonlocal dispatched
            while idle and len(in_flight) < concurrency:
                wid = idle.pop(0)
                task = asyncio.ensure_future(self._fit(loop, pool, wid, alive[wid], current, cfg.with_seed(cfg.seed + dispatched), codec,
                                                       ef_reset=wid not in fitted, version=version))
                in_flight[task] = (wid, version)
                fitted.add(wid)
                dispatched += 1

        async def collect() -> List[asyncagg.Reply]:
            """the checked replies of the fits that ended by the time the first of them did"""
            done, _ = await asyncio.wait(list(in_flight), return_when=asyncio.FIRST_COMPLETED)
            got = []
            for task in done:
                wid, base = in_flight.pop(task)
                update, loss, n = task.result()
                if update is None:
                    result["dropped"].append(wid)
                    alive.pop(wid, None)
                    continue
                self.metrics.worker_loss(wid, loss)
                result["losses"][wid] = loss
                got.append(asyncagg.Reply(wid, base, update, n, loss))
                idle.append(wid)
            return got

        t0 = time.time()
        sent0 = {wid: traffic(w) for wid, w in to_train.items()}
        while steps < self.enabled_round and (in_flight or idle):
            dispatch()
            buffer += await collect()
            while len(buffer) >= st.buffer and steps < self.enabled_round:
                batch, buffer = buffer[:st.buffer], buffer[st.buffer:]
                rec = self._async_step(th, ring, batch, version, st, codec, len(in_flight))
                version += 1
                current = th.detach().to("cpu", copy=True)
                if self._fed_eval_round(steps):
                    while in_flight:                                    # drain: the fits in flight count toward the next step
                        buffer += await collect()
                    rec["fed_eval"] = result["fed_eval"] = await self._remote_fed_eval(alive, current, eval_classes, loop, pool, ae=anomaly.is_autoencoder(model))
                sent = {wid: traffic(w) for wid, w in to_train.items()}
                rec["bytes_out"] = sum(sent[w][0] - sent0[w][0] for w in sent)
                rec["bytes_in"] = sum(sent[w][1] - sent0[w][1] for w in sent)
                result["bytes_out"] = result.get("bytes_out", 0) + rec["bytes_out"]
                result["bytes_in"] = result.get("bytes_in", 0) + rec["bytes_in"]
                sent0 = sent
                self.metrics.end_round(steps, time.time() - t0, **rec)
                self._maybe_checkpoint(model, current, steps, {"workers": list(to_train.keys()), "mode": "remote", **self._model_meta(model, result)})
                steps += 1
                t0 = time.time()
        # after the last step: nothing new is dispatched; what is still in flight is awaited, then discarded with the buffer
        left = len(in_flight)
        if in_flight:
            _, late = await asyncio.wait(list(in_flight), timeout=self.fit_timeout)
            for task in late:
                task.cancel()
        result["async_discarded"] = left + len(buffer)
        result["async_steps"] = steps
        return current

    def _async_step(self, th: torch.Tensor, ring: Optional[torch.Tensor], batch, version: int, st, codec: UplinkCodec,
                    in_flight: int) -> Dict[str, Any]:
        """One asynchronous server step on ``th`` at global ``version`` with the buffered replies ``batch``: returns the step's
        record (``selected``, ``n_k`` and ``async``, plus ``agg_weights`` under a distance-based aggregator)."""
        plan = asyncagg.plan_step(batch, version, st, self.args.weighted)
        rec: Dict[str, Any] = {"selected": [r.device for r in plan.kept], "n_k": [r.n for r in plan.kept]}
        if plan.kept:
            w = torch.tensor(plan.weights, dtype=torch.float32, device=self.device)
            if ring is None:
                wire = uplink.stack([r.update for r in plan.kept], codec, self.device)
                agg_w = self._server_update(th, partial(uplink.server_apply, th, wire, w, codec), len(plan.kept))
            else:
                models = torch.stack([r.update for r in plan.kept]).to(self.device)
                agg_w = self._server_update(th, partial(ops.fedavg_apply_based, th, models, ring, [st.slot(r.base) for r in plan.kept], w,
                                                        st.slot(version + 1)), len(plan.kept))
            if agg_w is not None:
                rec["agg_weights"] = agg_w
        elif ring is not None:
            ring[st.slot(version + 1)].copy_(th)                   # nothing applied: version + 1 is the same model
        rec["async"] = {"version": version, "replies": plan.record, "stale_dropped": plan.stale_dropped, "in_flight": in_flight}
        return rec

    async def _remote_fed_eval(self, alive, theta: torch.Tensor, classes: int, loop, pool, ae: bool = False) -> Dict[str, Any]:
        """Federated evaluation of ``theta`` (the true global model, fp32) on every live device's evaluation data.  Every reply
        must be the summary of ``classes`` output columns (the coordinator's model, never what the device claims) and pass
        ``fedeval.from_wire``'s checks, or the device is listed under ``eval_excluded``; a device without evaluation data is
        listed under ``eval_missing``.  ``ae``: the model is an autoencoder, the replies are reconstruction-error summaries
        (``anomaly.from_wire``) and the record carries the federated alarm threshold (``anomaly.record``)."""
        bins, thr = self.args.eval_bins, self.args.eval_threshold
        decode = (lambda resp: anomaly.from_wire(resp, bins)) if ae else (lambda resp: fedeval.from_wire(resp, classes, bins))

        async def ask(wid, worker):
            try:
                resp = await loop.run_in_executor(pool, lambda: worker.evaluate(theta, self.args.model, bins, thr, timeout=self.fit_timeout))
                if not resp.get("ok", False):
                    return wid, "missing" if resp.get("eval_missing") else "excluded"
                return wid, decode(resp)
            except Exception as e:  # noqa: BLE001 - a device's reply is untrusted: it is left out of the total
                log.info("Worker %s: evaluation reply refused: %r", wid, e)
                return wid, "excluded"

        answers = await asyncio.gather(*[ask(wid, w) for wid, w in alive.items()])
        good = {wid: a for wid, a in answers if isinstance(a, (fedeval.Summary, anomaly.ReconSummary))}
        excluded, missing = [wid for wid, a in answers if a == "excluded"], [wid for wid, a in answers if a == "missing"]
        if ae:
            return anomaly.record(good, self.args.alarm_fpr, bins, excluded=excluded, missing=missing)
        if category.is_category(MODEL_REGISTRY.get(self.args.model)):
            return category.record(good, excluded=excluded, missing=missing)
        return fedeval.record(good, excluded=excluded, missing=missing)

    async def _secagg_setup(self, alive, tag: str, loop, pool, result) -> Optional[Dict[str, Any]]:
        """Secure aggregation's key agreement: every device returns a fresh public key for the training ``tag``, then every
        device that did gets the key list in setup order and derives its pair seeds.  A device that fails either step leaves
        the training.  Returns ``{"tag", "order", "clip", "frac_bits"}`` (``frac_bits`` for the devices left, see
        :func:`fl.secagg.frac_bits`), or None when fewer than two are left."""
        clip = self.args.secagg_clip_value()
        before = {wid: traffic(w) for wid, w in alive.items()}
        handles = dict(alive)

        async def call(wid, fn):
            try:
                return wid, await loop.run_in_executor(pool, fn)
            except Exception as e:  # noqa: BLE001 - a failing device leaves the training, the others go on
                log.info("Worker %s failed the secure-aggregation setup: %r", wid, e)
                result["dropped"].append(wid)
                alive.pop(wid, None)
                return wid, None

        keys = await asyncio.gather(*[call(wid, lambda w=w: pk_to_bytes(pk_from_bytes(w.secagg_setup(tag, timeout=self.fit_timeout))))
                                      for wid, w in alive.items()])
        ids = [wid for wid, pk in keys if pk is not None]
        pks = [pk for _, pk in keys if pk is not None]
        await asyncio.gather(*[call(wid, lambda w=alive[wid]: w.secagg_peers(tag, ids, pks, timeout=self.fit_timeout)) for wid in ids])
        result["secagg_setup_bytes_out"] = sum(traffic(w)[0] - before[wid][0] for wid, w in handles.items())
        result["secagg_setup_bytes_in"] = sum(traffic(w)[1] - before[wid][1] for wid, w in handles.items())
        if len(alive) < 2:
            log.info("Secure aggregation needs at least two devices, %d left after the setup: no rounds", len(alive))
            return None
        f = frac_bits(clip, len(alive))
        result["secagg_frac_bits"] = f
        return {"tag": tag, "order": list(ids), "clip": clip, "frac_bits": f}

    async def _secagg_round(self, theta, r: int, u1: List[str], ids: List[str], replies, alive, sa, loop, pool, result):
        """Unmask and apply round ``r`` of secure aggregation.  ``replies``: the checked masked replies of the devices ``ids``
        (the survivors U2); the others of ``u1`` dropped (D).  Every survivor is asked for its self seed and its pair seeds with
        the dropped devices; if fewer than two survived or one of them does not answer, the round is abandoned (theta
        unchanged, a device that did not answer leaves the training).  Returns ``(theta, the round's secagg record)``."""
        got = dict(zip(ids, replies))
        survivors = [w for w in u1 if w in got]
        dropped = [w for w in u1 if w not in got]
        rec = {"secagg_u2": len(survivors), "secagg_dropped": len(dropped), "secagg_clipped": sum(got[w][1] for w in survivors),
               "secagg_nonfinite": sum(got[w][2] for w in survivors), "secagg_abandoned": True}
        if len(survivors) < 2:
            log.info("Secure aggregation round %d abandoned: %d device(s) survived", r, len(survivors))
            return theta, rec

        async def ask(wid):
            try:
                resp = await loop.run_in_executor(pool, lambda: alive[wid].secagg_unmask(sa["tag"], r, survivors, timeout=self.fit_timeout))
                return wid, check_unmask_reply(resp, dropped)
            except Exception as e:  # noqa: BLE001 - a device that does not answer abandons the round
                log.info("Worker %s failed the unmask of round %d: %r", wid, r, e)
                return wid, None

        answers = await asyncio.gather(*[ask(w) for w in survivors])
        failed = [w for w, a in answers if a is None]
        if failed:
            log.info("Secure aggregation round %d abandoned: no seeds from %s", r, failed)
            for w in failed:
                result["dropped"].append(w)
                alive.pop(w, None)
            return theta, rec
        keys, signs = correction_streams(sa["order"], survivors, dropped, dict(answers))
        masked = torch.from_numpy(np.stack([got[w][0] for w in survivors]).view(np.int32))
        th = theta.to(self.device)
        self._server_update(th, partial(ops.fedavg_apply_secagg, th, masked.to(self.device), keys, signs, sa["frac_bits"], len(survivors)),
                            len(survivors))
        rec["secagg_abandoned"] = False
        return th.cpu(), rec

    @staticmethod
    def _downlink_fields(down: UplinkCodec, theta: torch.Tensor, replica: torch.Tensor, nonce: str, r: int, seed: int) -> Dict[str, Any]:
        """The downlink fields of round ``r``'s fit request, built once for every device.  Round 0: the codec and the replica's
        tag (the request carries the fp32 model, which becomes the replica).  Later rounds: the wire of ``theta - replica``
        (rounded with ``downlink_key(seed)``), the tag it applies to and the new tag; ``replica`` advances by the wire."""
        fields: Dict[str, Any] = {"downlink": down.kind, "downlink_topk": down.k, "replica": f"{nonce}:{r}"}
        if r == 0:
            return fields
        wire = ops.encode_downlink(theta.to(replica.device), replica, down, downlink_key(seed))
        fields["replica_base"] = f"{nonce}:{r - 1}"
        fields.update(uplink.wire_fields(down, wire, prefix="d"))
        return fields

    def _server_update(self, theta: torch.Tensor, apply, k: int) -> Optional[List[float]]:
        """One server step on ``theta`` in place: ``apply`` is a fused FedAvg apply of :mod:`ops` bound to theta and the round's
        ``k`` rows (``partial(uplink.server_apply, theta, wire, w, codec)`` and the like); it gets the
        aggregate of ``--aggregator`` (mean, median / trimmed mean, geometric median / norm-bounded mean) and the step of
        ``--server-opt``.  Returns the final weight of every row under a distance-based aggregator (0 for a row it excluded),
        None otherwise."""
        agg = self.args.client_aggregator()
        kw: Dict[str, Any] = {"aggregator": agg}
        if agg.distance_based:
            kw["agg_weights_out"] = torch.zeros(k, dtype=torch.float32, device=theta.device)
        if self.args.server_opt == "sgd":
            kw["server_lr"] = self.args.server_lr
        else:
            kw["opt"] = self._server_opt_state = server_opt_state(self._server_opt_state, self.args.server_optimizer(), theta)
        apply(**kw)
        return kw["agg_weights_out"].cpu().tolist() if agg.distance_based else None

    @staticmethod
    def _average_buffers(model, buffers, weights) -> None:
        """BatchNorm models in remote mode: the devices return their running statistics next to the parameters; the global
        model gets their FedAvg-weighted mean (PySyft's federated_avg averages parameters only — with it the reference could
        not train a BatchNorm model remotely at all; documented in docs/PARITY.md).  They keep this mean under a robust
        ``--aggregator`` too: only the parameters get the median / trimmed mean / geometric median / norm-bounded mean."""
        mine = [b for b in model.buffers() if b.is_floating_point()]
        total = sum(b.numel() for b in mine)
        if not mine or any(b is None or b.numel() != total or not bool(torch.isfinite(b).all()) for b in buffers):
            return
        avg = (torch.stack([b.float() for b in buffers]) * weights.view(-1, 1).float()).sum(0)
        off = 0
        with torch.no_grad():
            for b in mine:
                b.copy_(avg[off:off + b.numel()].view_as(b).to(b.device))
                off += b.numel()

    # ------------------------------------------------------------------ inference (remote only)
    def _inference(self, worker: RemoteWorkerClient) -> None:
        model = self._load_model()
        flat = flatten_params(model)
        alarm = None
        if anomaly.is_autoencoder(model):
            # the alarm threshold travels with the checkpoint (its JSON sidecar); without one an autoencoder flags nothing
            from ..utils.checkpoint import load_meta
            alarm = (load_meta(self.path).get("anomaly") or {}) if os.path.exists(self.path) else {}
            if alarm.get("alarm_bin") is None or alarm.get("bins") is None:
                log.info("Inference refused: the autoencoder checkpoint at %s has no alarm threshold (train it with --fed-eval-every)",
                         self.path)
                self.known_workers.pop(worker.id, None)
                worker.close()
                return
        try:
            count = worker.search("inference")
            log.info("inference tensors found: %d", count)
            if count > 0:
                pred = worker.predict(flat, self.args.model, alarm=alarm)
                self.last_predictions = pred
                log.info(pred)
                if category.is_category(model):
                    log.info("attack categories: %s", [category.CATEGORIES[i] if 0 <= i < len(category.CATEGORIES) else i for i in pred])
            else:
                log.info("Inference data not found!")
        finally:
            self.known_workers.pop(worker.id, None)
            worker.close()


# --------------------------------------------------------------------------------------------------
def train_virtual_workers(theta: torch.Tensor, model, fed, cfg: FitConfig, round_idx: int):
    """One round of local training for every virtual worker, each starting from ``theta``.

    On a GPU with a persistent-kernel instantiation all K workers train **concurrently in one
    launch** (one CTA per worker); otherwise they run one after the other through ``local_fit``.
    Returns ``(flats[K,P], last_losses[K], sample_counts[K])``.
    """
    k = len(fed.workers)
    device = theta.device
    flats = theta.unsqueeze(0).repeat(k, 1).contiguous()
    counts = [len(fed[w]) for w in fed.workers]
    losses = [0.0] * k
    spec = model.spec if isinstance(model, MLPNet) else None
    fused = (spec is not None and device.type == "cuda" and ops.net_kind_for(spec.dims, spec.out_activation) is not None)
    if fused:
        loss_out = torch.zeros(k, 2, device=device)
        tasks, idx = [], []
        for i, wid in enumerate(fed.workers):
            sh = fed[wid]
            if len(sh) == 0:
                continue
            perm = make_perm(len(sh), cfg.with_seed(cfg.seed + 31 * i), device, round_idx)
            x = sh.x.view(len(sh), -1).contiguous().float()
            y = sh.y.contiguous().float().view(len(sh), -1)
            tasks.append(ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=flats[i], perm=perm, loss_out=loss_out[i]))
            idx.append(i)
        if tasks:
            descs = ops.build_client_descs(tasks, device)
            ops.mlp_local_sgd_multi(spec.dims, spec.out_activation, descs, len(tasks), cfg.batch_size, cfg.lr,
                                    cfg.epochs, cfg.max_nr_batches, resolve_loss(cfg.model, cfg.loss))
            vals = loss_out[:, 0].tolist()
            for i in idx:
                losses[i] = vals[i]
        return flats, losses, counts
    if spec is not None and device.type == "cpu" and ops.host.available() and spec.out_activation in ("none", "sigmoid"):
        # CPU box: the native host executor trains the K workers concurrently on K threads (ops/csrc/mlp_host.cpp)
        idx = [i for i, wid in enumerate(fed.workers) if len(fed[wid]) > 0]
        if idx:
            shards = [fed[fed.workers[i]] for i in idx]
            perms = [make_perm(len(sh), cfg.with_seed(cfg.seed + 31 * i), device, round_idx)
                     for i, sh in zip(idx, shards)]
            res = ops.host.mlp_local_sgd_multi(spec.dims, spec.out_activation, [flats[i] for i in idx], [sh.x for sh in shards],
                                               [sh.y for sh in shards], perms, cfg.batch_size, cfg.lr, cfg.epochs,
                                               cfg.max_nr_batches, resolve_loss(cfg.model, cfg.loss))
            for j, i in enumerate(idx):
                losses[i] = float(res[j, 0])
        return flats, losses, counts
    for i, wid in enumerate(fed.workers):
        sh = fed[wid]
        if len(sh) == 0:
            continue
        wcfg = cfg.with_seed(cfg.seed + 31 * i)
        last, _ = local_fit(flats[i], model, sh.x, sh.y, wcfg, round_idx)
        losses[i] = float(last)
    return flats, losses, counts
