"""Worker handles and the device-side worker runtime.

Replaces PySyft's ``VirtualWorker`` / ``WebsocketClientWorker`` / ``WebsocketServerWorker``
(instantiated at ``federated_coordinator.py:149,167`` and ``remote_worker.py:95``; SURVEY L0).

* :class:`VirtualWorker` — in-process worker object (local mode, fc.py:139-149).
* :class:`WorkerServer` — device-side runtime (``remote_worker.py`` hosts one): owns the private
  dataset under key ``"training"`` (rw.py:108) and tagged inference tensors (rw.py:102-104) and
  serves ``fit`` / ``search`` / ``predict`` / ``ping`` RPCs.
* :class:`RemoteWorkerClient` — coordinator-side handle with the same verbs.

Wire format: 4-byte big-endian length + msgpack map; tensors travel as raw little-endian fp32
bytes of the **flat arena** (9.6 kB for FFNN instead of ≈36 kB of TorchScript+msgpack per leg,
SURVEY §2.5).  Workers never execute code received from the wire: the model is chosen by name
from the registry and the loss by name — unlike the reference, which ships TorchScript.
"""
from __future__ import annotations

import logging
import socket
import socketserver
import struct
import threading
import zlib
from typing import Any, Dict, List, Optional, Tuple

import msgpack
import numpy as np
import torch

from ..data import dataset_tensors
from ..fl import anomaly, category, fedeval
from ..fl.trainer import FitConfig, local_fit
from ..fl.evaluate import predict as predict_fn
from ..fl.secagg import SecAggDevice
from ..fl.uplink import FIELDS, UplinkCodec, check_reply, device_reply, echo, request_fields, uplink_key
from ..models import build_model, num_params

log = logging.getLogger(__name__)


class VirtualWorker:
    """In-process worker.  Data arrives via ``federate()`` at training time (reference local mode)
    or can be attached up-front with :meth:`add_dataset`."""

    def __init__(self, worker_id: str, device: Optional[torch.device] = None) -> None:
        self.id = worker_id
        self.device = device
        self.datasets: Dict[str, Tuple[torch.Tensor, torch.Tensor]] = {}
        self.tagged: Dict[str, List[torch.Tensor]] = {}

    def add_dataset(self, dataset, key: str = "training") -> None:
        self.datasets[key] = dataset_tensors(dataset, self.device)

    def load_data(self, tensors: List[torch.Tensor], tag: str = "inference") -> None:
        self.tagged.setdefault(tag, []).extend(tensors)

    def search(self, tag: str) -> List[torch.Tensor]:
        return list(self.tagged.get(tag, []))

    def close(self) -> None:
        pass

    def __repr__(self) -> str:
        return f"<VirtualWorker id:{self.id}>"


# ---------------------------------------------------------------------------------------------
# framing
# ---------------------------------------------------------------------------------------------
def _send_msg(sock: socket.socket, obj: Dict[str, Any]) -> int:
    """Returns the number of bytes put on the wire (frame header included)."""
    data = msgpack.packb(obj, use_bin_type=True)
    sock.sendall(struct.pack(">I", len(data)) + data)
    return 4 + len(data)


def _recv_exact(sock: socket.socket, n: int) -> bytes:
    buf = bytearray()
    while len(buf) < n:
        chunk = sock.recv(n - len(buf))
        if not chunk:
            raise ConnectionError("peer closed the connection")
        buf.extend(chunk)
    return bytes(buf)


MAX_FRAME = 1 << 30   # 1 GiB: five times the largest arena in the model zoo (wide MLP, 201.6 MB)


def _recv_msg(sock: socket.socket, counter: Optional[List[int]] = None) -> Dict[str, Any]:
    (n,) = struct.unpack(">I", _recv_exact(sock, 4))
    if n > MAX_FRAME:
        raise ConnectionError(f"frame of {n} bytes exceeds the {MAX_FRAME}-byte limit")
    if counter is not None:
        counter[0] += 4 + n
    return msgpack.unpackb(_recv_exact(sock, n), raw=False)


def _to_bytes(t: torch.Tensor) -> bytes:
    return t.detach().to("cpu", torch.float32).contiguous().numpy().tobytes()


def _from_bytes(b: bytes, device=None) -> torch.Tensor:
    t = torch.from_numpy(np.frombuffer(b, dtype=np.float32).copy())
    return t.to(device) if device is not None else t


def replica_crc(replica: torch.Tensor) -> int:
    """crc32 of a downlink replica's fp32 bytes: a device reports it after every fit, the coordinator compares it with its own"""
    return zlib.crc32(_to_bytes(replica))


def _codec(kind: str, k: Any) -> UplinkCodec:
    """The codec a fit request names; ``k`` only counts for topk"""
    return UplinkCodec(kind, k=k) if kind == "topk" else UplinkCodec(kind)


# ---------------------------------------------------------------------------------------------
# device-side runtime
# ---------------------------------------------------------------------------------------------
class WorkerServer:
    def __init__(self, worker_id: str, host: str, port: int, device: Optional[torch.device] = None,
                 verbose: bool = False, ssl_context=None) -> None:
        self.id = worker_id
        self.ssl_context = ssl_context          # control/tls.py::server_context(...): the reference's cert_path / key_path stub
        self.device = device or torch.device("cuda" if torch.cuda.is_available() else "cpu")
        self.verbose = verbose
        self.datasets: Dict[str, Tuple[torch.Tensor, torch.Tensor]] = {}
        # attack-category class indices [N, 1] of a hosted dataset that has them (fl/category.py), under the same key
        self.categories: Dict[str, torch.Tensor] = {}
        self.tagged: Dict[str, List[torch.Tensor]] = {}
        self.fits_served = 0
        self._round = 0
        # one model instance + one flat arena per architecture, reused across fits: the trainers behind local_fit
        # (layer-wise MLP, conv net) cache their buffers / CUDA graphs per (model, arena)
        self._models: Dict[str, Tuple[torch.nn.Module, torch.Tensor]] = {}
        # topk uplink: the error-feedback residual [1, P] per architecture, on this device (memory only, like the arenas)
        self._residuals: Dict[str, torch.Tensor] = {}
        # compressed downlink: (tag, replica [P]) per architecture, the model as the coordinator last sent it (memory only)
        self._replicas: Dict[str, Tuple[str, torch.Tensor]] = {}
        self._work_lock = threading.Lock()   # fits / predictions share those buffers: one at a time
        # secure aggregation (fl/secagg.py): key pairs, pair seeds and per-round self seeds per training (memory only)
        self._secagg = SecAggDevice()
        self._secagg_lock = threading.Lock()
        outer = self

        class Handler(socketserver.BaseRequestHandler):
            def setup(self) -> None:
                self.tls_failed = False
                if outer.ssl_context is not None:
                    self.request.settimeout(10.0)
                    try:
                        self.request = outer.ssl_context.wrap_socket(self.request, server_side=True)
                        self.request.settimeout(None)
                    except (OSError, ValueError) as e:
                        log.info("TLS handshake with %s failed: %r", self.client_address, e)
                        self.tls_failed = True

            def handle(self) -> None:
                while not self.tls_failed:
                    try:
                        req = _recv_msg(self.request)
                    except (ConnectionError, OSError, struct.error):
                        return
                    try:
                        resp = outer._dispatch(req)
                    except Exception as e:  # noqa: BLE001 - report to the coordinator, keep serving
                        log.exception("worker RPC failed")
                        resp = {"ok": False, "error": repr(e)}
                    try:
                        _send_msg(self.request, resp)
                    except OSError:
                        return
                    if req.get("op") == "close":
                        return

        class Server(socketserver.ThreadingMixIn, socketserver.TCPServer):
            allow_reuse_address = True
            daemon_threads = True

        self._server = Server((host, port), Handler)
        self.host, self.port = self._server.server_address[:2]
        self._thread: Optional[threading.Thread] = None

    # -- data hosting (rw.py:97-108) -------------------------------------------------------
    def add_dataset(self, dataset, key: str = "training") -> None:
        self.datasets[key] = dataset_tensors(dataset, self.device)
        self.categories.pop(key, None)
        if getattr(dataset, "categories", None) is not None:
            self.categories[key] = category.labels(dataset, self.device)[1]

    def hold_out_evaluation(self, fraction: float, seed: int) -> None:
        """Move a seeded ``fraction`` of the training rows to the evaluation set (``fedeval.split_eval``), their attack
        categories with them when the training data has some"""
        x, y = self.datasets["training"]
        xt, yt, xe, ye = fedeval.split_eval(x, y, fraction, seed)
        self.datasets["training"], self.datasets["evaluation"] = (xt, yt), (xe, ye)
        self.categories.pop("evaluation", None)
        if "training" in self.categories:           # the same rows: the split depends on n and the seed only
            _, ct, _, ce = fedeval.split_eval(x, self.categories["training"], fraction, seed)
            self.categories["training"], self.categories["evaluation"] = ct, ce

    def _labels(self, model, key: str, y: torch.Tensor) -> Tuple[Optional[torch.Tensor], Optional[str]]:
        """``(labels, None)`` the model trains and is scored on: the attack categories for a category model, ``y`` otherwise;
        ``(None, reason)`` when this device's ``key`` data has no categories"""
        if not category.is_category(model):
            return y, None
        codes = self.categories.get(key)
        if codes is None:
            return None, f"{model.__class__.__name__} trains on attack categories: this device's {key} data has none"
        return codes, None

    def load_data(self, tensors: List[torch.Tensor], tag: str = "inference") -> None:
        self.tagged.setdefault(tag, []).extend(t.to(self.device) for t in tensors)

    # -- RPC -----------------------------------------------------------------------------------
    def _dispatch(self, req: Dict[str, Any]) -> Dict[str, Any]:
        op = req.get("op")
        if self.verbose:
            log.info("worker %s <- %s", self.id, op)
        if op == "ping":
            return {"ok": True, "id": self.id}
        if op == "close":
            return {"ok": True}
        if op == "search":
            return {"ok": True, "count": len(self.tagged.get(req["tag"], []))}
        if op in ("secagg_setup", "secagg_unmask"):
            # secure aggregation (fl/secagg.py): "secagg_setup" with a tag returns this device's public key for the training,
            # with "ids" / "pks" it takes the key list; "secagg_unmask" reveals one round's seeds for the survivors "u2"
            try:
                with self._secagg_lock:
                    if op == "secagg_unmask":
                        return {"ok": True, **self._secagg.unmask(req.get("tag"), req.get("t"), req.get("u2"))}
                    if "pks" in req:
                        self._secagg.learn_peers(req.get("tag"), req.get("ids"), req.get("pks"))
                        return {"ok": True}
                    return {"ok": True, "pk": self._secagg.setup(req.get("tag"))}
            except ValueError as e:
                return {"ok": False, "error": f"secure aggregation refused: {e}"}
        if op == "fit":
            return self._fit(req)
        if op == "evaluate":
            # federated evaluation (fl/fedeval.py): the model in "params" (fp32) scored on the rows hosted under "evaluation";
            # only the summary's counts leave the device
            held = self.datasets.get("evaluation")
            if held is None:
                return {"ok": False, "eval_missing": True, "error": "no evaluation data on this device"}
            if "params" not in req:
                return {"ok": False, "error": "evaluate request without params"}
            with self._work_lock:
                try:
                    model, flat, err = self._model_and_arena(req.get("model"), req["params"])
                    if err:
                        return {"ok": False, "error": err}
                    spec = getattr(model, "spec", None)
                    if spec is not None and not spec.flatten_input and held[0].shape[1] != spec.dims[0]:
                        return {"ok": False, "error": f"evaluation data has {held[0].shape[1]} features, {req.get('model')} wants {spec.dims[0]}"}
                    if anomaly.is_autoencoder(model):
                        return {"ok": True, **anomaly.to_wire(anomaly.summarize(model, flat, held[0], held[1], int(req.get("bins", 256)))[0])}
                    ey, why = self._labels(model, "evaluation", held[1])
                    if why:
                        return {"ok": False, "error": f"evaluation refused: {why}"}
                    s = fedeval.summarize(model, flat, held[0], ey, int(req.get("bins", 256)), float(req.get("threshold", 0.5)))[0]
                except (ValueError, TypeError) as e:
                    return {"ok": False, "error": f"evaluation refused: {e}"}
                return {"ok": True, **fedeval.to_wire(s)}
        if op == "predict":
            data = self.tagged.get(req.get("tag", "inference"), [])
            if not data:
                return {"ok": True, "pred": [], "count": 0}
            with self._work_lock:
                model, flat, err = self._model_and_arena(req["model"], req["params"])
                if err:
                    return {"ok": False, "error": err}
                spec = getattr(model, "spec", None)
                keep_shape = spec is None                       # conv nets take [C, H, W] samples as they are
                x = torch.stack([d if keep_shape else d.reshape(-1) for d in data]).float()
                if anomaly.is_autoencoder(model):
                    # per-row alarms at the federated threshold the request carries ("alarm_bin" of "bins" error bins)
                    j, bins = req.get("alarm_bin"), req.get("bins")
                    if not isinstance(j, int) or not isinstance(bins, int) or isinstance(j, bool) or isinstance(bins, bool):
                        return {"ok": False, "error": f"{req['model']} predicts alarms: the request needs an integer alarm_bin and bins"}
                    try:
                        pred = anomaly.predict(model, flat, x, j, bins)
                    except ValueError as e:
                        return {"ok": False, "error": f"prediction refused: {e}"}
                    return {"ok": True, "pred": pred.reshape(-1).tolist(), "count": len(data)}
                pred = predict_fn(model, x, flat)
                return {"ok": True, "pred": pred.reshape(-1).tolist(), "count": len(data)}
        return {"ok": False, "error": f"unknown op {op!r}"}

    def _fit(self, req: Dict[str, Any]) -> Dict[str, Any]:
        """A fit request: its refusals, the model it trains (the fp32 ``params`` or the downlink replica), the fit and the
        reply with the update in the format the request asks for.  A refused request trains nothing and is not counted."""
        cfg = FitConfig.from_dict(req["config"])
        key = req.get("dataset_key", "training")
        x, y = self.datasets[key]
        # "uplink": send the quantized or top-k delta instead of the model (fl/uplink.py); absent = the fp32 model.
        # topk carries "topk" (k in 1..32, anything else is refused before the fit) and "ef_reset" (zero the residual)
        codec = _codec(req.get("uplink", "fp32"), req.get("topk"))
        # "downlink": the model arrives as a compressed delta to the replica this device keeps (fl/uplink.py); absent = fp32
        down = _codec(req.get("downlink", "fp32"), req.get("downlink_topk"))
        if down.kind != "fp32" and not isinstance(req.get("replica"), str):
            return {"ok": False, "error": "a compressed downlink needs the replica's tag"}
        # "secagg": send the masked fixed-point delta (fl/secagg.py) instead of the model; absent = no secure aggregation
        sa = req.get("secagg")
        if sa is not None and (not isinstance(sa, dict) or codec.kind != "fp32"):
            return {"ok": False, "error": "secure aggregation takes a dict of fields and no uplink codec"}
        with self._work_lock:
            model, flat, wire = self._restore(req, cfg.model, down)
            if model is None:
                return {"ok": False, "error": wire}
            spec = getattr(model, "spec", None)
            if spec is not None and not spec.flatten_input and x.shape[1] != spec.dims[0]:
                return {"ok": False, "error": f"dataset has {x.shape[1]} features, {cfg.model} wants {spec.dims[0]}"}
            if anomaly.is_autoencoder(model):
                x, y = anomaly.training_rows(x, y)       # the benign rows, the input as the target; n = their count
            y, why = self._labels(model, key, y)
            if why:
                return {"ok": False, "error": why}
            if sa is not None:
                if any(b.is_floating_point() for b in model.buffers()):
                    return {"ok": False, "error": f"secure aggregation refused: {cfg.model}'s floating-point buffers would travel in the clear"}
                try:
                    with self._secagg_lock:
                        sa_keys, sa_signs = self._secagg.begin_round(sa.get("tag"), sa.get("t"), sa.get("u1"), sa.get("clip"),
                                                                     sa.get("frac_bits"))
                except ValueError as e:
                    return {"ok": False, "error": f"secure aggregation refused: {e}"}
            replica = None
            if down.kind != "fp32":
                if wire is not None:                  # round t >= 1: advance the replica by the wire, train from it
                    from .. import ops
                    replica = self._replicas[cfg.model][1]
                    ops.apply_downlink(replica, wire[0].to(replica.device), wire[1].to(replica.device), down)
                    flat.copy_(replica)
                else:                                 # round 0: the fp32 model is the replica
                    replica = flat.clone()
                self._replicas[cfg.model] = (str(req.get("replica")), replica)
            # the theta the coordinator decodes against
            received = flat.clone() if codec.kind != "fp32" or sa is not None else None
            from ..utils.threads import small_model_threads
            with small_model_threads(flat.numel(), flat.device):   # tiny models on a CPU device: no OpenMP fork/join
                loss, path = local_fit(flat, model, x, y, cfg, round_idx=self._round)
            self._round += 1
            self.fits_served += 1
            if sa is not None:
                from .. import ops
                masked, clipped, nonfinite = ops.secagg_mask(flat, received, sa_keys, sa_signs, sa["clip"], sa["frac_bits"])
                update = {"secagg": "masked", "masked": masked.cpu().numpy().astype("<u4").tobytes(), "clipped": clipped,
                          "nonfinite": nonfinite}
            else:
                update = device_reply(codec, flat, received, uplink_key(self.id, cfg.seed), self._residuals, cfg.model,
                                      bool(req.get("ef_reset")))
            reply = {"ok": True, **update, "loss": float(loss), "n": int(x.shape[0]), "path": path}
            # floating-point buffers the fit updated on this device (BatchNorm running statistics): the flat arena holds
            # named_parameters only, so without them the coordinator would save trained weights next to the INITIAL running
            # stats and every eval-mode use of the checkpoint would be meaningless (FFNN / MLPs have none: nothing is sent)
            bufs = [b.detach().reshape(-1).float() for b in model.buffers() if b.is_floating_point()]
            if bufs:
                reply["buffers"] = _to_bytes(torch.cat(bufs))
            if replica is not None:
                reply["replica_crc"] = replica_crc(replica)
            if "version" in req:                      # asynchronous aggregation: the global version this fit started from
                reply["version"] = req["version"]
            return reply

    def _restore(self, req: Dict[str, Any], name: str, down: UplinkCodec):
        """``(model, arena, downlink wire)`` a fit request trains from, or ``(None, None, reason)``: the fp32 ``params`` (wire
        None), or from round t >= 1 of a compressed downlink the arena as it is plus the checked wire that advances the
        replica (the caller applies it once nothing else refuses the request)."""
        if down.kind != "fp32" and "replica_base" in req:
            model, flat, _ = self._model_and_arena(name, None)
            wire = self._downlink_wire(req, down, name, flat.numel())
            return (None, None, wire) if isinstance(wire, str) else (model, flat, wire)
        if "params" not in req:
            return None, None, "fit request without params"
        return self._model_and_arena(name, req["params"])

    def _downlink_wire(self, req: Dict[str, Any], codec: UplinkCodec, model: str, p: int):
        """The two wire tensors of a round t >= 1 downlink, or the reason it is refused: this device must hold the replica
        of ``model`` tagged ``replica_base``, and the wire must pass the checks the coordinator runs on replies."""
        held = self._replicas.get(model)
        if held is None or held[0] != req.get("replica_base") or held[1].numel() != p:
            return f"no replica {req.get('replica_base')!r} of {model} on this device (it holds {held[0] if held else None!r})"
        try:
            return check_reply({**echo(codec), **{name: req.get("d" + name) for name in FIELDS[codec.kind]}}, codec, p)
        except ValueError as e:
            return f"downlink refused: {e}"

    def _model_and_arena(self, name: str, params: Optional[bytes]):
        """(model, arena holding ``params``, error) — instances are created once per architecture; ``params`` None leaves
        the arena as it is."""
        if name not in self._models:
            model = build_model(name).to(self.device)
            self._models[name] = (model, torch.empty(num_params(model), device=self.device))
        model, flat = self._models[name]
        if params is None:
            return model, flat, None
        incoming = _from_bytes(params)
        if incoming.numel() != flat.numel():
            return None, None, f"param count {incoming.numel()} != {flat.numel()} for {name}"
        flat.copy_(incoming)
        return model, flat, None

    def start(self, block: bool = True) -> None:
        if block:
            self._server.serve_forever()
        else:
            self._thread = threading.Thread(target=self._server.serve_forever, name=f"worker-{self.id}", daemon=True)
            self._thread.start()

    def stop(self) -> None:
        self._server.shutdown()
        self._server.server_close()


# ---------------------------------------------------------------------------------------------
# coordinator-side handle
# ---------------------------------------------------------------------------------------------
class RemoteWorkerClient:
    def __init__(self, worker_id: str, host: str, port: int, timeout: Optional[float] = 10.0,
                 verbose: bool = False, ssl_context=None) -> None:
        self.id = worker_id
        self.host, self.port = host, port
        self.verbose = verbose
        self._lock = threading.Lock()
        sock = socket.create_connection((host, port), timeout=timeout)
        if ssl_context is not None:
            sock = ssl_context.wrap_socket(sock, server_hostname=host)
        self._sock: Optional[socket.socket] = sock
        self._sock.settimeout(None)
        # application-level traffic of this handle (the paper's §4.3 measures the same two directions with psutil:
        # ~36 kB per worker and round towards the device, ~30.6 kB back, for a 9.6 kB model)
        self.bytes_sent = 0
        self.bytes_received = 0

    def _call(self, req: Dict[str, Any], timeout: Optional[float] = None, check: bool = True) -> Dict[str, Any]:
        with self._lock:
            if self._sock is None:
                raise ConnectionError(f"worker {self.id} is closed")
            try:
                self._sock.settimeout(timeout)
                self.bytes_sent += _send_msg(self._sock, req)
                got = [0]
                resp = _recv_msg(self._sock, got)
                self.bytes_received += got[0]
            except (OSError, ConnectionError, struct.error):
                # a timed-out / broken exchange leaves the stream out of step (the late reply would be read as the
                # answer to the next request): the handle is dead from here on
                try:
                    self._sock.close()
                finally:
                    self._sock = None
                raise
        if check and not resp.get("ok", False):
            raise RuntimeError(f"worker {self.id}: {resp.get('error')}")
        return resp

    def ping(self) -> bool:
        return bool(self._call({"op": "ping"}, timeout=5.0).get("ok"))

    def fit(self, flat: torch.Tensor, cfg: FitConfig, dataset_key: str = "training",
            timeout: Optional[float] = None, version: Optional[int] = None) -> Tuple[torch.Tensor, float, int]:
        """Broadcast leg + remote local-SGD + gather leg (cf.py:209-211) in one RPC: the trained fp32 model (unchecked), the
        loss and the sample count.  ``version`` as in :meth:`fit_update`."""
        update, loss, n = self.fit_update(flat, cfg, UplinkCodec(), version=version, dataset_key=dataset_key, timeout=timeout)
        return update["params"], loss, n

    def fit_update(self, flat: torch.Tensor, cfg: FitConfig, codec: UplinkCodec, *, ef_reset: bool = False,
                   secagg: Optional[Dict[str, Any]] = None, downlink: Optional[Dict[str, Any]] = None, version: Optional[int] = None,
                   dataset_key: str = "training", timeout: Optional[float] = None) -> Tuple[Dict[str, Any], float, int]:
        """One fit RPC from ``flat``: the reply's update fields unchecked (untrusted input: the coordinator checks them; an fp32
        model is decoded to a tensor), the loss and the sample count.  ``codec``: the update's format (topk: ``ef_reset`` zeroes
        the device's residual first); ``secagg``: the round's ``{"tag", "t", "u1", "clip", "frac_bits"}``, for a masked delta;
        ``downlink``: :meth:`Coordinator._downlink_fields`, which from round 1 on replace ``flat`` by a wire to the device's
        replica and add ``replica_crc`` to the update; ``version``: the global version of ``flat`` under asynchronous
        aggregation (the device echoes it; None sends no version field)."""
        req: Dict[str, Any] = {"op": "fit", "config": cfg.to_dict()}
        if downlink is None or "replica_base" not in downlink:
            req["params"] = _to_bytes(flat)
        req["dataset_key"] = dataset_key
        req.update(request_fields(codec, ef_reset))
        if secagg is not None:
            req["secagg"] = secagg
        if version is not None:
            req["version"] = int(version)
        resp = self._call({**req, **(downlink or {})}, timeout=timeout)
        self.last_buffers = _from_bytes(resp["buffers"]) if resp.get("buffers") else None     # BatchNorm statistics, if any
        if secagg is not None:
            update = {k: resp.get(k) for k in ("secagg", "masked", "clipped", "nonfinite")}
        elif codec.kind == "fp32":
            update = {"params": _from_bytes(resp["params"])}
        else:
            update = {k: resp.get(k) for k in (*echo(codec), *FIELDS[codec.kind])}
        if downlink is not None:
            update["replica_crc"] = resp.get("replica_crc")
        return update, float(resp["loss"]), int(resp["n"])

    def secagg_setup(self, tag: str, timeout: Optional[float] = None) -> Any:
        """The device's public key for the training ``tag`` (unchecked bytes)"""
        return self._call({"op": "secagg_setup", "tag": tag}, timeout=timeout).get("pk")

    def secagg_peers(self, tag: str, ids: List[str], pks: List[bytes], timeout: Optional[float] = None) -> None:
        """The training's key list in setup order: the device derives its pair seeds"""
        self._call({"op": "secagg_setup", "tag": tag, "ids": ids, "pks": pks}, timeout=timeout)

    def secagg_unmask(self, tag: str, t: int, survivors: List[str], timeout: Optional[float] = None) -> Dict[str, Any]:
        """Round ``t``'s seeds for the survivor list: the reply ``{"self_seed", "pair_seeds"}`` unchecked"""
        resp = self._call({"op": "secagg_unmask", "tag": tag, "t": t, "u2": survivors}, timeout=timeout)
        return {k: resp.get(k) for k in ("self_seed", "pair_seeds")}

    def evaluate(self, flat: torch.Tensor, model_name: str, bins: int, threshold: float, timeout: Optional[float] = None) -> Dict[str, Any]:
        """Federated evaluation of the fp32 model ``flat``: the device's reply as it came (``ok: False`` with ``eval_missing``
        when it holds no evaluation data); ``fl.fedeval.from_wire`` checks it."""
        return self._call({"op": "evaluate", "params": _to_bytes(flat.float()), "model": model_name, "bins": int(bins),
                           "threshold": float(threshold)}, timeout=timeout, check=False)

    def search(self, tag: str) -> int:
        return int(self._call({"op": "search", "tag": tag}).get("count", 0))

    def predict(self, flat: torch.Tensor, model_name: str, tag: str = "inference", alarm: Optional[Dict[str, Any]] = None) -> List[int]:
        """The device's predictions on its ``tag`` rows; an autoencoder needs ``alarm`` (``alarm_bin`` and ``bins`` of the
        checkpoint's federated threshold) and returns 0 / 1 alarms"""
        req = {"op": "predict", "params": _to_bytes(flat), "model": model_name, "tag": tag}
        if alarm is not None:
            req.update(alarm_bin=int(alarm["alarm_bin"]), bins=int(alarm["bins"]))
        return list(self._call(req)["pred"])

    def close(self) -> None:
        with self._lock:
            if self._sock is None:
                return
            try:
                _send_msg(self._sock, {"op": "close"})
                _recv_msg(self._sock)
            except (OSError, ConnectionError, struct.error):
                pass
            try:
                self._sock.close()
            finally:
                self._sock = None

    def __repr__(self) -> str:
        return f"<RemoteWorkerClient id:{self.id}>"
