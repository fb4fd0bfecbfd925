"""Uplink compression of the client updates: what a client sends back after a fit instead of its fp32 model.

A client that received the global model ``theta`` and trained it into ``theta_k`` sends its delta ``d = theta_k - theta``,
either stochastically quantized (QSGD, Alistarh et al., NeurIPS 2017; FedPAQ, Reisizadeh et al., AISTATS 2020) as ``int8``
(or ``int4``) codes with one float32 scale per block of 256 elements, or sparsified to its ``k`` largest entries per block
with error feedback (``topk``; EF-SGD, Seide et al. 2014, Stich et al. 2018, Karimireddy et al. 2019):

====  ======  ======================================  =======================
kind  levels  payload bytes for P parameters          ratio to fp32 (large P)
====  ======  ======================================  =======================
fp32  --      4 P (the model itself)                  1
int8  127     P + 4 ceil(P / 256)                     ~3.9
int4  7       ceil(P / 2) + 4 ceil(P / 256)           ~7.5
topk  --      5 E, E = k (nblk - 1) + min(k, m_last)  ~205 / k (~25 at k = 8)
====  ======  ======================================  =======================

int8 / int4: per block, ``step = max |d_j| / L``; element ``j`` is rounded up or down to a multiple of ``step`` with the
probability that makes the decoded value ``q_j step`` an unbiased estimate of ``d_j`` (``|q_j step - d_j| <= step``).  The
rounding noise is keyed by :func:`uplink_key` (the device's id and the fit's seed): two devices never share it and a rerun
reproduces a round.  The arithmetic is defined once in ``ops/csrc/uplink_quant.cuh``; ``ops.reference.encode_delta`` /
``decode_delta`` transcribe it.

topk: the device adds the residual ``e`` it carries over from its earlier fits (zero at the start of a training) to its
delta, ``v = d + e``, sends the ``k`` entries of largest ``|v|`` of every 256-element block (``nblk`` blocks, the last one
``m_last`` long) as a uint8 offset and the fp32 value ``v_j`` each, and keeps the rest as its new residual: nothing is
dropped, only delayed.  The selection is deterministic (ties go to the lower index, NaN / Inf are always sent), so there
are no scales and no keys.  Defined in ``ops/csrc/uplink_topk.cuh``; ``ops.reference.encode_topk_delta`` /
``decode_topk_delta`` transcribe it.  The residuals live in memory only, like the server optimizer state.

The coordinator decodes against the model it sent.

Downlink: the same codecs compress what the coordinator sends.  Coordinator and devices keep a replica ``r`` of the model
the devices hold; round 0 of a training sends the global model as fp32 (``r = theta``), every later round encodes ``theta -
r`` once (int8 / int4 rounded with :func:`downlink_key`, or its top-k entries), broadcasts the same bytes to every device, and
both sides advance ``r`` by what was sent, bit for bit alike.  Devices train from ``r`` and send their deltas to ``r``; what
was not delivered yet stays in ``theta - r`` and goes out in later rounds.  Defined in ``ops/csrc/downlink.cuh``;
``ops.reference.encode_downlink`` / ``apply_downlink`` transcribe it.

Each format's wire is defined here alone: the request fields (:func:`request_fields`, :func:`echo`), the update fields
(:data:`FIELDS`), the device's encode (:func:`device_reply`, :func:`encode`), the coordinator's reply check
(:func:`check_reply`) and its server step over K checked replies (:func:`stack`, :func:`server_apply`).
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import Any, ClassVar, Dict, List, Optional, Sequence

import numpy as np
import torch

KINDS = {"fp32": 32, "int8": 8, "int4": 4, "topk": 32}    # bits of one value on the wire
LEVELS = {"fp32": 0, "int8": 127, "int4": 7, "topk": 0}
TOPK_MAX = 32                     # entries per 256-element block: one per lane of the warp that owns the block


def uplink_key(worker_id: str, seed: int) -> int:
    """The uint32 key of a device's rounding noise for one fit."""
    return zlib.crc32(f"{worker_id}:{int(seed)}".encode())


def downlink_key(seed: int) -> int:
    """The uint32 key of the downlink's rounding noise for the round of ``seed``: one broadcast, so every device shares it."""
    return zlib.crc32(f"downlink:{int(seed)}".encode())


@dataclass(frozen=True)
class UplinkCodec:
    """What a device sends back after a fit: its fp32 model (``fp32``), its quantized delta (``int8`` / ``int4``), or the
    ``k`` largest entries per block of its delta plus residual (``topk``, ``k`` in 1..32; ``k`` is ignored by the other kinds)."""
    kind: str = "fp32"
    k: int = 8
    BLOCK: ClassVar[int] = 256

    def __post_init__(self) -> None:
        if self.kind not in KINDS:
            raise ValueError(f"unknown uplink codec {self.kind!r}; expected one of {', '.join(KINDS)}")
        if self.kind == "topk" and not (isinstance(self.k, int) and not isinstance(self.k, bool) and 1 <= self.k <= TOPK_MAX):
            raise ValueError(f"topk keeps 1..{TOPK_MAX} entries per block of {self.BLOCK}, not {self.k!r}")

    @property
    def bits(self) -> int:
        return KINDS[self.kind]

    @property
    def levels(self) -> int:
        """L: the codes lie in [-L, L] (0 for fp32)."""
        return LEVELS[self.kind]

    @property
    def quantized(self) -> bool:
        """int8 / int4: the stochastic codec (payload + scales)."""
        return self.kind in ("int8", "int4")

    @property
    def sparse(self) -> bool:
        """topk: (offset, value) entries with error feedback."""
        return self.kind == "topk"

    def entries(self, p: int) -> int:
        """topk: entries of ``p`` parameters, ``k (nblk - 1) + min(k, m_last)`` (0 for the other kinds)."""
        if not self.sparse:
            return 0
        nblk = math.ceil(p / self.BLOCK)
        return self.k * (nblk - 1) + min(self.k, p - (nblk - 1) * self.BLOCK)

    def payload_bytes(self, p: int) -> int:
        """Bytes of the codes of ``p`` parameters on the wire (fp32: the model itself; topk: 1-byte offsets and fp32 values)."""
        if self.kind == "fp32":
            return 4 * p
        if self.sparse:
            return 5 * self.entries(p)
        return p if self.kind == "int8" else (p + 1) // 2

    def scale_count(self, p: int) -> int:
        """Number of float32 block scales (0 for fp32 and topk)."""
        return math.ceil(p / self.BLOCK) if self.quantized else 0

    @property
    def max_scale(self) -> float:
        """The largest float32 ``step`` whose product with ``L`` is finite in float32 (``FLT_MAX / L``, one ulp below where
        the division rounds up): no decoded value ``q step`` (``|q| <= L``) can overflow.  The coordinator refuses any larger
        (or non-finite) scale; an encoder only exceeds it for a block whose largest delta is within an ulp of ``FLT_MAX``."""
        if not self.quantized:
            return math.inf
        L = np.float32(self.levels)
        x = np.float32(np.finfo(np.float32).max) / L
        with np.errstate(over="ignore"):
            while not np.isfinite(L * x):
                x = np.nextafter(x, np.float32(0.0))
        return float(x)


# ---- the wire of each format ------------------------------------------------------------------------------------------------------
# the update fields of a reply, in wire order; the compressed downlink sends its wire under the same names with a "d" prefix
FIELDS = {"fp32": ("params",), "int8": ("payload", "scales"), "int4": ("payload", "scales"), "topk": ("indices", "values")}


def echo(codec: UplinkCodec) -> Dict[str, Any]:
    """The fields that name the format: a fit request carries them and the device's reply echoes them (none for fp32)"""
    if codec.kind == "fp32":
        return {}
    return {"uplink": codec.kind, "topk": codec.k} if codec.sparse else {"uplink": codec.kind}


def request_fields(codec: UplinkCodec, ef_reset: bool = False) -> Dict[str, Any]:
    """The uplink fields of a fit request: :func:`echo`, and for topk whether the device zeroes its residual first"""
    return {**echo(codec), "ef_reset": bool(ef_reset)} if codec.sparse else echo(codec)


def wire_fields(codec: UplinkCodec, wire: Sequence[torch.Tensor], prefix: str = "") -> Dict[str, bytes]:
    """The wire tensors of one update (or of the downlink, ``prefix`` "d") as the fields of :data:`FIELDS`"""
    return {prefix + name: t.detach().cpu().contiguous().numpy().tobytes() for name, t in zip(FIELDS[codec.kind], wire)}


def encode(codec: UplinkCodec, flats: torch.Tensor, base: Optional[torch.Tensor], keys: Sequence[int],
           residual: Optional[torch.Tensor] = None):
    """The wire tensors of K trained models ``flats`` [K, P]: their deltas to ``base`` as ``(payload, scales)`` rounded with
    ``keys`` (one per row) or as ``(indices, values)`` plus ``residual`` [K, P], which keeps what was not sent; fp32 ``(flats,)``"""
    from .. import ops
    if codec.quantized:
        return ops.encode_delta(flats, base, codec, keys)
    if codec.sparse:
        return ops.encode_topk_delta(flats, base, residual, codec)
    return (flats,)


def device_reply(codec: UplinkCodec, flat: torch.Tensor, received: Optional[torch.Tensor], key: int,
                 residuals: Dict[str, torch.Tensor], model: str, ef_reset: bool) -> Dict[str, Any]:
    """A device's reply fields for ``flat`` trained from ``received``: :func:`echo` and the update.  topk keeps its residual
    [1, P] in ``residuals[model]``, zeroed on ``ef_reset`` and whenever the model's size or device changed."""
    res = None
    if codec.sparse:
        res = residuals.get(model)
        if ef_reset or res is None or res.numel() != flat.numel() or res.device != flat.device:
            res = residuals[model] = torch.zeros(1, flat.numel(), device=flat.device)
    return {**echo(codec), **wire_fields(codec, encode(codec, flat.unsqueeze(0), received, [key], res))}


def stack(updates: List[Any], codec: UplinkCodec, device) -> List[torch.Tensor]:
    """K checked replies (:func:`check_reply`) as one [K, ...] tensor per field on ``device``"""
    rows = [(u,) for u in updates] if codec.kind == "fp32" else updates
    return [torch.stack(field).to(device) for field in zip(*rows)]


def server_apply(theta: torch.Tensor, wire: Sequence[torch.Tensor], w: torch.Tensor, codec: UplinkCodec, **server):
    """One server step on ``theta`` in place from K updates, ``wire`` (:func:`encode` or :func:`stack`), weighted by ``w``:
    the fused FedAvg apply of the format; ``server`` are its aggregator and server-optimizer keywords."""
    from .. import ops
    if codec.quantized:
        return ops.fedavg_apply_quantized(theta, *wire, w, codec, **server)
    if codec.sparse:
        return ops.fedavg_apply_topk(theta, *wire, w, codec, **server)
    return ops.fedavg_apply(theta, *wire, w, **server)


# ---- checks of untrusted wire bytes: a device's reply on the coordinator, the coordinator's downlink on a device ----------------
def check_quantized_reply(update: Dict[str, Any], codec: UplinkCodec, p: int):
    """``(payload uint8 [codec.payload_bytes(p)], scales fp32 [codec.scale_count(p)])`` of a device's quantized reply, or
    ValueError.  A reply is untrusted input: it must echo the codec asked for, carry exactly the bytes the codec defines for
    ``p`` parameters, and only finite scales with ``|step| <= codec.max_scale`` (no decoded value can overflow)."""
    if update.get("uplink") != codec.kind:
        raise ValueError(f"uplink {update.get('uplink')!r} returned, {codec.kind!r} asked for")
    payload, scales = update.get("payload"), update.get("scales")
    if not isinstance(payload, bytes) or len(payload) != codec.payload_bytes(p):
        raise ValueError(f"payload of {len(payload) if isinstance(payload, bytes) else None} bytes, expected {codec.payload_bytes(p)}")
    if not isinstance(scales, bytes) or len(scales) != 4 * codec.scale_count(p):
        raise ValueError(f"{len(scales) // 4 if isinstance(scales, bytes) else None} scales, expected {codec.scale_count(p)}")
    s = torch.from_numpy(np.frombuffer(scales, dtype="<f4").copy())
    if not bool(torch.isfinite(s).all()) or float(s.abs().max()) > codec.max_scale:
        raise ValueError("non-finite or oversize block scale returned")
    return torch.from_numpy(np.frombuffer(payload, dtype=np.uint8).copy()), s


def check_topk_reply(update: Dict[str, Any], codec: UplinkCodec, p: int):
    """``(indices uint8 [codec.entries(p)], values fp32 [codec.entries(p)])`` of a device's top-k reply, or ValueError.  A
    reply is untrusted input: it must echo the codec and ``k`` asked for, carry exactly ``codec.entries(p)`` offsets and
    values, offsets strictly ascending inside each block and below the block's length (so the decode sees each coordinate
    at most once per device), and only finite values."""
    if update.get("uplink") != codec.kind or type(update.get("topk")) is not int or update.get("topk") != codec.k:
        raise ValueError(f"uplink {update.get('uplink')!r} / topk {update.get('topk')!r} returned, {codec.kind!r} / {codec.k} asked for")
    e = codec.entries(p)
    indices, values = update.get("indices"), update.get("values")
    if not isinstance(indices, bytes) or len(indices) != e:
        raise ValueError(f"{len(indices) if isinstance(indices, bytes) else None} offsets returned, expected {e}")
    if not isinstance(values, bytes) or len(values) != 4 * e:
        raise ValueError(f"{len(values) // 4 if isinstance(values, bytes) else None} values returned, expected {e}")
    idx = np.frombuffer(indices, dtype=np.uint8).astype(np.int64)
    blk = np.arange(e) // codec.k
    if (idx >= np.minimum(codec.BLOCK, p - blk * codec.BLOCK)).any():
        raise ValueError("offset past the end of its block returned")
    if ((idx[1:] <= idx[:-1]) & (blk[1:] == blk[:-1])).any():
        raise ValueError("offsets not strictly ascending inside a block returned")
    v = torch.from_numpy(np.frombuffer(values, dtype="<f4").copy())
    if not bool(torch.isfinite(v).all()):
        raise ValueError("non-finite value returned")
    return torch.from_numpy(idx.astype(np.uint8)), v


def check_reply(update: Dict[str, Any], codec: UplinkCodec, p: int):
    """The checked update of a device's reply in the format ``codec``, or ValueError: :func:`check_quantized_reply`,
    :func:`check_topk_reply`, or for fp32 the model ``update["params"]`` (as ``RemoteWorkerClient`` decodes it) as a flat
    fp32 tensor of ``p`` finite parameters: a wrong-length or non-finite model would poison (or abort) the whole average."""
    if codec.quantized:
        return check_quantized_reply(update, codec, p)
    if codec.sparse:
        return check_topk_reply(update, codec, p)
    flat = torch.as_tensor(update.get("params"), dtype=torch.float32).reshape(-1)
    if flat.numel() != p:
        raise ValueError(f"model of {flat.numel()} parameters returned, expected {p}")
    if not bool(torch.isfinite(flat).all()):
        raise ValueError("model with non-finite parameters returned")
    return flat
