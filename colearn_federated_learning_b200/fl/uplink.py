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

The coordinator decodes against the ``theta`` it sent; the downlink stays fp32.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import ClassVar

import numpy as np

KINDS = {"fp32": 32, "int8": 8, "int4": 4, "topk": 32}    # bits of one value on the wire
LEVELS = {"fp32": 0, "int8": 127, "int4": 7, "topk": 0}
TOPK_MAX = 32                     # entries per 256-element block: one per lane of the warp that owns the block


def uplink_key(worker_id: str, seed: int) -> int:
    """The uint32 key of a device's rounding noise for one fit."""
    return zlib.crc32(f"{worker_id}:{int(seed)}".encode())


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
