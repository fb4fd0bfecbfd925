"""Uplink compression of the client updates: unbiased stochastic quantization of the delta a client sends back (QSGD,
Alistarh et al., NeurIPS 2017; FedPAQ, Reisizadeh et al., AISTATS 2020).

A client that received the global model ``theta`` and trained it into ``theta_k`` sends ``d = theta_k - theta`` as
``int8`` (or ``int4``) codes with one float32 scale per block of 256 elements instead of its fp32 model:

=====  ======  ==============================  =========================
kind   levels  payload bytes for P parameters  ratio to fp32 (large P)
=====  ======  ==============================  =========================
fp32   --      4 P (the model itself)          1
int8   127     P + 4 ceil(P / 256)             ~3.9
int4   7       ceil(P / 2) + 4 ceil(P / 256)   ~7.5
=====  ======  ==============================  =========================

Per block, ``step = max |d_j| / L``; element ``j`` is rounded up or down to a multiple of ``step`` with the probability
that makes the decoded value ``q_j step`` an unbiased estimate of ``d_j`` (``|q_j step - d_j| <= step``).  The rounding
noise is keyed by :func:`uplink_key` (the device's id and the fit's seed): two devices never share it and a rerun
reproduces a round.  The coordinator decodes against the ``theta`` it sent; the downlink stays fp32.  The arithmetic is
defined once in ``ops/csrc/uplink_quant.cuh``; ``ops.reference.encode_delta`` / ``decode_delta`` transcribe it.
"""
from __future__ import annotations

import math
import zlib
from dataclasses import dataclass
from typing import ClassVar

import numpy as np

KINDS = {"fp32": 32, "int8": 8, "int4": 4}
LEVELS = {"fp32": 0, "int8": 127, "int4": 7}


def uplink_key(worker_id: str, seed: int) -> int:
    """The uint32 key of a device's rounding noise for one fit."""
    return zlib.crc32(f"{worker_id}:{int(seed)}".encode())


@dataclass(frozen=True)
class UplinkCodec:
    """What a device sends back after a fit: its fp32 model (``fp32``), or its quantized delta (``int8`` / ``int4``)."""
    kind: str = "fp32"
    BLOCK: ClassVar[int] = 256

    def __post_init__(self) -> None:
        if self.kind not in KINDS:
            raise ValueError(f"unknown uplink codec {self.kind!r}; expected one of {', '.join(KINDS)}")

    @property
    def bits(self) -> int:
        return KINDS[self.kind]

    @property
    def levels(self) -> int:
        """L: the codes lie in [-L, L] (0 for fp32)."""
        return LEVELS[self.kind]

    @property
    def quantized(self) -> bool:
        return self.kind != "fp32"

    def payload_bytes(self, p: int) -> int:
        """Bytes of the codes of ``p`` parameters on the wire (fp32: the model itself)."""
        if self.kind == "fp32":
            return 4 * p
        return p if self.kind == "int8" else (p + 1) // 2

    def scale_count(self, p: int) -> int:
        """Number of float32 block scales (0 for fp32)."""
        return 0 if self.kind == "fp32" else math.ceil(p / self.BLOCK)

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
