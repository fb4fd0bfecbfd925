"""Tracing / profiling hooks (SURVEY §5 "Tracing / profiling").

The reference profiles out-of-band with psutil scripts attached to the coordinator's PID
(``data/ps_util_test.py``; PID logged at fc.py:605).  Here: NVTX ranges around the phases of a
round (visible in Nsight tools), a CUDA-event phase timer for device-side timing without a
profiler, and helpers for profiling runs.
"""
from __future__ import annotations

import contextlib
import os
import time
from collections import defaultdict
from typing import Dict, Iterator, List, Optional

import torch

_ENABLED = os.environ.get("COLEARN_NVTX", "0") == "1"


@contextlib.contextmanager
def nvtx_range(name: str) -> Iterator[None]:
    """NVTX range when ``COLEARN_NVTX=1`` and CUDA is present; free otherwise."""
    if _ENABLED and torch.cuda.is_available():
        torch.cuda.nvtx.range_push(name)
        try:
            yield
        finally:
            torch.cuda.nvtx.range_pop()
    else:
        yield


class PhaseTimer:
    """Accumulates per-phase time.  CUDA: event pairs on the current stream (resolved lazily at
    :meth:`summary`, so no sync is inserted into the measured region); CPU: ``perf_counter``."""

    def __init__(self, device: Optional[torch.device] = None) -> None:
        self.cuda = device is not None and torch.device(device).type == "cuda"
        self._events: Dict[str, List] = defaultdict(list)
        self._cpu: Dict[str, float] = defaultdict(float)

    @contextlib.contextmanager
    def phase(self, name: str) -> Iterator[None]:
        with nvtx_range(name):
            if self.cuda:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                try:
                    yield
                finally:
                    e1.record()
                    self._events[name].append((e0, e1))
            else:
                t0 = time.perf_counter()
                try:
                    yield
                finally:
                    self._cpu[name] += (time.perf_counter() - t0) * 1e3

    def summary(self) -> Dict[str, float]:
        out = dict(self._cpu)
        if self.cuda:
            torch.cuda.synchronize()
            for name, pairs in self._events.items():
                out[name] = out.get(name, 0.0) + sum(a.elapsed_time(b) for a, b in pairs)
        return out
