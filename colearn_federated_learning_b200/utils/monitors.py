"""Resource monitors (reference ``data/ps_util_test.py``, ``data/temperature_test.py``; SURVEY C31)
plus the GPU analogue: an NVML sampler (SM clock, power, temperature, throttle reasons) used by
``bench.py`` to record clocks *during* the timed region.

File formats are the reference's (``Monitoring: <i> <timestamp>`` blocks, SURVEY §2.7) so the
published ``data/`` logs and new logs can be post-processed by the same scripts.  The network
monitor zero-bases ``pkts_rcv`` with ``packets_recv`` (the reference uses ``packets_sent``,
SURVEY §2.8-11).
"""
from __future__ import annotations

import argparse
import logging
import statistics
import threading
import time
from datetime import datetime
from typing import Any, Dict, List, Optional

import psutil

log = logging.getLogger(__name__)


def bytes2human(n: float) -> str:
    symbols = ("K", "M", "G", "T", "P")
    for i, s in reversed(list(enumerate(symbols))):
        unit = 1 << ((i + 1) * 10)
        if abs(n) >= unit:
            return "%.1f%s" % (n / unit, s)
    return "%sB" % int(n)


def monitor_cpu(pid: int, path: str = "monitoring_cpu.txt", samples: int = 3000, interval: float = 1.0,
                stop: Optional[threading.Event] = None) -> None:
    p = psutil.Process(pid)
    with open(path, "w+") as f:
        f.write(str(p) + "\n")
        for i in range(samples):
            if stop is not None and stop.is_set():
                break
            f.write("Monitoring: " + str(i) + " " + str(datetime.now()) + "\n")
            f.write(str(p.cpu_times()) + "\n")
            f.write(str(p.cpu_percent(interval=interval)) + "\n")
            f.flush()


def monitor_network(interface: str, path: str = "monitoring_network.txt", samples: int = 3000,
                    interval: float = 1.0, stop: Optional[threading.Event] = None) -> None:
    base = None
    with open(path, "w+") as f:
        for i in range(samples):
            if stop is not None and stop.is_set():
                break
            io_all = psutil.net_io_counters(pernic=True)
            if interface not in psutil.net_if_stats() or interface not in io_all:
                log.info("Interface not valid")
                break
            io = io_all[interface]
            if base is None:
                base = io  # zero-base every counter at the first sample
            f.write("Monitoring: " + str(i) + " " + str(datetime.now()) + "\n")
            f.write("    incoming       : bytes=%s, pkts=%s, errs=%s, drops=%s\n" % (
                bytes2human(io.bytes_recv - base.bytes_recv), io.packets_recv - base.packets_recv,
                io.errin - base.errin, io.dropin - base.dropin))
            f.write("    outgoing       : bytes=%s, pkts=%s, errs=%s, drops=%s\n\n" % (
                bytes2human(io.bytes_sent - base.bytes_sent), io.packets_sent - base.packets_sent,
                io.errout - base.errout, io.dropout - base.dropout))
            f.flush()
            time.sleep(interval)


def monitor_temperature(path: str = "monitoring_temp.txt", interval: float = 1.0,
                        stop: Optional[threading.Event] = None, samples: Optional[int] = None) -> None:
    i = 0
    with open(path, "w+") as f:
        while (stop is None or not stop.is_set()) and (samples is None or i < samples):
            f.write("Monitoring: " + str(i) + " : " + str(datetime.now()) + "\n")
            temps = psutil.sensors_temperatures() if hasattr(psutil, "sensors_temperatures") else {}
            f.write(str(temps) + "\n")
            f.flush()
            time.sleep(interval)
            i += 1


THROTTLE_BITS = {  # nvmlClocksEventReasons
    0x1: "gpu_idle", 0x2: "applications_clocks_setting", 0x4: "sw_power_cap", 0x8: "hw_slowdown",
    0x10: "sync_boost", 0x20: "sw_thermal_slowdown", 0x40: "hw_thermal_slowdown", 0x80: "hw_power_brake_slowdown",
    0x100: "display_clock_setting",
}
BAD_REASONS = {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}


class NvmlSampler:
    """Background sampler of SM clock / power / temperature / throttle reasons for one GPU."""

    def __init__(self, index: int = 0, period_s: float = 0.05) -> None:
        self.index, self.period = index, period_s
        self.samples: List[Dict[str, Any]] = []
        self._stop = threading.Event()
        self._thread: Optional[threading.Thread] = None
        self._ok = False
        try:
            import pynvml
            pynvml.nvmlInit()
            self._nv = pynvml
            self._h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self._ok = True
        except Exception as e:  # noqa: BLE001 - no NVML on CPU boxes
            self._err = repr(e)

    def _loop(self) -> None:
        nv = self._nv
        while not self._stop.is_set():
            try:
                reasons = nv.nvmlDeviceGetCurrentClocksEventReasons(self._h) if hasattr(nv, "nvmlDeviceGetCurrentClocksEventReasons") \
                    else nv.nvmlDeviceGetCurrentClocksThrottleReasons(self._h)
                self.samples.append({
                    "t": time.time(),
                    "sm_mhz": nv.nvmlDeviceGetClockInfo(self._h, nv.NVML_CLOCK_SM),
                    "power_w": nv.nvmlDeviceGetPowerUsage(self._h) / 1000.0,
                    "temp_c": nv.nvmlDeviceGetTemperature(self._h, nv.NVML_TEMPERATURE_GPU),
                    "reasons": int(reasons),
                })
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(self.period)

    def start(self) -> "NvmlSampler":
        if self._ok:
            self._thread = threading.Thread(target=self._loop, name="nvml-sampler", daemon=True)
            self._thread.start()
        return self

    def stop(self) -> Dict[str, Any]:
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=2)
        return self.summary()

    def summary(self) -> Dict[str, Any]:
        if not self._ok:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "note": "nvml unavailable"}
        try:
            sm_max = self._nv.nvmlDeviceGetMaxClockInfo(self._h, self._nv.NVML_CLOCK_SM)
        except Exception:  # noqa: BLE001
            sm_max = None
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": sm_max, "reasons": [], "samples": 0}
        bits = 0
        for s in self.samples:
            bits |= s["reasons"]
        reasons = sorted(name for b, name in THROTTLE_BITS.items() if bits & b and name != "gpu_idle")
        return {"sm_mhz": statistics.median(s["sm_mhz"] for s in self.samples), "sm_max_mhz": sm_max,
                "reasons": reasons, "samples": len(self.samples),
                "power_w_max": max(s["power_w"] for s in self.samples),
                "temp_c_max": max(s["temp_c"] for s in self.samples),
                "bad": sorted(BAD_REASONS & set(reasons))}


class NvlinkCounters:
    """Cumulative NVLink payload bytes sent / received by one GPU, summed over its links (NVML field values
    ``NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX / RX``, KiB).  The difference of two ``read()`` calls around a loop of kernel
    launches is the hardware's own count of what crossed the links — the evidence for the fused collectives that ncu cannot
    give (its kernel replay cannot save / restore peer-mapped and multicast memory).  ``uuid`` selects the device the way
    torch names it, so CUDA_VISIBLE_DEVICES does not shift the index."""

    ALL_LINKS = 0xFFFFFFFF

    def __init__(self, index: int = 0, uuid: Optional[str] = None) -> None:
        self.ok, self.err = False, None
        try:
            import pynvml
            pynvml.nvmlInit()
            self._nv = pynvml
            self._h = None
            if uuid:
                u = str(uuid)
                try:
                    self._h = pynvml.nvmlDeviceGetHandleByUUID(u if u.startswith("GPU-") else "GPU-" + u)
                except Exception:  # noqa: BLE001 - unknown spelling of the UUID: fall back to the index
                    self._h = None
            if self._h is None:
                self._h = pynvml.nvmlDeviceGetHandleByIndex(index)
            self.ok = self.read() is not None
        except Exception as e:  # noqa: BLE001 - no NVML / no NVLink on this box
            self.err = repr(e)

    def read(self) -> Optional[Dict[str, int]]:
        """{"tx_bytes", "rx_bytes"} (payload, cumulative since driver load) or None when the driver does not report them."""
        nv = self._nv
        try:
            vals = nv.nvmlDeviceGetFieldValues(self._h, [(nv.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX, self.ALL_LINKS),
                                                         (nv.NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX, self.ALL_LINKS)])
        except Exception as e:  # noqa: BLE001
            self.err = repr(e)
            return None
        out = {}
        for name, v in zip(("tx_bytes", "rx_bytes"), vals):
            if v.nvmlReturn != 0:
                self.err = "nvmlReturn %d for field %d" % (v.nvmlReturn, v.fieldId)
                return None
            out[name] = int(v.value.ullVal) * 1024
        return out

    @staticmethod
    def delta(a: Optional[Dict[str, int]], b: Optional[Dict[str, int]]) -> Optional[Dict[str, int]]:
        if a is None or b is None:
            return None
        return {k: b[k] - a[k] for k in a}


def monitor_gpu(index: int = 0, path: str = "monitoring_gpu.txt", samples: int = 3000, interval: float = 1.0,
                stop: Optional[threading.Event] = None) -> None:
    """GPU analogue of :func:`monitor_cpu`: one ``Monitoring: <i> <timestamp>`` block per sample with SM clock,
    power, temperature and the active throttle reasons (NVML)."""
    sampler = NvmlSampler(index, period_s=interval)
    with open(path, "w+") as f:
        if not sampler._ok:
            f.write("nvml unavailable\n")
            return
        nv, h = sampler._nv, sampler._h
        for i in range(samples):
            if stop is not None and stop.is_set():
                break
            try:
                reasons = nv.nvmlDeviceGetCurrentClocksEventReasons(h) if hasattr(nv, "nvmlDeviceGetCurrentClocksEventReasons") \
                    else nv.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                names = sorted(n for b, n in THROTTLE_BITS.items() if int(reasons) & b)
                f.write("Monitoring: " + str(i) + " " + str(datetime.now()) + "\n")
                f.write("    sm_mhz=%s power_w=%.1f temp_c=%s reasons=%s\n" % (
                    nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM), nv.nvmlDeviceGetPowerUsage(h) / 1000.0,
                    nv.nvmlDeviceGetTemperature(h, nv.NVML_TEMPERATURE_GPU), ",".join(names) or "none"))
                f.flush()
            except Exception as e:  # noqa: BLE001
                f.write("nvml error: %r\n" % (e,))
                break
            time.sleep(interval)


def build_parser() -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser(description="Process monitoring")
    parser.add_argument("--pid", "-p", type=int, default=None, help="process pid to monitor")
    parser.add_argument("--network", "-n", type=str, default=None, help="Start monitor a network interface")
    parser.add_argument("--temperature", "-T", action="store_true", help="also sample temperatures")
    parser.add_argument("--gpu", "-g", type=int, default=None, help="also sample this GPU through NVML")
    parser.add_argument("--samples", type=int, default=3000)
    return parser


def main(argv=None) -> None:
    args = build_parser().parse_args(argv)
    logging.basicConfig(format="%(asctime)s: %(message)s", level=logging.INFO, datefmt="%H:%M:%S")
    threads = []
    if args.pid is not None:
        logging.info("Starting CPU monitor thread")
        threads.append(threading.Thread(target=monitor_cpu, args=(args.pid,), kwargs={"samples": args.samples}))
    if args.network is not None:
        logging.info("Starting network monitoring")
        threads.append(threading.Thread(target=monitor_network, args=(args.network,), kwargs={"samples": args.samples}))
    if args.temperature:
        threads.append(threading.Thread(target=monitor_temperature, kwargs={"samples": args.samples}))
    if args.gpu is not None:
        threads.append(threading.Thread(target=monitor_gpu, args=(args.gpu,), kwargs={"samples": args.samples}))
    for t in threads:
        t.start()
    logging.info("Waiting for the threads ending")
    for t in threads:
        t.join()
    logging.info("Join complete")


if __name__ == "__main__":
    main()
