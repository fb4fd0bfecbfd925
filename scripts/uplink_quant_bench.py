#!/usr/bin/env python
"""Cost and saving of the uplink codec (int8 / int4 quantized client deltas, fl/uplink.py).

    python scripts/uplink_quant_bench.py [--iters 20] [--passes 3] [--parts kernel,encode,traffic] [--out result.json]

1. Coordinator apply: ``ops.fedavg_apply`` on K fp32 client models against ``ops.fedavg_apply_quantized`` on K int8 / int4
   deltas (decode fused into the reduce), kernel time from device events around --iters back-to-back launches, median over
   --passes with the three kinds alternating inside every pass, at K in {4, 8, 16, 32, 100} for P = 4,994 (cfg2, MLP
   10-64-64-2) and P = 50,397,186 (wide MLP 10-4096x4-2).  Bytes moved, from the shapes: fp32 (K + 2) P 4 (K slots read,
   theta read and written); quantized K (codes + 4 ceil(P / 256)) + 2 P 4.  The share of 3.35 TB/s (H100 SXM data sheet
   HBM3 bandwidth) is those bytes over the kernel time.  --max-gb skips a case whose fp32 slots exceed it.
2. Encode: ``ops.encode_delta`` (quantize_delta_kernel) of K = 1 and 8 wide-MLP models, time and bytes/s (K P 4 model
   bytes + K P 4 theta bytes read, codes and scales written).
3. Remote-mode traffic: ``bytes_in`` / ``bytes_out`` per round of the FFNN (2,401 parameters) for each codec, two worker
   servers on localhost, CPU devices.  A count, not a time.

The card's name, power limit and SM clock are read (nvidia-smi, read-only queries) in the same run.  Prints one JSON document."""
import argparse
import json
import os
import socket
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
KS = (4, 8, 16, 32, 100)
SIZES = {"cfg2": 4994, "wide_mlp": 50397186}
CODECS = ("fp32", "int8", "int4")


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def _bytes(kind, K, P):
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    c = UplinkCodec(kind)
    return (K + 2) * P * 4 if kind == "fp32" else K * (c.payload_bytes(P) + 4 * c.scale_count(P)) + 2 * P * 4


def _time(fn, iters, passes_out):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    passes_out.append(e0.elapsed_time(e1) / iters)


def kernel_times(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    dev = torch.device("cuda", 0)
    rows = []
    for name, P in SIZES.items():
        for K in KS:
            gb = K * P * 4 / 1e9
            if gb > args.max_gb:
                rows.append({"model": name, "P": P, "K": K, "skipped": f"{gb:.1f} GB of fp32 slots > --max-gb"})
                continue
            g = torch.Generator(device=dev).manual_seed(K)
            theta0 = torch.randn(P, device=dev, generator=g)
            theta = theta0.clone()
            w = torch.full((K,), 1.0 / K, device=dev)
            work = {}
            slots = torch.randn(K, P, device=dev, generator=g)
            work["fp32"] = lambda: ops.fedavg_apply(theta, slots, w)
            for kind in ("int8", "int4"):
                c = UplinkCodec(kind)
                row = (c.payload_bytes(P) + 15) // 16 * 16
                payload = torch.randint(0, 256, (K, row), device=dev, dtype=torch.uint8, generator=g)
                scales = torch.rand(K, c.scale_count(P), device=dev, generator=g) * 1e-3
                work[kind] = (lambda p=payload, s=scales, c=c: ops.fedavg_apply_quantized(theta, p, s, w, c))
            for fn in work.values():
                fn()                                                           # warm-up (module load)
            per = {k: [] for k in work}
            for _ in range(args.passes):
                for kind, fn in work.items():                                  # kinds alternate inside every pass
                    theta.copy_(theta0)
                    _time(fn, args.iters, per[kind])
            rec = {"model": name, "P": P, "K": K, "iters": args.iters, "bytes": {}, "ms": {}, "hbm_share": {}}
            for kind in work:
                ms = statistics.median(per[kind])
                rec["bytes"][kind] = _bytes(kind, K, P)
                rec["ms"][kind] = round(ms, 5)
                rec["hbm_share"][kind] = round(rec["bytes"][kind] / (ms * 1e-3) / HBM_BYTES_PER_S, 4)
            rec["speedup_vs_fp32"] = {k: round(rec["ms"]["fp32"] / rec["ms"][k], 3) for k in ("int8", "int4")}
            rec["byte_ratio_vs_fp32"] = {k: round(rec["bytes"]["fp32"] / rec["bytes"][k], 3) for k in ("int8", "int4")}
            rows.append(rec)
            del slots, work, theta, theta0
            torch.cuda.empty_cache()
    return rows


def encode_times(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    dev = torch.device("cuda", 0)
    P = SIZES["wide_mlp"]
    rows = []
    for K in (1, 8):
        g = torch.Generator(device=dev).manual_seed(K)
        theta = torch.randn(P, device=dev, generator=g)
        models = theta + 0.01 * torch.randn(K, P, device=dev, generator=g)
        for kind in ("int8", "int4"):
            c = UplinkCodec(kind)
            keys = list(range(K))
            ops.encode_delta(models, theta, c, keys)
            per = []
            for _ in range(args.passes):
                _time(lambda: ops.encode_delta(models, theta, c, keys), args.iters, per)
            ms = statistics.median(per)
            nbytes = 2 * K * P * 4 + K * (c.payload_bytes(P) + 4 * c.scale_count(P))
            rows.append({"model": "wide_mlp", "P": P, "K": K, "codec": kind, "ms": round(ms, 5), "bytes": nbytes,
                         "hbm_share": round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 4)})
        del models, theta
        torch.cuda.empty_cache()
    return rows


def _free_port() -> int:
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def remote_traffic(args) -> dict:
    import torch

    from colearn_federated_learning_b200 import settings
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw
    cpu = torch.device("cpu")
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for kind in CODECS:
            workers = []
            for seed in (1, 2):
                port = _free_port()
                w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=cpu)
                w.add_dataset(BaseDataset(*synthetic_unsw(256, seed=seed)))
                w.start(block=False)
                workers.append((w, port))
            try:
                a = Arguments(model="ffnn", lr=0.05, federate_after_n_batches=50, uplink=kind, synthetic=64)
                broker, clock = InProcessBroker(), FakeClock()
                c = Coordinator(1, True, 3, False, False, args=a, broker=broker, timer_factory=clock, path=os.path.join(d, f"{kind}.pth"),
                                device=cpu, evaluate_after=False)
                c.connect()
                c.subscribe("topic/state")
                pub = BusClient("pub", broker=broker)
                pub.connect()
                for _, port in workers:
                    pub.publish("topic/state", f"(127.0.0.1, {port}, TRAINING)")
                c.drain()
                clock.advance(1.0)
                recs = [r for r in c.metrics.records if "bytes_in" in r]
                out[kind] = {"bytes_in_per_round": [r["bytes_in"] for r in recs], "bytes_out_per_round": [r["bytes_out"] for r in recs],
                             "bytes_in_per_device_and_round": recs[0]["bytes_in"] / 2}
            finally:
                for w, _ in workers:
                    w.stop()
                settings.training_devices.clear()
    for kind in ("int8", "int4"):
        out[kind]["bytes_in_ratio_vs_fp32"] = round(out["fp32"]["bytes_in_per_round"][0] / out[kind]["bytes_in_per_round"][0], 3)
    return {"description": "remote mode, FFNN (2,401 parameters), 2 devices on localhost, 3 rounds", **out}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--max-gb", type=float, default=24.0)
    ap.add_argument("--parts", default="kernel,encode,traffic")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    parts = args.parts.split(",")
    result = {}
    if "kernel" in parts or "encode" in parts:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("uplink_quant_bench.py measures the kernels on a GPU; none is visible (--parts traffic counts bytes on CPU)")
        result["gpu"] = gpu_info()
        result["hbm_bytes_per_s_datasheet"] = HBM_BYTES_PER_S
    if "kernel" in parts:
        result["fedavg_apply"] = kernel_times(args)
    if "encode" in parts:
        result["encode_delta"] = encode_times(args)
    if "traffic" in parts:
        result["remote_traffic"] = remote_traffic(args)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
