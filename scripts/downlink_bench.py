#!/usr/bin/env python
"""Cost of the compressed downlink (fl/uplink.py, ops/csrc/downlink.cuh) on the GPU.

    python scripts/downlink_bench.py [--iters 50] [--passes 5] [--out result.json]

1. Coordinator encode-and-advance: ``ops.encode_downlink`` (downlink_quant_kernel for int8 / int4, downlink_topk_kernel for
   topk at k in {1, 8, 32}) of theta - replica, once per round for every device.
2. Device apply: ``ops.apply_downlink`` (replica_apply_q_kernel / replica_apply_topk_kernel) of the same wires.
At P = 4,994 (cfg2, MLP 10-64-64-2) and P = 50,397,186 (wide MLP 10-4096x4-2).  Kernel time from device events around
--iters back-to-back launches, median over --passes, every kind alternating inside every pass; the replica is reset before
each timed window (the kernels' work does not depend on the values: a block always sends k entries or 256 codes).  Bytes
moved, from the shapes: encode int8 / int4 12 P (theta and replica read, replica written) + the codes + 4 ceil(P / 256) of
scales; encode topk 8 P + 5 E (entries written) + 4 E (the sent replica elements written); apply int8 / int4 8 P (replica
read and written) + codes + scales; apply topk 5 E + 8 E.  The share of 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth) is
those bytes over the kernel time.  The card's name, power limit and SM clock are read (nvidia-smi, read-only queries) in
the same run.  Prints one JSON document."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
SIZES = {"cfg2": 4994, "wide_mlp": 50397186}


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def _time(fn, iters, passes_out):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    passes_out.append(e0.elapsed_time(e1) / iters)


def _bytes(codec, P, part):
    wire = codec.payload_bytes(P) + 4 * codec.scale_count(P)
    if codec.quantized:
        return (12 if part == "encode" else 8) * P + wire
    e = codec.entries(P)
    return (8 * P + 9 * e) if part == "encode" else 13 * e


def run(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec, downlink_key
    dev = torch.device("cuda", 0)
    codecs = {"int8": UplinkCodec("int8"), "int4": UplinkCodec("int4"), "topk1": UplinkCodec("topk", 1),
              "topk8": UplinkCodec("topk", 8), "topk32": UplinkCodec("topk", 32)}
    rows = []
    for name, P in SIZES.items():
        g = torch.Generator(device=dev).manual_seed(P)
        theta = torch.randn(P, device=dev, generator=g)
        rep0 = theta + 0.01 * torch.randn(P, device=dev, generator=g)
        replica = rep0.clone()
        key = downlink_key(1)
        work, nbytes = {}, {}
        for kind, c in codecs.items():
            a, b = ops.encode_downlink(theta, rep0.clone(), c, key)               # the wire the apply replays (warms the encode up)
            if c.quantized:                                                       # codes in a 16-byte padded buffer, as received
                pad = torch.zeros((a.numel() + 15) // 16 * 16, dtype=torch.uint8, device=dev)
                pad[:a.numel()] = a
                a = pad
            work[f"encode_{kind}"] = (lambda c=c: ops.encode_downlink(theta, replica, c, key))
            work[f"apply_{kind}"] = (lambda c=c, a=a, b=b: ops.apply_downlink(replica, a, b, c))
            nbytes[f"encode_{kind}"] = _bytes(c, P, "encode")
            nbytes[f"apply_{kind}"] = _bytes(c, P, "apply")
        for fn in work.values():
            fn()                                                                  # warm-up (module load)
        per = {kind: [] for kind in work}
        for _ in range(args.passes):
            for kind, fn in work.items():                                         # kinds alternate inside every pass
                replica.copy_(rep0)
                _time(fn, args.iters, per[kind])
        rec = {"model": name, "P": P, "iters": args.iters, "passes": args.passes, "bytes": nbytes, "ms": {}, "hbm_share": {},
               "wire_bytes": {kind: c.payload_bytes(P) + 4 * c.scale_count(P) for kind, c in codecs.items()}}
        for kind in work:
            ms = statistics.median(per[kind])
            rec["ms"][kind] = round(ms, 5)
            rec["hbm_share"][kind] = round(nbytes[kind] / (ms * 1e-3) / HBM_BYTES_PER_S, 4)
        rows.append(rec)
        del theta, rep0, replica, work
        torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("downlink_bench.py measures the kernels on a GPU; none is visible")
    result = {"gpu": gpu_info(), "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S, "downlink": run(args)}
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
