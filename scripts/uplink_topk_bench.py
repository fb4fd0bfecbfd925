#!/usr/bin/env python
"""Cost of the top-k uplink with error feedback (fl/uplink.py, kind "topk") on the GPU.

    python scripts/uplink_topk_bench.py [--iters 20] [--passes 3] [--parts apply,encode] [--max-gb 24] [--out result.json]

1. Coordinator apply: ``ops.fedavg_apply_topk`` on K sparse deltas at k in {1, 8, 32} against ``ops.fedavg_apply`` on K
   fp32 client models and ``ops.fedavg_apply_quantized`` on K int8 deltas, in the same run: kernel time from device events
   around --iters back-to-back launches, median over --passes with all kinds alternating inside every pass, at K in
   {4, 8, 16, 32, 100} for P = 4,994 (cfg2, MLP 10-64-64-2) and P = 50,397,186 (wide MLP 10-4096x4-2).  Bytes moved, from
   the shapes: fp32 (K + 2) P 4; int8 K (P + 4 ceil(P / 256)) + 2 P 4; topk K 5 E(P, k) + 2 P 4 (entries read, theta read and
   written).  The offsets of a block are k distinct ascending values spread over the block (the cost does not depend on
   which).
2. Encode: ``ops.encode_topk_delta`` (topk_delta_kernel) of K models at the same sizes and k: 16 B per element (model,
   theta and residual read, residual written) plus K 5 E(P, k) entry bytes written.
The share of 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth) is those bytes over the kernel time.  --max-gb skips a case
whose fp32 inputs (K P 4 slots for the apply, 2 K P 4 models and residual for the encode) exceed it.  The card's name, power
limit and SM clock are read (nvidia-smi, read-only queries) in the same run.  Prints one JSON document."""
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
KS = (4, 8, 16, 32, 100)
TOPK = (1, 8, 32)
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


def _sparse_entries(K, P, k, dev, g):
    """(indices uint8 [K, E], values fp32 [K, E]): per block k distinct ascending offsets, block-randomly shifted"""
    import torch

    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    nblk = (P + 255) // 256
    stride = 256 // k
    shift = torch.randint(0, stride, (K, nblk, 1), device=dev, generator=g)
    off = (torch.arange(k, device=dev) * stride).view(1, 1, k) + shift
    last = P - (nblk - 1) * 256
    off[:, -1, :] = torch.arange(k, device=dev).clamp(max=last - 1)
    e = UplinkCodec("topk", k).entries(P)
    indices = off.reshape(K, nblk * k)[:, :e].to(torch.uint8).contiguous()
    values = torch.randn(K, e, device=dev, generator=g) * 1e-3
    return indices, values


def _share(nbytes, ms):
    return round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 4)


def apply_times(args) -> list:
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
            work, nbytes = {}, {}
            slots = torch.randn(K, P, device=dev, generator=g)
            work["fp32"] = lambda: ops.fedavg_apply(theta, slots, w)
            nbytes["fp32"] = (K + 2) * P * 4
            c8 = UplinkCodec("int8")
            payload = torch.randint(0, 256, (K, (P + 15) // 16 * 16), device=dev, dtype=torch.uint8, generator=g)
            scales = torch.rand(K, c8.scale_count(P), device=dev, generator=g) * 1e-3
            work["int8"] = lambda: ops.fedavg_apply_quantized(theta, payload, scales, w, c8)
            nbytes["int8"] = K * (c8.payload_bytes(P) + 4 * c8.scale_count(P)) + 2 * P * 4
            for k in TOPK:
                c = UplinkCodec("topk", k)
                idx, val = _sparse_entries(K, P, k, dev, g)
                work[f"topk{k}"] = (lambda i=idx, v=val, c=c: ops.fedavg_apply_topk(theta, i, v, w, c))
                nbytes[f"topk{k}"] = K * c.payload_bytes(P) + 2 * P * 4
            for fn in work.values():
                fn()                                                           # warm-up (module load)
            per = {kind: [] for kind in work}
            for _ in range(args.passes):
                for kind, fn in work.items():                                  # kinds alternate inside every pass
                    theta.copy_(theta0)
                    _time(fn, args.iters, per[kind])
            rec = {"model": name, "P": P, "K": K, "iters": args.iters, "bytes": nbytes, "ms": {}, "hbm_share": {}}
            for kind in work:
                ms = statistics.median(per[kind])
                rec["ms"][kind] = round(ms, 5)
                rec["hbm_share"][kind] = _share(nbytes[kind], ms)
            rec["speedup_vs_fp32"] = {kind: round(rec["ms"]["fp32"] / rec["ms"][kind], 3) for kind in work if kind != "fp32"}
            rec["speedup_vs_int8"] = {f"topk{k}": round(rec["ms"]["int8"] / rec["ms"][f"topk{k}"], 3) for k in TOPK}
            rows.append(rec)
            del slots, work, theta, theta0, payload, scales
            torch.cuda.empty_cache()
    return rows


def encode_times(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    dev = torch.device("cuda", 0)
    rows = []
    for name, P in SIZES.items():
        for K in KS:
            gb = 2 * K * P * 4 / 1e9
            if gb > args.max_gb:
                rows.append({"model": name, "P": P, "K": K, "skipped": f"{gb:.1f} GB of models and residuals > --max-gb"})
                continue
            g = torch.Generator(device=dev).manual_seed(K)
            theta = torch.randn(P, device=dev, generator=g)
            models = theta + 0.01 * torch.randn(K, P, device=dev, generator=g)
            residual = torch.zeros(K, P, device=dev)
            for k in TOPK:
                c = UplinkCodec("topk", k)
                ops.encode_topk_delta(models, theta, residual, c)                  # warm-up
                per = []
                for _ in range(args.passes):
                    _time(lambda: ops.encode_topk_delta(models, theta, residual, c), args.iters, per)
                ms = statistics.median(per)
                nbytes = 16 * K * P + K * c.payload_bytes(P)
                rows.append({"model": name, "P": P, "K": K, "k": k, "ms": round(ms, 5), "bytes": nbytes, "hbm_share": _share(nbytes, ms),
                             "GBps": round(nbytes / (ms * 1e-3) / 1e9, 1)})
            del models, theta, residual
            torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--max-gb", type=float, default=24.0)
    ap.add_argument("--parts", default="apply,encode")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("uplink_topk_bench.py measures the kernels on a GPU; none is visible")
    parts = args.parts.split(",")
    result = {"gpu": gpu_info(), "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S}
    if "apply" in parts:
        result["fedavg_apply"] = apply_times(args)
    if "encode" in parts:
        result["encode_topk_delta"] = encode_times(args)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
