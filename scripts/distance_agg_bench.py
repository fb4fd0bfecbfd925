"""Cost of the distance-based robust aggregators (the weighted geometric median ``geomed`` and the norm-bounded mean
``norm_clip``, ``ops/csrc/distance_agg.cuh``) next to the mean and the coordinate-wise median.

    python scripts/distance_agg_bench.py [--iters 20] [--passes 3] [--max-gb 12] [--out result.json]

``ops.fedavg_apply`` (fp32 rows) and ``ops.fedavg_apply_quantized`` (int8 rows) kernel time: device events around --iters
back-to-back calls, median over --passes, for mean, median, geomed with L = 1 and L = 3, and norm_clip, at K in {4, 8, 16, 32,
100} rows of P = 2,401 (FFNN), 4,994 (cfg2) and 50,397,186 (wide MLP) parameters.  Bytes each kind must move, from the shapes
and the pass count: R = the bytes of the K rows (4 K P fp32; K P codes + 4 K ceil(P / 256) steps int8), one read per pass
(mean and median: 1; geomed: L + 1; norm_clip: 2), plus theta read and written (8 P) and read once per distance pass (fp32
rows).  The share of 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth) is that over the time.  int8 has no median row (the
coordinate-wise kinds run there too, but are not the comparison here).  --max-gb skips a case whose rows exceed it.

The card's name, power limit and SM clock are read (nvidia-smi, read-only queries) in the same run.  Prints one JSON document."""
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
SIZES = {"ffnn": 2401, "cfg2": 4994, "wide_mlp": 50397186}


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def kinds():
    from colearn_federated_learning_b200.fl.aggregate import Aggregator
    return {"mean": (Aggregator("mean"), 1), "median": (Aggregator("median"), 1), "geomed_L1": (Aggregator("geomed", iters=1), 2),
            "geomed_L3": (Aggregator("geomed", iters=3), 4), "norm_clip": (Aggregator("norm_clip", clip_norm=1.0), 2)}


def time_call(fn, iters, passes) -> float:
    import torch
    fn()
    per = []
    for _ in range(passes):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        per.append(e0.elapsed_time(e1) / iters)
    return statistics.median(per)


def run(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    dev = torch.device("cuda", 0)
    rows = []
    for rowtype in ("fp32", "int8"):
        for name, P in SIZES.items():
            for K in KS:
                row_bytes = 4 * K * P if rowtype == "fp32" else K * P + 4 * K * ((P + 255) // 256)
                if row_bytes / 1e9 > args.max_gb:
                    rows.append({"rows": rowtype, "model": name, "P": P, "K": K, "skipped": f"{row_bytes / 1e9:.1f} GB > --max-gb"})
                    continue
                g = torch.Generator(device=dev).manual_seed(K)
                theta0 = torch.randn(P, device=dev, generator=g)
                theta = theta0.clone()
                w = torch.full((K,), 1.0 / K, device=dev)
                if rowtype == "fp32":
                    x = theta0 + 0.01 * torch.randn(K, P, device=dev, generator=g)
                else:
                    codec = UplinkCodec("int8")
                    payload = torch.randint(-127, 128, (K, (P + 15) // 16 * 16), device=dev, dtype=torch.int8, generator=g).view(torch.uint8)
                    scales = torch.full((K, (P + 255) // 256), 1e-4, device=dev)
                rec = {"rows": rowtype, "model": name, "P": P, "K": K, "ms": {}, "bytes": {}, "hbm_share": {}}
                big = row_bytes > 1e9
                for kind, (agg, reads) in kinds().items():
                    if rowtype == "int8" and kind == "median":
                        continue
                    if rowtype == "fp32":
                        fn = lambda: ops.fedavg_apply(theta, x, w, aggregator=agg)  # noqa: E731
                    else:
                        fn = lambda: ops.fedavg_apply_quantized(theta, payload, scales, w, codec, aggregator=agg)  # noqa: E731
                    ms = time_call(fn, max(2, args.iters // 5) if big else args.iters, args.passes)
                    theta.copy_(theta0)
                    dist_reads = reads - 1 if agg.distance_based and rowtype == "fp32" else 0
                    b = reads * row_bytes + 8 * P + 4 * P * dist_reads
                    rec["ms"][kind] = round(ms, 5)
                    rec["bytes"][kind] = b
                    rec["hbm_share"][kind] = round(b / (ms * 1e-3) / HBM_BYTES_PER_S, 4)
                rec["vs_mean"] = {k: round(v / rec["ms"]["mean"], 3) for k, v in rec["ms"].items()}
                rows.append(rec)
                del theta, theta0
                x = payload = scales = None
                torch.cuda.empty_cache()
    return rows


def main(argv=None) -> int:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--passes", type=int, default=3)
    p.add_argument("--max-gb", type=float, default=12.0)
    p.add_argument("--out", default=None)
    args = p.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "needs a CUDA device"}))
        return 1
    doc = {"gpu": gpu_info(), "kernels": run(args), "gpu_after": gpu_info()}
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    return 0


if __name__ == "__main__":
    sys.exit(main())
