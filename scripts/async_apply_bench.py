#!/usr/bin/env python
"""Apply time of asynchronous buffered aggregation's rows (``ROWS_F32_BASED``: every model read as its delta to a base in the
version ring, the new theta also stored to the ring) against the synchronous fp32 apply at equal K.

    python scripts/async_apply_bench.py [--iters 20] [--passes 5] [--out result.json]

For P = 2,401 (FFNN) and P = ResNet-18's arena, K in {4, 16, 64} and S in {1, 4, 16}: ``ops.fedavg_apply`` (K fp32 models)
and ``ops.fedavg_apply_based`` (the same K models, bases spread over the S + 1 readable ring slots) with the mean and plain
FedAvg.  Device events around --iters back-to-back calls after one warm-up call per shape; the median over --passes.  The
card's name, power limit and SM clock are read (nvidia-smi, read-only query) in the same run.  Prints one JSON document."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KS = (4, 16, 64)
SS = (1, 4, 16)


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return dict(zip(q.split(","), [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def timed(fn, iters: int, passes: int) -> float:
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(passes):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / iters)
    return statistics.median(times)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.models import build_model, flatten_params
    if not torch.cuda.is_available():
        raise SystemExit("async_apply_bench needs a GPU: nothing was measured")
    dev = torch.device("cuda")
    sizes = {"ffnn": 2401, "resnet18": flatten_params(build_model("resnet18")).numel()}
    rows = []
    for name, p in sizes.items():
        g = torch.Generator(device=dev).manual_seed(0)
        theta = torch.randn(p, device=dev, generator=g)
        for k in KS:
            models = torch.randn(k, p, device=dev, generator=g)
            w = torch.full((k,), 1.0 / k, device=dev)
            t = theta.clone()
            sync_us = timed(lambda: ops.fedavg_apply(t, models, w, 1.0), args.iters, args.passes)
            for s in SS:
                ring = torch.randn(s + 2, p, device=dev, generator=g)
                bases = [i % (s + 1) for i in range(k)]           # slots 0 .. S, the write slot is S + 1
                based_us = timed(lambda: ops.fedavg_apply_based(t, models, ring, bases, w, s + 1), args.iters, args.passes)
                rows.append({"model": name, "P": p, "K": k, "S": s, "fedavg_apply_us": round(sync_us, 2),
                             "fedavg_apply_based_us": round(based_us, 2), "ratio": round(based_us / sync_us, 3)})
                print(json.dumps(rows[-1]), file=sys.stderr)
            del models
        torch.cuda.empty_cache()
    doc = {"gpu": gpu_info(), "iters": args.iters, "passes": args.passes, "rows": rows}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(doc, f, indent=1)
    print(json.dumps(doc))
    return 0


if __name__ == "__main__":
    sys.exit(main())
