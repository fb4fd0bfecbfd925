#!/usr/bin/env python
"""Cost of the Byzantine-robust aggregators (coordinate-wise median / trimmed mean) fused into the FedAvg kernels.

    python scripts/robust_agg_bench.py [--iters 20] [--passes 3] [--steps 20] [--out result.json]

1. ``ops.fedavg_apply`` kernel time (device events around --iters back-to-back launches, median over --passes) for mean,
   median and trimmed_mean (beta 0.1) at K in {4, 8, 16, 32, 100} client models of P = 4,994 (cfg2, MLP 10-64-64-2) and
   P = 50,397,186 (wide MLP 10-4096x4-2) parameters.  Bytes moved = (K + 2) P 4 (K slots read, theta read and written); the
   share of 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth) is that over the kernel time.  At K = 100, P = 50 M the slots
   take 20 GB; --max-gb skips any case above it.
2. cfg2 star rounds/s at world 1 for each kind (FederatedEngine.run_rounds(1), device events, median over passes).
3. With >= 2 GPUs: wide-MLP two-shot rounds/s at world = #GPUs for mean (NVLS where the engine uses it) and median (P2P).

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
KINDS = (("mean", 0.1), ("median", 0.1), ("trimmed_mean", 0.1))


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def kernel_times(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.fl.aggregate import Aggregator
    dev = torch.device("cuda", 0)
    rows = []
    for name, P in SIZES.items():
        for K in KS:
            gb = (K + 1) * P * 4 / 1e9
            if gb > args.max_gb:
                rows.append({"model": name, "P": P, "K": K, "skipped": f"{gb:.1f} GB > --max-gb"})
                continue
            g = torch.Generator(device=dev).manual_seed(K)
            slots = torch.randn(K, P, device=dev, generator=g)
            w = torch.full((K,), 1.0 / K, device=dev)
            theta0 = torch.randn(P, device=dev, generator=g)
            theta = theta0.clone()
            iters = args.iters if P * K * K < 2e11 else max(2, args.iters // 10)     # the general path at K = 100, P = 50 M
            rec = {"model": name, "P": P, "K": K, "bytes": (K + 2) * P * 4, "iters": iters, "ms": {}, "hbm_share": {}}
            for kind, beta in KINDS:
                agg = Aggregator(kind, beta)
                ops.fedavg_apply(theta, slots, w, aggregator=agg)                     # warm-up (module load)
                per = []
                for _ in range(args.passes):
                    theta.copy_(theta0)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(iters):
                        ops.fedavg_apply(theta, slots, w, aggregator=agg)
                    e1.record()
                    e1.synchronize()
                    per.append(e0.elapsed_time(e1) / iters)
                ms = statistics.median(per)
                rec["ms"][kind] = round(ms, 5)
                rec["hbm_share"][kind] = round(rec["bytes"] / (ms * 1e-3) / HBM_BYTES_PER_S, 4)
            rec["vs_mean"] = {k: round(rec["ms"][k] / rec["ms"]["mean"], 3) for k, _ in KINDS}
            rows.append(rec)
            del slots, theta, theta0
            torch.cuda.empty_cache()
    return rows


def star_rounds(args) -> dict:
    import torch

    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.fl.aggregate import Aggregator
    from colearn_federated_learning_b200.parallel import FederatedEngine
    engines = {}
    for kind, beta in KINDS:
        eng = FederatedEngine("mlp", backend="fused", device=torch.device("cuda", 0), batch_size=1, lr=0.01, seed=1,
                              aggregator=Aggregator(kind, beta))
        x, y = synthetic_unsw(8192, seed=0)
        eng.set_local_data(x, y)
        for _ in range(args.warmup):
            eng.run_rounds(1)
        engines[kind] = eng
    torch.cuda.synchronize()
    per = {k: [] for k in engines}
    for _ in range(args.passes):
        for k, eng in engines.items():                      # kinds alternate inside every pass
            ms = sum(eng.run_rounds(1).device_ms for _ in range(args.steps))
            per[k].append(args.steps / (ms * 1e-3))
    return {"description": "star, MLP 10-64-64-2, batch 1, 8192 samples, world 1",
            "rounds_per_s": {k: round(statistics.median(v), 2) for k, v in per.items()}, "rounds_per_s_passes": per}


def _twoshot_rank(rank, world, port, out, steps, warmup, passes):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from colearn_federated_learning_b200.data import shard_bounds, synthetic_unsw
        from colearn_federated_learning_b200.fl.aggregate import Aggregator
        from colearn_federated_learning_b200.parallel import FederatedEngine
        x, y = synthetic_unsw(8192 * world, seed=0)
        lo, hi = list(shard_bounds(8192 * world, world))[rank]
        res = {}
        for kind in ("mean", "median"):
            eng = FederatedEngine("wide_mlp", backend="fused", device=torch.device("cuda", rank), batch_size=1024, lr=0.01, seed=1,
                                  bf16_shadow=True, aggregator=Aggregator(kind))
            eng.set_local_data(x[lo:hi], y[lo:hi])
            for _ in range(warmup):
                eng.run_rounds(1)
            per = []
            for _ in range(passes):
                rep = [eng.run_rounds(1) for _ in range(steps)]
                per.append(steps / (sum(r.device_ms for r in rep) * 1e-3))
            res[kind] = {"rounds_per_s": round(statistics.median(per), 2), "nvls": rep[-1].extra.get("nvls")}
            del eng
            torch.cuda.empty_cache()
        if rank == 0:
            torch.save(res, out)
    finally:
        dist.destroy_process_group()


def twoshot_rounds(args) -> dict:
    import torch
    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        return {"not measured": f"needs >= 2 GPUs, {world} visible"}
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "twoshot.pt")
        mp.spawn(_twoshot_rank, args=(world, port, out, args.steps, args.warmup, args.passes), nprocs=world, join=True)
        res = torch.load(out, weights_only=False)
    return {"description": f"two-shot, wide MLP 10-4096x4-2, batch 1024, bf16 shadow, world {world}", **res}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--max-gb", type=float, default=24.0)
    ap.add_argument("--parts", default="kernel,star,twoshot")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("robust_agg_bench.py measures on a GPU; none is visible")
    parts = args.parts.split(",")
    result = {"gpu": gpu_info(), "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S}
    if "kernel" in parts:
        result["fedavg_apply"] = kernel_times(args)
    if "star" in parts:
        result["star_cfg2"] = star_rounds(args)
    if "twoshot" in parts:
        result["twoshot_wide_mlp"] = twoshot_rounds(args)
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
