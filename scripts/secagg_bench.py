#!/usr/bin/env python
"""Cost of secure aggregation (fl/secagg.py, ops/csrc/secagg.cuh) on the GPU.

    python scripts/secagg_bench.py [--iters 20] [--passes 5] [--out result.json]

1. Device mask: ``ops.secagg_mask`` (secagg_mask_kernel) of one update with S = 2 / 10 / 100 streams (the self stream plus
   S - 1 pair streams).
2. Coordinator unmask-apply: ``ops.fedavg_apply_secagg`` (fedavg_secagg_kernel, after secagg_streams_kernel when the streams
   are split) for K = 10 / 100 survivors and |D| = 0 / 1 / 10 dropped devices, S = K (1 + |D|) correction streams, next to
   ``ops.fedavg_apply`` of K fp32 models (the apply without secure aggregation).
At P = 2,401 (FFNN) and P = 50,397,186 (wide MLP 10-4096x4-2).  Kernel time from device events around --iters back-to-back
calls, median over --passes, the variants alternating inside every pass.  ChaCha20 blocks per second: S ceil(P / 16) over the
time.  Bytes streamed: mask 12 P (model, theta read, row written); unmask-apply 4 K P (rows) + 8 P (theta read and written);
fp32 apply 4 K P + 8 P.  The share of 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth) is those bytes over the time.  The card's
name, power limit and SM clock are read (nvidia-smi, read-only queries) in the same run.  Prints one JSON document."""
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
SIZES = {"ffnn": 2401, "wide_mlp": 50397186}


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def _time(fn, iters, out):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    out.append(e0.elapsed_time(e1) / iters)


def run(args) -> list:
    import numpy as np
    import torch

    from colearn_federated_learning_b200 import ops
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0)
    rows = []
    for name, P in SIZES.items():
        cols = (P + 15) // 16
        g = torch.Generator(device=dev).manual_seed(P)
        theta = torch.randn(P, device=dev, generator=g)
        model = theta + 0.01 * torch.randn(P, device=dev, generator=g)
        work, blocks, nbytes = {}, {}, {}
        for S in (2, 10, 100):
            kw = ops.secagg_key_words([bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(S)], dev)
            sg = torch.tensor([1 if i % 2 else -1 for i in range(S)], dtype=torch.int32, device=dev)
            work[f"mask_S{S}"] = (lambda kw=kw, sg=sg: ops.secagg_mask(model, theta, kw, sg, 1.0, 24))
            blocks[f"mask_S{S}"], nbytes[f"mask_S{S}"] = S * cols, 12 * P
        target = theta.clone()
        for K in (10, 100):
            masked = torch.empty((K, P), dtype=torch.int32, device=dev).random_(generator=g)   # 20 GB for the wide MLP at K = 100
            for nd in (0, 1, 10):
                S = K * (1 + nd)
                kw = ops.secagg_key_words([bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(S)], dev)
                sg = torch.full((S,), -1, dtype=torch.int32, device=dev)
                key = f"unmask_K{K}_D{nd}"
                work[key] = (lambda masked=masked, kw=kw, sg=sg, K=K: ops.fedavg_apply_secagg(target, masked, kw, sg, 24, K))
                blocks[key], nbytes[key] = S * cols, 4 * K * P + 8 * P
            models = masked.view(torch.float32)
            w = torch.full((K,), 1.0 / K, device=dev)
            work[f"fedavg_fp32_K{K}"] = (lambda models=models, w=w: ops.fedavg_apply(target, models, w))
            blocks[f"fedavg_fp32_K{K}"], nbytes[f"fedavg_fp32_K{K}"] = 0, 4 * K * P + 8 * P
            for fn in work.values():
                fn()                                                               # warm-up (module load, first launches)
            per = {k: [] for k in work}
            for _ in range(args.passes):
                for k, fn in work.items():
                    target.copy_(theta)
                    _time(fn, args.iters, per[k])
            rec = {"model": name, "P": P, "K": K, "iters": args.iters, "passes": args.passes, "ms": {}, "chacha_blocks_per_s": {},
                   "hbm_share": {}}
            for k in work:
                ms = statistics.median(per[k])
                rec["ms"][k] = round(ms, 5)
                rec["hbm_share"][k] = round(nbytes[k] / (ms * 1e-3) / HBM_BYTES_PER_S, 4)
                if blocks[k]:
                    rec["chacha_blocks_per_s"][k] = float(f"{blocks[k] / (ms * 1e-3):.4g}")
            rows.append(rec)
            for k in [k for k in work if not k.startswith("mask_")]:
                del work[k]
            del masked, models
            torch.cuda.empty_cache()
        del theta, model, target, work
        torch.cuda.empty_cache()
    return rows


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("secagg_bench.py measures the kernels on a GPU; none is visible")
    result = {"gpu": gpu_info(), "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S, "secagg": run(args)}
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
