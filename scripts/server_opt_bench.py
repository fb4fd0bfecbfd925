#!/usr/bin/env python
"""Cost of the server optimizers fused into the FedAvg kernels, at world 1 on one GPU.

    python scripts/server_opt_bench.py [--steps 20] [--warmup 3] [--passes 3] [--out result.json]

Two configs of bench.py: cfg2 (star path, MLP 10-64-64-2, batch 1, 8192 samples) and the cfg5 shape (two-shot path, wide MLP
10-4096x4-2, batch 1024, 8192 samples, bf16 shadow).  For each, the kinds sgd (plain FedAvg), avgm and adam run as separate
engines; every pass times --steps single-round calls of each kind in turn (device events, FederatedEngine.run_rounds(1)),
and the median over the passes is reported as rounds/s.  A second set of engines with COLEARN_PHASE_TIMING semantics
(phase_timing=True) reports the per-round device time of the reduce + apply phase.  The card's name, power limit and SM clock
are read (nvidia-smi, read-only queries) in the same run.  Prints one JSON document."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

CONFIGS = {  # name: (model, samples, batch size, bf16 shadow, description)
    "cfg2": ("mlp", 8192, 1, False, "star, MLP 10-64-64-2, batch 1"),
    "cfg5": ("wide_mlp", 8192, 1024, True, "two-shot, wide MLP 10-4096x4-2, batch 1024, bf16 shadow"),
}
KINDS = ("sgd", "avgm", "adam")


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def make_engine(model, n, bsz, shadow, kind, phase_timing):
    import torch

    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.fl.server_opt import ServerOpt
    from colearn_federated_learning_b200.parallel import FederatedEngine

    eng = FederatedEngine(model, backend="fused", device=torch.device("cuda", 0), batch_size=bsz, lr=0.01, seed=1,
                          bf16_shadow=shadow, phase_timing=phase_timing, server_opt=None if kind == "sgd" else ServerOpt(kind))
    x, y = synthetic_unsw(n, seed=0)
    eng.set_local_data(x, y)
    return eng


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--configs", default="cfg2,cfg5")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("server_opt_bench.py measures on a GPU; none is visible")
    result = {"gpu": gpu_info(), "world": 1, "steps": args.steps, "passes": args.passes, "configs": {}}
    for name in args.configs.split(","):
        model, n, bsz, shadow, desc = CONFIGS[name]
        engines = {k: make_engine(model, n, bsz, shadow, k, False) for k in KINDS}
        for eng in engines.values():
            for _ in range(args.warmup):
                eng.run_rounds(1)
        torch.cuda.synchronize()
        per_pass = {k: [] for k in KINDS}
        for _ in range(args.passes):
            for k, eng in engines.items():                 # kinds alternate inside every pass
                ms = sum(eng.run_rounds(1).device_ms for _ in range(args.steps))
                per_pass[k].append(args.steps / (ms * 1e-3))
        del engines
        rec = {"description": desc, "params": None, "rounds_per_s": {}, "rounds_per_s_passes": per_pass, "reduce_apply_ms": {}}
        for k in KINDS:
            rec["rounds_per_s"][k] = round(statistics.median(per_pass[k]), 2)
        # per-phase device time (event pairs around the reduce + apply launches), separate engines: the events add to the round
        for k in KINDS:
            eng = make_engine(model, n, bsz, shadow, k, True)
            rec["params"] = eng.P
            for _ in range(args.warmup):
                eng.run_rounds(1)
            phase = []
            for _ in range(args.steps):
                ph = eng.run_rounds(1).extra.get("phases_ms") or {}
                phase.append(sum(v for key, v in ph.items() if "reduce_apply" in key))
            rec["reduce_apply_ms"][k] = round(statistics.median(phase), 4)
            del eng
        base = rec["rounds_per_s"]["sgd"]
        rec["slowdown_vs_sgd"] = {k: round(base / rec["rounds_per_s"][k], 4) for k in KINDS}
        result["configs"][name] = rec
        torch.cuda.empty_cache()
    text = json.dumps(result, indent=1)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
