"""Local optimizers on one GPU: µs per batch-1 step of the FFNN's local fit at 8 192 samples, for one client and for 132
clients in one launch (one CTA per SM of an H100 SXM), four ways: variant 5 plain SGD (the default kernel), variant 1 plain SGD
(the shared-memory kernel the optimizer instances are built on), SGD with momentum 0.9 and Adam (mlp_persistent_opt.cu).  CUDA
events around one launch, after a warm-up launch of each; the four launches alternate within every repetition, so drifting
clocks and neighbours on the card hit all alike.  Prints one JSON line with the card's name, power limit and SM clock, read in
the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from colearn_federated_learning_b200 import ops  # noqa: E402
from colearn_federated_learning_b200.data import synthetic_unsw  # noqa: E402
from colearn_federated_learning_b200.fl.local_opt import LocalOpt  # noqa: E402
from colearn_federated_learning_b200.models import build_model, flatten_params  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else torch.cuda.get_device_name(0)


def launches(clients, n, dev):
    m = build_model("ffnn")
    theta = flatten_params(m).to(dev)
    outs = torch.empty(clients, theta.numel(), device=dev)
    tasks, keep = [], []
    for i in range(clients):
        x, y = synthetic_unsw(n, seed=1 + i, device=dev)
        perm = ops.device_permutation(n, 1, seed=3 + i, device=dev)
        keep += [x, y, perm]
        tasks.append(ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=outs[i], perm=perm))
    descs = ops.build_client_descs(tasks, dev)
    dims, act = m.spec.dims, m.spec.out_activation

    def run(**kw):
        return lambda: ops.mlp_local_sgd_multi(dims, act, descs, clients, batch_size=1, lr=0.01, loss="bce", **kw)
    return keep, {"v5_sgd": run(variant=5), "v1_sgd": run(variant=1),
                  "momentum": run(local_opt=LocalOpt("SGD", momentum=0.9)), "adam": run(local_opt=LocalOpt("Adam"))}


def timed(run, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1000.0 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "local_opt_bench.py measures on a GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "samples": a.samples, "reps": a.reps, "net": "ffnn", "batch_size": 1}
    for clients in (1, 132):
        keep, runs = launches(clients, a.samples, dev)
        for r in runs.values():
            r()
        torch.cuda.synchronize()
        times = {k: [] for k in runs}
        for _ in range(a.reps):
            for k, r in runs.items():
                times[k].append(timed(r, a.samples))
        row = {}
        for k, t in times.items():
            t = sorted(t)
            row[k] = {"median_us_per_step": t[len(t) // 2], "min": t[0], "max": t[-1]}
        res[f"clients_{clients}"] = row
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
