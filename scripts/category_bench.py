"""Attack categorisation on one GPU: µs per batch-1 SGD step of the persistent kernel at 8 192 samples (CUDA events, after a
warm-up launch) for ``ffnn`` at variant 5 and ``ffnn_category`` at variants 5, 6, 3 and 1, each timed ``--reps`` times, and
rounds/s of a local-mode ``ffnn_category`` training at bench.py's default configuration (``bench.py --gpus 1``: one virtual
worker on 8 192 rows, batch 1, lr 0.01, one local epoch per round, FedAvg), host clock around ``--rounds`` rounds that end in a
device synchronise.  Prints one JSON line with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from colearn_federated_learning_b200 import ops  # noqa: E402
from colearn_federated_learning_b200.data import synthetic_category, synthetic_unsw  # noqa: E402
from colearn_federated_learning_b200.models import build_model, flatten_params  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else torch.cuda.get_device_name(0)


def step_us(model, variant, n, reps, dev):
    m = build_model(model)
    theta = flatten_params(m).to(dev)
    if model == "ffnn":
        x, y = synthetic_unsw(n, seed=1, device=dev)
        loss = "bce"
    else:
        x, y = synthetic_category(n, seed=1, device=dev)
        loss = "xent"
    perm = ops.device_permutation(n, 1, seed=3, device=dev)
    act = m.spec.out_activation
    out = torch.empty_like(theta)
    task = ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=out, perm=perm)
    descs = ops.build_client_descs([task], dev)
    run = lambda: ops.mlp_local_sgd_multi(m.spec.dims, act, descs, 1, batch_size=1, lr=0.01, loss=loss, variant=variant)  # noqa: E731
    run()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1000.0 / n)
    return times


def rounds_per_s(dev, rounds, workers=1):
    from colearn_federated_learning_b200.control.coordinator import train_virtual_workers
    from colearn_federated_learning_b200.data import BaseDataset, federate
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    model = build_model("ffnn_category").to(dev)
    theta = flatten_params(model).to(dev)
    x, y = synthetic_category(8192, seed=0)
    fed = federate(BaseDataset(x, y), [f"w{i}" for i in range(workers)], dev)
    cfg = FitConfig(model="ffnn_category", loss="xent", batch_size=1, epochs=1, max_nr_batches=-1, lr=0.01, shuffle=True, seed=0)
    train_virtual_workers(theta, model, fed, cfg, 0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for r in range(rounds):
        flats, _, counts = train_virtual_workers(theta, model, fed, cfg, r + 1)
        w = torch.full((len(counts),), 1.0 / len(counts), device=dev)
        ops.fedavg_apply(theta, flats, w, 1.0)
    torch.cuda.synchronize()
    return rounds / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=8192)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--rounds", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "category_bench.py measures on a GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card()}
    for model, v in (("ffnn", 5), ("ffnn_category", 5), ("ffnn_category", 6), ("ffnn_category", 3), ("ffnn_category", 1)):
        t = sorted(step_us(model, v, a.samples, a.reps, dev))
        res[f"{model}_v{v}_us_per_step"] = {"median": t[len(t) // 2], "min": t[0], "max": t[-1]}
    res["ffnn_category_rounds_per_s"] = rounds_per_s(dev, a.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
