"""Class-weighted training on one GPU: µs per batch-1 SGD step of the persistent kernel at variant 5, weighted
(mlp_persistent_cw.cu, balanced-looking weights) against unweighted, for ``ffnn`` and ``ffnn_category`` at 8 192 samples, with
the timing protocol of scripts/category_bench.py (CUDA events around one launch, after a warm-up launch of each build).  The two
builds' launches alternate within every repetition, so drifting clocks and neighbours on the card hit both alike.  Prints one
JSON line with the card's name, power limit and SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from colearn_federated_learning_b200 import ops  # noqa: E402
from colearn_federated_learning_b200.data import synthetic_category, synthetic_unsw  # noqa: E402
from colearn_federated_learning_b200.models import build_model, flatten_params  # noqa: E402

WEIGHTS = {"ffnn": [0.55, 5.2], "ffnn_category": [10.0, 0.381, 0.445, 8.05, 10.0]}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else torch.cuda.get_device_name(0)


def launches(model, n, dev):
    """(unweighted launch, weighted launch) of one client's fit over n samples"""
    m = build_model(model)
    theta = flatten_params(m).to(dev)
    x, y = (synthetic_unsw if model == "ffnn" else synthetic_category)(n, seed=1, device=dev)
    loss = "bce" if model == "ffnn" else "xent"
    perm = ops.device_permutation(n, 1, seed=3, device=dev)
    out = torch.empty_like(theta)
    descs = ops.build_client_descs([ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=out, perm=perm)], dev)
    dims, act = m.spec.dims, m.spec.out_activation
    plain = lambda: ops.mlp_local_sgd_multi(dims, act, descs, 1, batch_size=1, lr=0.01, loss=loss, variant=5)  # noqa: E731
    weighted = lambda: ops.mlp_local_sgd_multi(dims, act, descs, 1, batch_size=1, lr=0.01, loss=loss, variant=5,  # noqa: E731
                                               class_weights=WEIGHTS[model])
    return plain, weighted


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
    ap.add_argument("--reps", type=int, default=9)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "class_weight_bench.py measures on a GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "samples": a.samples, "reps": a.reps}
    for model in ("ffnn", "ffnn_category"):
        plain, weighted = launches(model, a.samples, dev)
        plain()
        weighted()
        torch.cuda.synchronize()
        tp, tw = [], []
        for _ in range(a.reps):
            tp.append(timed(plain, a.samples))
            tw.append(timed(weighted, a.samples))
        tp, tw = sorted(tp), sorted(tw)
        res[model] = {"unweighted_us_per_step": {"median": tp[len(tp) // 2], "min": tp[0], "max": tp[-1]},
                      "weighted_us_per_step": {"median": tw[len(tw) // 2], "min": tw[0], "max": tw[-1]},
                      "weighted_over_unweighted": tw[len(tw) // 2] / tp[len(tp) // 2]}
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
