"""Local optimizers on the layer-wise wgmma trainer, one GPU: ms per step of `Net` (784-128-64-10, batch 32) and `wide_mlp`
(10-4096x4-2, batch 128) under plain SGD, SGD with momentum 0.9 and Adam.  CUDA events around whole fits (every step's forward,
backward and update, with the host loop that launches them), after a warm-up fit of each; the three optimizers alternate within
every repetition, so drifting clocks and neighbours on the card hit all alike.  Prints one JSON line with the card's name,
power limit and SM clock, read in the same run, and the extra HBM traffic the optimizer epilogue adds per step, computed from
the shapes (not measured).  Fails without a GPU."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from colearn_federated_learning_b200 import ops  # noqa: E402
from colearn_federated_learning_b200.fl import FitConfig  # noqa: E402
from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer  # noqa: E402
from colearn_federated_learning_b200.fl.local_opt import LocalOpt  # noqa: E402
from colearn_federated_learning_b200.models import build_model, flatten_params  # noqa: E402

OPTS = {"sgd": None, "momentum": LocalOpt("SGD", momentum=0.9), "adam": LocalOpt("Adam")}
CASES = {"net": (32, 50), "wide_mlp": (128, 20)}     # model -> (batch size, steps per timed fit)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else torch.cuda.get_device_name(0)


def extra_bytes(trainer, kind):
    """HBM bytes per step the optimizer adds over plain SGD, from shapes: per parameter element, momentum reads and writes m
    (8 B), Adam m and v (16 B); plain SGD moves 10 B per element of the fused layers (master read + write, bf16 shadow)"""
    per = {"sgd": 0, "momentum": 8, "adam": 16}[kind]
    fused = sum(trainer.dims[l] * trainer.dims[l + 1] for l in range(trainer.L) if trainer.exact[l])
    return {"extra_bytes_per_step": per * trainer.n_params, "fused_layer_elems": fused,
            "plain_fused_bytes_per_step": 10 * fused, "extra_fused_bytes_per_step": per * fused}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "layerwise_opt_bench.py measures on a GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": a.reps}
    for name, (b, steps) in CASES.items():
        torch.manual_seed(0)
        model = build_model(name)
        flat0 = flatten_params(model).to(dev)
        spec = model.spec
        n = b * steps
        x = torch.rand(n, spec.dims[0], device=dev)
        y = torch.randint(0, spec.dims[-1], (n, 1), device=dev).float()
        perm = ops.device_permutation(n, 1, seed=1, device=dev)
        cfg = FitConfig(model=name, loss="xent", batch_size=b, lr=0.001, epochs=1)
        flat = flat0.clone()
        tr = LayerwiseMLPTrainer(spec, flat, b)

        def fit(lo):
            tr.fit(flat, x, y, cfg, perm, local_opt=lo)
        for lo in OPTS.values():
            flat.copy_(flat0)
            fit(lo)
        torch.cuda.synchronize()
        times = {k: [] for k in OPTS}
        for _ in range(a.reps):
            for k, lo in OPTS.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                flat.copy_(flat0)                                  # every fit starts from the same model (not timed)
                e0.record()
                fit(lo)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) / steps)
        row = {"batch_size": b, "steps": steps, "params": tr.n_params}
        for k, t in times.items():
            t = sorted(t)
            row[k] = {"median_ms_per_step": t[len(t) // 2], "min": t[0], "max": t[-1], **extra_bytes(tr, k)}
        res[name] = row
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
