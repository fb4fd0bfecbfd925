"""Federated anomaly detection on one GPU: the autoencoder's local fit and the reconstruction-error summary.

    python scripts/anomaly_bench.py [--steps 8192] [--repeats 5] [--iters 20] [--out result.json]

* fit: one client's whole local fit of 8192 batch-1 SGD steps in one persistent-kernel launch (``ops.mlp_local_sgd``,
  variant 5), the autoencoder (10-32-4-32-10, MSE on its input) next to the FFNN (10-50-30-10-1, BCE) in the same call; device
  events around each fit, median and spread over the repeats.
* recon_summary: ``ops.recon_summary`` (one memset + recon_summary_kernel; kernel time from torch.profiler, call time from
  device events) against an eager-torch equivalent of the same counts at 10^5, 10^6 and 10^7 rows of 10 columns with labels.
  Bytes = N (2 D 4 + 4): x̂, x and the labels, read once; the share is against 3.35 TB/s (H100 SXM data sheet HBM3).

The card's name, power limit and SM clocks are read (nvidia-smi) before and after, in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from eval_summary_bench import HBM_BYTES_PER_S, events, gpu_info  # noqa: E402

BINS = 256


def fit_times(steps: int, repeats: int) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.data import synthetic_anomaly, synthetic_unsw
    from colearn_federated_learning_b200.models import build_model, flatten_params
    dev = torch.device("cuda", 0)
    rows = []
    for name, loss in (("autoencoder", "mse"), ("ffnn", "bce")):
        torch.manual_seed(0)
        model = build_model(name)
        theta0 = flatten_params(model).to(dev)
        if name == "autoencoder":
            x, _ = synthetic_anomaly(steps, seed=1, attack_fraction=0.0, device=dev)
            y = x
        else:
            x, y = synthetic_unsw(steps, seed=1, device=dev)
        spec = model.spec
        per = []
        for r in range(repeats + 1):
            flat = theta0.clone()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ops.mlp_local_sgd(flat, spec.dims, x, y, None, 1, 0.01, 1, -1, loss, spec.out_activation)
            e1.record()
            e1.synchronize()
            if r:                                      # the first fit loads the module and sets the smem attribute
                per.append(e0.elapsed_time(e1) * 1e3)
        rows.append({"model": name, "steps": steps, "fit_us_median": round(statistics.median(per), 1), "fit_us_min": round(min(per), 1),
                     "fit_us_max": round(max(per), 1), "us_per_step": round(statistics.median(per) / steps, 4)})
    return rows


def torch_recon(xh, x, y, bins: int):
    """the counts and error sum of one segment from eager torch ops (ops.reference.recon_summary defines them)"""
    import torch
    d = (xh - x).double()
    e = (d * d).sum(1)
    valid = torch.isfinite(xh).all(1) & torch.isfinite(x).all(1) & ((y == 0) | (y == 1))
    u = e.float().view(torch.int32).long() & 0xFFFFFFFF
    sub = (bins // 32).bit_length() - 1
    b = (((u >> 23) - 103) << sub) + ((u & 0x7FFFFF) >> (23 - sub))
    b = torch.where(u < 0x33800000, 0, torch.where(u >= 0x43800000, bins - 1, b))
    counts = torch.bincount((2 + y.long() * bins + b)[valid], minlength=2 + 2 * bins)
    return counts, torch.where(valid, e, 0.0).sum()


def kernel_time(fn, iters: int) -> float:
    """device time per call of recon_summary_kernel and the memset in front of it (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    us = sum(ev.device_time for ev in prof.events()
             if ev.device_type.name == "CUDA" and ("recon_summary_kernel" in ev.name or "Memset" in ev.name))
    return us / iters


def summary_times(iters: int, passes: int) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    dev = torch.device("cuda", 0)
    rows = []
    for n in (100_000, 1_000_000, 10_000_000):
        g = torch.Generator(device=dev).manual_seed(n)
        x = torch.rand(n, 10, device=dev, generator=g)
        xh = x + 0.05 * torch.randn(n, 10, device=dev, generator=g)
        y = (torch.rand(n, device=dev, generator=g) < 0.1).float()
        fn = lambda: ops.recon_summary(xh, x, y, BINS)  # noqa: E731
        c0, s0, _, _ = fn()
        c1, s1 = torch_recon(xh, x, y, BINS)
        agree = bool(torch.equal(c0[0, 2:], c1[2:])) and abs(float(s0[0]) - float(s1)) <= 1e-9 * max(1.0, abs(float(s1)))
        k_us = kernel_time(fn, iters)
        call_us = events(fn, iters, passes)
        t_us = events(lambda: torch_recon(xh, x, y, BINS), iters, passes)
        b = n * (2 * 10 * 4 + 4)
        rows.append({"N": n, "bins": BINS, "bytes": b, "kernel_us": round(k_us, 2), "call_us": round(call_us, 2), "torch_us": round(t_us, 2),
                     "rows_per_s": round(n / (k_us * 1e-6)), "GBps": round(b / (k_us * 1e-6) / 1e9, 1),
                     "hbm_share": round(b / (k_us * 1e-6) / HBM_BYTES_PER_S, 4), "torch_over_kernel": round(t_us / k_us, 2),
                     "torch_agrees": agree})
    return rows


def main(argv=None) -> int:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--steps", type=int, default=8192)
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--passes", type=int, default=5)
    p.add_argument("--out", default=None)
    args = p.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "needs a CUDA device"}))
        return 1
    doc = {"gpu": gpu_info(), "fit": fit_times(args.steps, args.repeats), "recon_summary": summary_times(args.iters, args.passes),
           "gpu_after": gpu_info()}
    text = json.dumps(doc)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    return 0


if __name__ == "__main__":
    sys.exit(main())
