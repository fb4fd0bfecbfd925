"""Cost of the detection-metrics summary of federated evaluation (``ops/csrc/eval_summary.cuh``, ``eval_summary_kernel``)
next to the same summary composed from torch ops.

    python scripts/eval_summary_bench.py [--rows 733672] [--iters 50] [--passes 5] [--out result.json]

N = 733,672 rows (the full Bot-IoT set) of C = 1 (the FFNN's sigmoid score) and C = 10 (logits) outputs, B = 256 bins, one
segment, two score distributions: ``uniform`` (scores spread over every bin) and ``one_bin`` (every row's score in one bin, the
shape of a trained detector's output, which makes every shared-memory histogram update hit the same counter).

``kernel_us``: device time of the memset + ``eval_summary_kernel`` pair, from ``torch.profiler`` (CUDA activities) over
--iters calls in a run of its own.  ``call_us``: CUDA events around --iters back-to-back ``ops.eval_summary`` calls (median
over --passes), which adds the host's work-unit table and its copy to the device.  ``torch_us``: the same counts and loss sum
from torch ops (validity mask, softmax, ``bincount`` of the confusion and histogram words, float64 loss sum), CUDA events
likewise.  Bytes: the N (4 C + 4) input bytes every variant must read once; ``hbm_share`` = those bytes over ``kernel_us``
against 3.35 TB/s (H100 SXM data sheet HBM3 bandwidth).  The card's name, power limit and SM clocks are read (nvidia-smi,
read-only queries) in the same run.  Prints one JSON line."""
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
BINS = 256


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        vals = [v.strip() for v in out.stdout.strip().splitlines()[0].split(",")]
        return dict(zip(q.split(","), vals))
    except Exception as e:  # noqa: BLE001 - the numbers are still reported, marked as without card information
        return {"error": repr(e)}


def inputs(C: int, dist: str, n: int, dev):
    import torch
    g = torch.Generator(device=dev).manual_seed(C)
    y = (torch.rand(n, device=dev, generator=g) > 0.5).float() if C == 1 else torch.randint(0, C, (n,), device=dev, generator=g).float()
    if C == 1:
        s = torch.rand(n, 1, device=dev, generator=g) if dist == "uniform" else torch.full((n, 1), 0.999, device=dev)
    elif dist == "uniform":
        s = 2 * torch.randn(n, C, device=dev, generator=g)
    else:
        s = torch.full((n, C), -20.0, device=dev)
        s[:, 0] = 20.0
    return s, y


def torch_summary(s, y, bins: int, thr: float):
    """the counts and loss sum of one segment from torch ops (the comparison; ops.reference.eval_summary defines them)"""
    import torch
    n, C = s.shape
    k = 2 if C == 1 else C
    lab_ok = (y >= 0) & (y < k) & (y == torch.floor(y))
    if C == 1:
        p = s[:, 0]
        valid = (p >= 0) & (p <= 1) & lab_ok
        yi = torch.where(valid, y, 0).long()
        pd = p.double()
        loss = torch.where(yi == 1, -torch.log(pd).clamp(min=-100), -torch.log1p(-pd).clamp(min=-100))
        words = torch.stack([2 + 2 * yi + (p > thr).long(), 2 + k * k + yi * bins + (p * bins).long().clamp(max=bins - 1)], 1)
    else:
        valid = torch.isfinite(s).all(1) & lab_ok
        yi = torch.where(valid, y, 0).long()
        z = s.double()
        m = z.max(1, keepdim=True).values
        e = torch.exp(z - m)
        tot = e.sum(1, keepdim=True)
        loss = torch.log(tot[:, 0]) - (z.gather(1, yi[:, None])[:, 0] - m[:, 0])
        cls = torch.arange(C, device=s.device)
        hist = 2 + k * k + (2 * cls[None, :] + (yi[:, None] == cls[None, :]).long()) * bins + ((e / tot) * bins).long().clamp(max=bins - 1)
        words = torch.cat([(2 + C * yi + s.argmax(1))[:, None], hist], 1)
    length = 2 + k * k + C * 2 * bins
    counts = torch.bincount(words[valid].reshape(-1), minlength=length)
    return counts, torch.where(valid, loss, torch.zeros_like(loss)).sum()


def events(fn, iters: int, passes: int) -> float:
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
        per.append(e0.elapsed_time(e1) * 1e3 / iters)
    return statistics.median(per)


def kernel_time(fn, iters: int) -> float:
    """device time per call of eval_summary_kernel and the memset in front of it (torch.profiler, CUDA activities)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    us = 0.0
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and ("eval_summary_kernel" in ev.name or "Memset" in ev.name):
            us += ev.device_time
    return us / iters


def run(args) -> list:
    import torch

    from colearn_federated_learning_b200 import ops
    dev = torch.device("cuda", 0)
    rows = []
    for C in (1, 10):
        for dist in ("uniform", "one_bin"):
            s, y = inputs(C, dist, args.rows, dev)
            fn = lambda: ops.eval_summary(s, y, BINS, 0.5)  # noqa: E731
            c0, l0 = fn()
            c1, l1 = torch_summary(s, y, BINS, 0.5)
            agree = bool(torch.equal(c0[0, 2:], c1[2:])) and abs(float(l0[0]) - float(l1)) <= 1e-9 * max(1.0, abs(float(l1)))
            k_us = kernel_time(fn, args.iters)
            call_us = events(fn, args.iters, args.passes)
            t_us = events(lambda: torch_summary(s, y, BINS, 0.5), args.iters, args.passes)
            b = args.rows * (4 * C + 4)
            rows.append({"C": C, "dist": dist, "N": args.rows, "bins": BINS, "bytes": b, "kernel_us": round(k_us, 2),
                         "call_us": round(call_us, 2), "torch_us": round(t_us, 2), "hbm_share": round(b / (k_us * 1e-6) / HBM_BYTES_PER_S, 4),
                         "GBps": round(b / (k_us * 1e-6) / 1e9, 1), "torch_over_kernel": round(t_us / k_us, 2),
                         "torch_agrees": agree})
    return rows


def main(argv=None) -> int:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rows", type=int, default=733_672)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--passes", type=int, default=5)
    p.add_argument("--out", default=None)
    args = p.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "needs a CUDA device"}))
        return 1
    doc = {"gpu": gpu_info(), "eval_summary": run(args), "gpu_after": gpu_info()}
    text = json.dumps(doc)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)
    return 0


if __name__ == "__main__":
    sys.exit(main())
