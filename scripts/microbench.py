"""Single-GPU micro-benchmarks of the hand-written kernels (CUDA-event timed, warmed up).

Usage: python scripts/microbench.py [--out gpurun_out/microbench.json] [--quick]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.models import FFNN, MLP, flatten_params


def time_cuda(fn, warmup=3, iters=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def bench_mlp(results, quick):
    dev = torch.device("cuda", 0)
    for name, ctor, loss in (("mlp64", MLP, "xent"), ("ffnn", FFNN, "bce")):
        model = ctor()
        spec = model.spec
        theta = flatten_params(model).to(dev)
        for variant, bsz, n in ((5, 1, 1024), (5, 1, 8192), (6, 1, 8192), (3, 1, 8192), (1, 1, 8192), (5, 32, 8192), (6, 32, 8192), (3, 32, 8192)):
            x = torch.rand(n, spec.dims[0], device=dev)
            y = (torch.rand(n, 1, device=dev) > 0.5).float()
            perm = ops.device_permutation(n, 1, 0, dev)
            out = torch.empty_like(theta)
            loss_out = torch.zeros(2, device=dev)
            task = ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=out, perm=perm, loss_out=loss_out)
            descs = ops.build_client_descs([task], dev)
            fn = lambda: ops.mlp_local_sgd_multi(spec.dims, spec.out_activation, descs, 1, bsz, 0.01, 1, -1, loss, variant=variant)
            med, best = time_cuda(fn)
            steps = (n + bsz - 1) // bsz
            results.append({"kernel": "mlp_local_sgd_persistent", "variant": variant, "net": name, "batch": bsz, "samples": n,
                            "ms": med, "ms_best": best, "us_per_step": 1e3 * med / steps,
                            "samples_per_s": n / (med * 1e-3)})
            print(results[-1], flush=True)
        # many clients in one launch (one CTA each)
        n, k = 1024, 132
        x = torch.rand(n, spec.dims[0], device=dev)
        y = (torch.rand(n, 1, device=dev) > 0.5).float()
        perm = ops.device_permutation(n, 1, 0, dev)
        slots = torch.empty(k, theta.numel(), device=dev)
        tasks = [ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=slots[i], perm=perm) for i in range(k)]
        descs = ops.build_client_descs(tasks, dev)
        fn = lambda: ops.mlp_local_sgd_multi(spec.dims, spec.out_activation, descs, k, 1, 0.01, 1, -1, loss)
        med, best = time_cuda(fn)
        results.append({"kernel": "mlp_local_sgd_persistent", "net": name, "batch": 1, "samples": n, "clients": k,
                        "ms": med, "us_per_step": 1e3 * med / n, "agg_samples_per_s": k * n / (med * 1e-3)})
        print(results[-1], flush=True)
        # torch eager comparator (same semantics, stock autograd + optim.SGD), short run
        m = ctor().to(dev)
        opt = torch.optim.SGD(m.parameters(), lr=0.01)
        xs = torch.rand(256, spec.dims[0], device=dev)
        ys = (torch.rand(256, 1, device=dev) > 0.5).float()
        lossf = (lambda o, t: torch.nn.functional.cross_entropy(o, t.view(-1).long())) if loss == "xent" else \
            (lambda o, t: torch.nn.functional.binary_cross_entropy(o, t))

        def eager():
            for i in range(256):
                opt.zero_grad()
                l = lossf(m(xs[i:i + 1]), ys[i:i + 1])
                l.backward()
                opt.step()
        med, best = time_cuda(eager, warmup=1, iters=3)
        results.append({"kernel": "torch_eager_sgd", "net": name, "batch": 1, "samples": 256, "ms": med,
                        "us_per_step": 1e3 * med / 256})
        print(results[-1], flush=True)


def bench_gemm(results, quick):
    dev = torch.device("cuda", 0)
    shapes = [(1024, 4096, 4096), (4096, 4096, 4096), (8192, 8192, 8192)]
    if quick:
        shapes = shapes[:2]
    for m, n, k in shapes:
        a = (torch.randn(m, k, device=dev) * 0.1).to(torch.bfloat16)
        b = (torch.randn(n, k, device=dev) * 0.1).to(torch.bfloat16)
        out = torch.empty(m, n, device=dev, dtype=torch.bfloat16)
        ref = lambda: torch.matmul(a, b.t())
        rmed, rbest = time_cuda(ref)
        fl = 2.0 * m * n * k
        for tile_n, cluster in ((256, 1), (256, 2)):
            fn = lambda: ops.gemm_bf16(a, b, out_bf16=out, tile_n=tile_n, cluster=cluster)
            med, best = time_cuda(fn)
            results.append({"kernel": "gemm_wgmma", "tile_n": tile_n, "cluster": cluster, "m": m, "n": n, "k": k, "ms": med,
                            "tflops": fl / med / 1e9, "tflops_best": fl / best / 1e9, "cublas_ms": rmed,
                            "cublas_tflops": fl / rmed / 1e9})
            print(results[-1], flush=True)


def bench_elementwise(results, quick):
    dev = torch.device("cuda", 0)
    n = 50_397_186 // 4 * 4
    p, g = torch.randn(n, device=dev), torch.randn(n, device=dev)
    med, _ = time_cuda(lambda: ops.sgd_step(p, g, 0.01))
    results.append({"kernel": "sgd_step", "n": n, "ms": med, "GBps": 3 * 4 * n / med / 1e6})
    print(results[-1], flush=True)
    k = 8
    slots = torch.randn(k, n, device=dev)
    w = torch.full((k,), 1.0 / k, device=dev)
    theta = torch.zeros(n, device=dev)
    med, _ = time_cuda(lambda: ops.fedavg_apply(theta, slots, w, 1.0))
    results.append({"kernel": "fedavg_apply", "n": n, "k": k, "ms": med, "GBps": (k + 2) * 4 * n / med / 1e6})
    print(results[-1], flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/microbench.json")
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    res = []
    for name, fn in (("mlp", bench_mlp), ("gemm", bench_gemm), ("elementwise", bench_elementwise)):
        if args.only and name not in args.only.split(","):
            continue
        try:
            fn(res, args.quick)
        except Exception as e:  # keep going: one broken kernel must not hide the others
            res.append({"kernel": name, "error": repr(e)})
            print(res[-1], flush=True)
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump({"gpu": torch.cuda.get_device_name(0), "results": res, "when": time.time()}, f, indent=1)
