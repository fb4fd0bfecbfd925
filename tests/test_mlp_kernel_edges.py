"""The persistent MLP kernel (csrc/mlp_v2.cuh, variants 3 / 5 / 6; csrc/mlp_persistent.cu, variant 1) and its batched
forward against float64 at the edges where the kernel's bookkeeping changes: the CHUNK = 64 sample chunks (the deferred
batch-1 updates are flushed at every chunk end), batches that end short or span two chunks, ``max_nr_batches`` cutting an
epoch, permutation tables with fewer rows than epochs, the in-kernel shuffle, the write-out scale / delta, empty shards,
many clients in one launch, saturated heads and non-finite data.

The oracle is ``reference.mlp_local_sgd`` / ``mlp_forward`` in float64 from the same fp32 parameters and data, replayed
step by step (``_replay``) so that every step's loss is kept.  What is compared is the UPDATE ``Δ = θ_out − θ_0``, so the
bound scales with what the kernel computed, not with the parameters it started from:

* fits of 1-3 steps: an elementwise running-error bound (``_replay(absolute=True)``).  The reference is replayed on absolute
  values — ``|W|``, ``|x|``, ``|dz|`` — which gives, per parameter, the sum of the magnitudes that its fp32 dot products
  and rank-1 updates accumulate; times ``γ_k = k·u / (1 − k·u)`` with ``k`` the longest chain of roundings of one step
  (every fan-in, forward and back, plus the update).  The head adds the documented error of its MUFU instructions
  (``ex2.approx`` 2 ulp, ``rcp.approx`` 1 ulp, ``mlp_v2.cuh`` above ``exp_nonpos``) and the argument scaling ``z·log2 e``
  (``|z|`` ulp), carried back through the same absolute replay; each fp32 store of a weight adds ``u·|θ|``.
* longer fits, where fp32 rounding compounds: ``‖Δ − Δ64‖∞ ≤ C·‖Δ32 − Δ64‖∞ + 2⁻²⁰·‖Δ64‖∞`` with ``Δ32`` the fp32
  reference.  Kernel and fp32 reference run the same recurrence in fp32 and differ only in the order of the additions
  inside a dot product and in the head's approximations (≤ 3 ulp against libm's ≤ 1), so their distances from float64 are
  the same kind of random walk with steps at most ~4× longer: ``C = 8`` leaves a factor 2 for the walk.

Every test records its largest error as a fraction of its bound (printed at module end: run with ``-s``).

The CPU group (no mark) runs the kernel source through the SIMT build (``build.build_simt_emul``, one OS thread per
CUDA thread, so the shards are small); the ``gpu`` group runs the same cases, more of them and larger, on the device, and
adds what only a device shows: nvcc's bits against the claims (variant 6 = variant 5, run-to-run identity) and 300
clients in one launch.
"""
import importlib.util
import math
import os
import shutil

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200.models import build_model, flatten_params
from colearn_federated_learning_b200.ops import reference as R

gpu = pytest.mark.gpu
U = 2.0 ** -24
LR = float(np.float32(0.05))      # the kernel's fp32 learning rate, exactly
C_LONG = 8.0
NETS = {"ffnn": (0, (10, 50, 30, 10, 1), "sigmoid"), "mlp": (1, (10, 64, 64, 2), "none"),
        "testing_remote": (2, (2, 50, 10, 1), "none")}
NET_LOSSES = [("ffnn", "bce"), ("ffnn", "sse"), ("ffnn", "mse"), ("mlp", "xent"), ("testing_remote", "sse"),
              ("testing_remote", "mse")]
LOSS_CODES = {"bce": 0, "sse": 1, "xent": 2, "mse": 3}
FRACTIONS = {}


def _record(name, frac):
    FRACTIONS[name] = max(FRACTIONS.get(name, 0.0), float(frac))


@pytest.fixture(scope="module", autouse=True)
def _report_fractions():
    yield
    if FRACTIONS:
        print("\nlargest error / bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(FRACTIONS.items())))


# ---- data ------------------------------------------------------------------------------------------------------------
def _theta0(net):
    torch.manual_seed(NETS[net][0])
    return flatten_params(build_model(net)).clone()


def _data(net, loss, n, seed=0):
    dims = NETS[net][1]
    g = torch.Generator().manual_seed(1000 + 17 * n + seed)
    x = torch.rand(n, dims[0], generator=g)
    y = (torch.randint(0, dims[-1], (n, 1), generator=g).float() if loss == "xent"
         else (torch.rand(n, dims[-1], generator=g) > 0.5).float())
    return x, y


def _perm(n, rows, seed=5):
    return R.make_permutation(n, rows, seed) if n > 0 else torch.zeros(rows, 0, dtype=torch.int32)


# ---- float64 oracle ----------------------------------------------------------------------------------------------------
def _softplus_bce(z, y):
    """BCE of sigmoid(z) in the kernel's form max(z, 0) + log(1 + e^-|z|) − y·z.  The reference clamps log at −100 like
    F.binary_cross_entropy, which bites once sigmoid(z) rounds to 1 (|z| > ~100 in float64, ~17 in fp32): there the two
    differ by definition, and the kernel's value is the exact one."""
    return (torch.clamp(z, min=0) + torch.log1p(torch.exp(-z.abs())) - y * z).mean()


def _replay(theta0, net, loss, x, y, perm, B, epochs, max_b, dtype=torch.float64, absolute=False):
    """``reference.mlp_local_sgd`` step by step.  Returns (θ, [loss of every step], bound accumulator or None).

    absolute=True also accumulates, per parameter, Σ_steps lr·(D ⊗ |a|) where |a| is the forward on absolute values and D
    the backward of the head's error budget on absolute weights (see the module docstring)."""
    _, dims, act = NETS[net]
    flat = theta0.to(dtype).clone()
    n = x.shape[0]
    x, y = x.to(dtype), y.to(dtype)
    limit = max_b if max_b > 0 else None
    losses, it = [], 0
    acc = torch.zeros_like(flat) if absolute else None
    L = len(dims) - 1
    k = sum(dims[i] + dims[i + 1] + 4 for i in range(L))          # longest rounding chain of one step
    gam = k * U / (1 - k * U)
    for e in range(epochs):
        order = perm[e % perm.shape[0]].long()
        for lo in range(0, n, B):
            idx = order[lo:lo + B]
            xb, yb = x[idx], y[idx]
            out, acts = R.mlp_forward(flat, dims, xb, act)
            value, dz = R.loss_and_dz(out, yb, loss, act)
            if loss == "bce":
                z = R.mlp_forward(flat, dims, xb, "none")[0]
                value = _softplus_bce(z, yb.reshape(z.shape))
            g = R.mlp_backward(flat, dims, acts, dz)
            if absolute:
                views = R.mlp_views(flat, dims)
                h, aabs = xb.abs(), []
                for w, b in views:
                    aabs.append(h)
                    h = h @ w.abs().t() + b.abs()
                zabs = h
                z = R.mlp_forward(flat, dims, xb, "none")[0]
                scale = {"bce": 1.0 / z.numel(), "xent": 1.0 / xb.shape[0], "mse": 1.0 / xb.shape[0], "sse": 1.0}[loss]
                # |dz_L| as a magnitude (every operand of its formula taken absolutely) ...
                if loss == "xent":
                    mag = (torch.softmax(z, 1) + 1.0) * scale
                elif act == "sigmoid" and loss != "bce":
                    mag = 2 * (out.abs() + yb.abs().reshape(out.shape)) * (out.abs() + (1 - out).abs()) * scale
                else:
                    mag = (out.abs() + yb.abs().reshape(out.shape)) * (2.0 if loss != "bce" else 1.0) * scale
                # ... times γ_k, plus the head's own budget: MUFU ex2 (2 ulp) + rcp (1 ulp) + the rounding of z·log2(e) (|z| ulp)
                # + 5 fp32 roundings of the sigmoid / softmax formula, and the forward error of the logits (γ_k·|z|abs) through
                # the loss derivative (≤ 2·scale)
                mufu = (8 + 2 * z.abs()) * U if loss == "xent" or act == "sigmoid" else torch.zeros_like(z)
                if loss == "xent":
                    mufu = (8 + 2 * (z[:, 1:] - z[:, :1]).abs()) * U * torch.ones_like(z)
                D = gam * mag + mufu * mag + 2 * scale * gam * zabs
                for li in range(L - 1, -1, -1):
                    w, _ = views[li]
                    gw, gb = R.mlp_views(acc, dims)[li]
                    gw += LR * (D.t() @ aabs[li])
                    gb += LR * D.sum(0)
                    if li > 0:
                        D = (D @ w.abs()) * (acts[li] != 0).to(dtype)
            flat.sub_(LR * g)
            losses.append(value)
            it += 1
            if limit is not None and it >= limit:
                return flat, losses, acc
    return flat, losses, acc


def _steps(n, B, epochs, max_b):
    return 0 if n == 0 else R.total_steps(n, B, epochs, max_b)


def _reference(net, loss, x, y, perm, B, epochs, max_b, theta0):
    """(steps, float64 replay with the absolute one for short fits, fp32 replay for long fits)"""
    steps = _steps(x.shape[0], B, epochs, max_b)
    if steps == 0:
        return steps, None, None
    r64 = _replay(theta0, net, loss, x, y, perm, B, epochs, max_b, absolute=steps <= 3)
    r32 = _replay(theta0, net, loss, x, y, perm, B, epochs, max_b, dtype=torch.float32) if steps > 3 else None
    return steps, r64, r32


def _check_fit(tag, ref, theta0, got, got_losses):
    """got: fp32 θ_out at out_scale 1, got_losses: [last, mean] — against the replays of _reference."""
    steps, (ref64, l64, acc), r32 = ref[0], ref[1] or (None, None, None), ref[2]
    if steps == 0:
        assert torch.equal(got, theta0) and got_losses.tolist() == [0.0, 0.0]
        return
    d = got.double() - theta0.double()
    d64 = ref64 - theta0.double()
    err = (d - d64).abs()
    if steps <= 3:
        bound = steps * acc + steps * U * (theta0.double().abs() + d64.abs())
        frac = torch.where(err == 0, 0.0, err / bound).max().item()
        _record(f"{tag} Δ ≤ running bound", frac)
        assert frac <= 1.0, (tag, frac, err.max().item())
        ltol = lambda v: 2.0 ** -16 * (1 + abs(v))                             # noqa: E731
        lref = [float(l64[-1]), float(sum(l64) / len(l64))]
        for what, g, r in (("last", got_losses[0], lref[0]), ("mean", got_losses[1], lref[1])):
            f = abs(float(g) - r) / ltol(r)
            _record(f"{tag} loss {what}", f)
            assert f <= 1.0, (tag, what, float(g), r)
    else:
        ref32, l32, _ = r32
        d32 = ref32.double() - theta0.double()
        bound = C_LONG * (d32 - d64).abs().max().item() + 2.0 ** -20 * d64.abs().max().item()
        frac = err.max().item() / bound
        _record(f"{tag} ‖Δ‖ ≤ C·‖Δ32‖", frac)
        assert frac <= 1.0, (tag, frac)
        m64, m32 = float(sum(l64) / len(l64)), float(sum(l32) / len(l32))
        for what, g, r, r32 in (("last", got_losses[0], float(l64[-1]), float(l32[-1])), ("mean", got_losses[1], m64, m32)):
            b = C_LONG * abs(r32 - r) + 2.0 ** -16 * (1 + abs(r))
            f = abs(float(g) - r) / b
            _record(f"{tag} loss {what}", f)
            assert f <= 1.0, (tag, what, float(g), r, r32)


# ---- executors: the SIMT build on the CPU, the device ------------------------------------------------------------------
class Simt:
    def __init__(self, mod):
        self.m = mod

    def fit(self, net, loss, clients, B, epochs, max_b, variant, delta=False, flags=None):
        """clients: dicts x, y, perm (or perm_seed + perm_row0), out_scale, theta_in.  -> (outs [K, P], losses [K, 2])."""
        kind = NETS[net][0]
        theta_in = clients[0]["theta_in"]
        outs = [torch.full_like(theta_in, 7.0) for _ in clients]
        seed = clients[0].get("perm_seed", 0)
        kw = {}
        if seed:
            kw = dict(perm_seed=seed, perm_row0=clients[0]["perm_row0"],
                      perm_scratch=torch.full((len(clients), max(1, epochs * max(c["x"].shape[0] for c in clients))), -1, dtype=torch.int32))
        losses = self.m.mlp_local_sgd(kind, theta_in, outs, [c["x"] for c in clients], [c["y"] for c in clients],
                                      [c.get("perm") for c in clients], B, epochs, max_b, LOSS_CODES[loss], LR, variant,
                                      [c.get("out_scale", 1.0) for c in clients], delta, flags, **kw)
        return torch.stack(outs), losses

    def forward(self, net, theta, x):
        return self.m.mlp_forward(NETS[net][0], theta, x, NETS[net][1][-1])

    def table(self, n, rows, seed):
        return self.m.feistel_permutation(n, rows, seed)


class Device:
    def __init__(self):
        from colearn_federated_learning_b200 import ops
        self.ops, self.dev = ops, torch.device("cuda", 0)

    def fit(self, net, loss, clients, B, epochs, max_b, variant, delta=False, flags=None, desc_offset=0):
        ops, dev = self.ops, self.dev
        _, dims, act = NETS[net]
        K = len(clients)
        P = clients[0]["theta_in"].numel()
        # every slot and loss pair sits between 7.0 borders: a write outside them shows
        slots = torch.full((K, P + 8), 7.0, device=dev)
        lo = torch.full((K, 4), 7.0, device=dev)
        keep, tasks = [], []
        for i, c in enumerate(clients):
            x, y = c["x"].to(dev), c["y"].to(dev)
            th = c["theta_in"].to(dev)
            kw = {}
            if c.get("perm") is not None:
                kw["perm"] = c["perm"].to(dev, torch.int32).contiguous()
            elif c.get("perm_seed"):
                kw.update(perm_seed=c["perm_seed"], perm_row0=c["perm_row0"],
                          perm_scratch=torch.full((max(1, epochs * x.shape[0]),), -1, dtype=torch.int32, device=dev))
            if flags is not None:
                kw.update(signal_flag=flags[i], signal_value=7 + i, wait_flag=flags[K + i], wait_value=1)
            keep += [x, y, th, kw]
            tasks.append(ops.ClientTask(x=x, y=y, theta_in=th, theta_out=slots[i, 4:4 + P], loss_out=lo[i, 1:3],
                                        out_scale=c.get("out_scale", 1.0), delta_mode=c.get("delta", delta), **kw))
        pad = [ops.ClientTask(x=keep[0], y=keep[1], theta_in=keep[2], theta_out=slots[0, 4:4 + P])] * desc_offset
        descs = ops.build_client_descs(pad + tasks, dev)
        ops.mlp_local_sgd_multi(dims, act, descs, K, batch_size=B, lr=LR, epochs=epochs, max_nr_batches=max_b, loss=loss,
                                desc_offset=desc_offset, variant=variant)
        torch.cuda.synchronize()
        slots, lo = slots.cpu(), lo.cpu()
        assert bool((slots[:, :4] == 7).all() and (slots[:, 4 + P:] == 7).all()), "write outside theta_out"
        assert bool((lo[:, 0] == 7).all() and (lo[:, 3] == 7).all()), "write outside loss_out"
        return slots[:, 4:4 + P].clone(), lo[:, 1:3].clone()

    def forward(self, net, theta, x):
        _, dims, act = NETS[net]
        out = self.ops.mlp_forward(theta.to(self.dev), dims, x.to(self.dev), act)
        torch.cuda.synchronize()
        return out.cpu()

    def table(self, n, rows, seed):
        return self.ops.device_permutation(n, rows, seed, self.dev).cpu()


@pytest.fixture(scope="module")
def simt():
    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return Simt(mod)


@pytest.fixture(scope="module")
def device():
    return Device()


# ---- the cases ---------------------------------------------------------------------------------------------------------
def _fit_case(ex, tag, net, loss, n, B, epochs, max_b, variants, perm_rows=None, seed_row0=None, bits_pairs=False):
    theta0 = _theta0(net)
    x, y = _data(net, loss, n)
    c = dict(x=x, y=y, theta_in=theta0)
    if seed_row0 is not None:
        seed = 987654321
        c.update(perm_seed=seed, perm_row0=seed_row0)
        perm = ex.table(n, seed_row0 + epochs, seed)[seed_row0:] if n > 0 else torch.zeros(epochs, 0, dtype=torch.int32)
    else:
        perm = _perm(n, perm_rows or epochs)
        c["perm"] = perm
    ref = _reference(net, loss, x, y, perm, B, epochs, max_b, theta0)
    results = {}
    for v in variants:
        outs, losses = ex.fit(net, loss, [c], B, epochs, max_b, v)
        results[v] = (outs[0], losses[0])
        _check_fit(tag, ref, theta0, outs[0], losses[0])
    if bits_pairs:
        if 5 in results and 6 in results:
            assert torch.equal(results[5][0], results[6][0]) and torch.equal(results[5][1], results[6][1]), "variant 6 != 5"
        v = variants[0]
        outs, losses = ex.fit(net, loss, [c], B, epochs, max_b, v)
        assert torch.equal(outs[0], results[v][0]) and torch.equal(losses[0], results[v][1]), "two launches differ"
    return results


BATCH1_N = [0, 1, 2, 63, 64, 65, 127, 128, 129, 1000]
CPU_BATCH1_N = [0, 1, 2, 63, 64, 65, 127, 129]
BATCHES = [2, 7, 63, 64, 65, 100]


# --- CPU group (SIMT build of the kernel source) ---
@pytest.mark.parametrize("net,loss", NET_LOSSES)
@pytest.mark.parametrize("n", CPU_BATCH1_N)
def test_batch1_chunk_edges_cpu(simt, net, loss, n):
    variants = (5, 1, 3, 6) if n in (1, 65) else (5,)
    _fit_case(simt, "cpu b1", net, loss, n, 1, 1, -1, variants)


@pytest.mark.parametrize("net,loss", [("ffnn", "bce"), ("mlp", "xent"), ("testing_remote", "mse")])
@pytest.mark.parametrize("B,n", [(2, 9), (7, 75), (63, 130), (64, 129), (65, 131), (100, 203), (9, 9), (12, 7), (5, 0)])
def test_batches_cpu(simt, net, loss, B, n):
    _fit_case(simt, "cpu batch", net, loss, n, B, 2, -1, (5, 1) if B in (7, 65) else (5,))


@pytest.mark.parametrize("B,n,epochs,max_b,rows", [(1, 20, 3, 13, None), (7, 30, 3, 6, None), (1, 20, 2, 20, None),
                                                   (7, 30, 2, 100, None), (1, 23, 3, -1, 2), (7, 23, 5, -1, 2)])
def test_max_batches_and_short_tables_cpu(simt, B, n, epochs, max_b, rows):
    for net, loss in (("ffnn", "sse"), ("mlp", "xent")):
        _fit_case(simt, "cpu max_b", net, loss, n, B, epochs, max_b, (5, 1), perm_rows=rows)


@pytest.mark.parametrize("net,loss", [("ffnn", "bce"), ("mlp", "xent")])
def test_in_kernel_shuffle_row0_cpu(simt, net, loss):
    _fit_case(simt, "cpu perm_seed", net, loss, 70, 1, 2, -1, (5, 3), seed_row0=3)


def test_out_scale_delta_and_empty_clients_cpu(simt):
    """out_scale × delta_mode gives fl(s·θ) / fl(s·(θ − θ_in)) of the kernel's own scale-1 result, bit for bit, and the
    completion flag is raised for every client, empty ones (n = 0) included."""
    for net, loss in (("ffnn", "bce"), ("mlp", "xent")):
        theta0 = _theta0(net)
        clients = []
        for i, n in enumerate((0, 1, 64, 65)):
            x, y = _data(net, loss, n, seed=i)
            clients.append(dict(x=x, y=y, perm=_perm(n, 1), theta_in=theta0))
        base, base_l = simt.fit(net, loss, clients, 1, 1, -1, 5)
        for delta in (False, True):
            for s in (1.0, 0.37, 0.0, -1.0):
                flags = torch.zeros(len(clients), dtype=torch.int32)
                outs, losses = simt.fit(net, loss, [dict(c, out_scale=s) for c in clients], 1, 1, -1, 5, delta=delta, flags=flags)
                want = (base - theta0) if delta else base
                assert torch.equal(outs, (torch.tensor(s, dtype=torch.float32) * want)), (net, delta, s)
                assert torch.equal(losses, base_l)
                assert flags.tolist() == [7 + i for i in range(len(clients))]


@pytest.mark.parametrize("net,loss,scale", [("ffnn", "bce", 20), ("ffnn", "bce", 60), ("ffnn", "bce", 100), ("ffnn", "sse", 20),
                                            ("ffnn", "sse", 100), ("mlp", "xent", 20), ("mlp", "xent", 60), ("mlp", "xent", 100)])
def test_saturated_heads_cpu(simt, net, loss, scale):
    _saturated(simt, net, loss, scale, (5, 1))


@pytest.mark.parametrize("net,loss", NET_LOSSES[:2] + NET_LOSSES[3:5])
@pytest.mark.parametrize("what", ["x_nan", "x_inf", "x_-inf", "y_nan"])
def test_non_finite_data_cpu(simt, net, loss, what):
    _non_finite(simt, net, loss, what, (5, 1, 3))


@pytest.mark.parametrize("net", list(NETS))
def test_forward_cpu(simt, net):
    _forward(simt, net, (1, 263, 265))


def test_replay_is_the_reference():
    """The step-by-step replay above is reference.mlp_local_sgd (same final parameters, same last loss)."""
    for net, loss in NET_LOSSES:
        theta0 = _theta0(net)
        x, y = _data(net, loss, 23)
        perm = _perm(23, 2)
        for B, max_b in ((1, -1), (5, 7)):
            flat, losses, _ = _replay(theta0, net, loss, x, y, perm, B, 3, max_b)
            ref = theta0.double().clone()
            last = R.mlp_local_sgd(ref, NETS[net][1], x.double(), y.double(), perm, B, LR, 3, max_b, loss, NETS[net][2])
            assert torch.equal(flat, ref) and len(losses) == R.total_steps(23, B, 3, max_b)
            assert math.isclose(float(losses[-1]), float(last), rel_tol=1e-12)


# ---- shared bodies ---------------------------------------------------------------------------------------------------
def _saturated(ex, net, loss, scale, variants):
    """The head's weights scaled so that the logits reach ±scale: one step, gradient finite and within the bound.  BCE at
    |z| ≥ 88: the kernel's softplus loss is pinned (the reference's clamped log gives a different number by definition)."""
    _, dims, act = NETS[net]
    theta0 = _theta0(net)
    w, b = R.mlp_views(theta0, dims)[-1]
    x, y = _data(net, loss, 4)
    h = R.mlp_forward(theta0, dims, x, "none")[1][-1]                     # the head's inputs
    for v in variants:
        for i in range(4):
            th = theta0.clone()
            hw, hb = R.mlp_views(th, dims)[-1]
            z = h[i] @ w.t() + b
            sign = 1.0 if i % 2 == 0 else -1.0
            if loss == "xent":                                      # z1 − z0 = ±scale
                f = sign * scale / float(z[1] - z[0])
                hw[1], hb[1] = hw[0] + (hw[1] - hw[0]) * f, hb[0] + (hb[1] - hb[0]) * f
            else:                                                   # z = ±scale
                f = sign * scale / float(z[0])
                hw.mul_(f)
                hb.mul_(f)
            xi, yi = x[i:i + 1], y[i:i + 1]
            outs, losses = ex.fit(net, loss, [dict(x=xi, y=yi, perm=_perm(1, 1), theta_in=th)], 1, 1, -1, v)
            assert bool(torch.isfinite(outs[0]).all()), (net, loss, scale, v)
            if v == 1 and loss == "bce":
                # variant 1 computes BCE from the rounded probability with the reference's clamp (fp32: 100 once |z| > ~17)
                zz = R.mlp_forward(th, dims, xi, "none")[0]
                want = float(R.loss_and_dz(torch.sigmoid(zz), yi, "bce", "sigmoid")[0])
                assert math.isclose(float(losses[0, 0]), want, rel_tol=1e-4), (float(losses[0, 0]), want)
                continue
            _check_fit(f"saturated {loss}", _reference(net, loss, xi, yi, _perm(1, 1), 1, 1, -1, th), th, outs[0],
                       losses[0])


def _non_finite(ex, net, loss, what, variants):
    """One NaN / ±inf feature or a NaN label in a 5-sample shard: the non-finite parameters of the kernel's model are the
    float64 reference's, layer by layer, and the reported mean loss is NaN when the reference's is."""
    if what == "y_nan" and loss == "xent":
        pytest.skip("xent labels are class indices")
    _, dims, act = NETS[net]
    theta0 = _theta0(net)
    x, y = _data(net, loss, 5)
    if what == "y_nan":
        y[2, 0] = float("nan")
    else:
        x[2, 1] = float(what[2:])
    perm = _perm(5, 1)
    ref, l64, _ = _replay(theta0, net, loss, x, y, perm, 1, 1, -1)
    ref_mean = float(sum(l64) / len(l64))
    for v in variants:
        outs, losses = ex.fit(net, loss, [dict(x=x, y=y, perm=perm, theta_in=theta0)], 1, 1, -1, v)
        for li, ((gw, gb), (rw, rb)) in enumerate(zip(R.mlp_views(outs[0], dims), R.mlp_views(ref, dims))):
            assert torch.equal(~torch.isfinite(gw), ~torch.isfinite(rw)), (what, v, li, "W")
            assert torch.equal(~torch.isfinite(gb), ~torch.isfinite(rb)), (what, v, li, "b")
        assert math.isnan(float(losses[0, 1])) == math.isnan(ref_mean), (what, v, float(losses[0, 1]), ref_mean)
        assert not torch.isfinite(outs[0]).all(), (what, v)


def _forward(ex, net, sizes):
    """mlp_forward (grid capped at 264 CTAs: 265 and above take the grid-stride pass) against float64, NaN rows included."""
    _, dims, act = NETS[net]
    theta = _theta0(net)
    L = len(dims) - 1
    k = sum(dims[i] + 4 for i in range(L))
    gam = k * U / (1 - k * U)
    for n in sizes:
        g = torch.Generator().manual_seed(n)
        x = torch.rand(n, dims[0], generator=g) * 2 - 1
        nan_rows = [r for r in (0, n // 2, n - 1) if n > 2]
        for r in nan_rows:
            x[r, r % dims[0]] = float("nan")
        got = ex.forward(net, theta, x).double()
        want = R.mlp_forward(theta.double(), dims, x.double(), act)[0]
        h = x.double().abs()
        for w, b in R.mlp_views(theta.double(), dims):
            h = h @ w.abs().t() + b.abs()
        z = R.mlp_forward(theta.double(), dims, x.double(), "none")[0]
        bound = gam * h
        if act == "sigmoid":        # σ' ≤ 1/4 carries the logit error; __expf (2 ulp + |z| ulp of the argument) + the division
            bound = bound / 4 + (8 + 2 * z.abs()) * U * want.abs()
        bad = ~torch.isfinite(want)
        assert torch.equal(bad, ~torch.isfinite(got)), (net, n)
        assert bad.any(dim=1).sum().item() == len(nan_rows)
        ok = ~bad
        frac = ((got - want).abs()[ok] / bound[ok]).max().item()
        _record(f"forward {net}", frac)
        assert frac <= 1.0, (net, n, frac)


# --- GPU group (the same cases on the device, plus what only a device shows) ---
@gpu
@pytest.mark.parametrize("net,loss", NET_LOSSES)
@pytest.mark.parametrize("n", BATCH1_N)
def test_batch1_chunk_edges_gpu(device, net, loss, n):
    _fit_case(device, "gpu b1", net, loss, n, 1, 1, -1, (5, 6, 3, 1), bits_pairs=True)


@gpu
@pytest.mark.parametrize("net,loss", NET_LOSSES)
@pytest.mark.parametrize("B", BATCHES)
def test_batches_gpu(device, net, loss, B):
    for n in (203, B, B + 5, 0):
        _fit_case(device, "gpu batch", net, loss, n, B, 2, -1, (5, 6, 3, 1), bits_pairs=True)


@gpu
@pytest.mark.parametrize("B,n,epochs,max_b,rows", [(1, 100, 3, 150, None), (7, 100, 3, 20, None), (1, 100, 2, 100, None),
                                                   (7, 100, 2, 1000, None), (1, 97, 5, -1, 2), (7, 97, 5, -1, 3)])
def test_max_batches_and_short_tables_gpu(device, B, n, epochs, max_b, rows):
    for net, loss in NET_LOSSES:
        _fit_case(device, "gpu max_b", net, loss, n, B, epochs, max_b, (5, 6, 3, 1), perm_rows=rows,
                  bits_pairs=True)


@gpu
@pytest.mark.parametrize("net,loss", [("ffnn", "bce"), ("mlp", "xent"), ("testing_remote", "sse")])
def test_in_kernel_shuffle_row0_gpu(device, net, loss):
    _fit_case(device, "gpu perm_seed", net, loss, 333, 1, 3, -1, (5, 6, 3, 1), seed_row0=5, bits_pairs=True)


@gpu
@pytest.mark.parametrize("net,loss", [("ffnn", "bce"), ("mlp", "xent"), ("testing_remote", "mse")])
@pytest.mark.parametrize("B", [1, 7])
def test_many_clients_one_launch_gpu(device, net, loss, B):
    """300 clients (more than two waves of 132 CTAs), mixed n / out_scale / delta_mode, descriptors at an offset: each
    client's output and losses are those of the same client launched alone, bit for bit; completion flags raised."""
    theta0 = _theta0(net)
    sizes = (0, 1, 64, 65, 203)
    clients = []
    for i in range(300):
        n = sizes[i % 5]
        x, y = _data(net, loss, n, seed=i)
        clients.append(dict(x=x, y=y, perm=_perm(n, 2, seed=i), theta_in=theta0, out_scale=(1.0, 0.37, 0.0, -1.0)[i % 4],
                            delta=(i // 5) % 2 == 1))
    flags = torch.zeros(600, dtype=torch.int32, device=device.dev)
    flags[300:] = 1                                           # the "broadcast has landed" words the clients wait on
    for v in (5, 1):
        outs, losses = device.fit(net, loss, clients, B, 2, -1, v, flags=[flags[i:i + 1] for i in range(600)], desc_offset=3)
        assert flags[:300].cpu().tolist() == [7 + i for i in range(300)]
        flags[:300] = 0
        for i in range(0, 300, 7 if v == 5 else 23):
            o, lo = device.fit(net, loss, [clients[i]], B, 2, -1, v)
            assert torch.equal(outs[i], o[0]) and torch.equal(losses[i], lo[0]), (v, i)
            if clients[i]["x"].shape[0] == 0:
                want = torch.zeros_like(theta0) if clients[i]["delta"] else theta0
                assert torch.equal(outs[i], torch.tensor(clients[i]["out_scale"], dtype=torch.float32) * want) and losses[i].tolist() == [0.0, 0.0]


@gpu
@pytest.mark.parametrize("net,loss", [("ffnn", "bce"), ("mlp", "xent"), ("testing_remote", "sse")])
def test_out_scale_delta_gpu(device, net, loss):
    theta0 = _theta0(net)
    for B, n in ((1, 65), (7, 65), (1, 0)):
        x, y = _data(net, loss, n)
        c = dict(x=x, y=y, perm=_perm(n, 2), theta_in=theta0)
        for v in (5, 6, 3, 1):
            base, base_l = device.fit(net, loss, [c], B, 2, -1, v)
            for delta in (False, True):
                for s in (1.0, 0.37, 0.0, -1.0):
                    o, lo = device.fit(net, loss, [dict(c, out_scale=s, delta=delta)], B, 2, -1, v)
                    want = (base[0] - theta0) if delta else base[0]
                    assert torch.equal(o[0], torch.tensor(s, dtype=torch.float32) * want), (v, B, n, delta, s)
                    assert torch.equal(lo, base_l)


@gpu
@pytest.mark.parametrize("net,loss,scale", [(a, b, s) for a, b in (("ffnn", "bce"), ("ffnn", "sse"), ("mlp", "xent"))
                                            for s in (20, 60, 100)])
def test_saturated_heads_gpu(device, net, loss, scale):
    _saturated(device, net, loss, scale, (5, 6, 3, 1))


@gpu
@pytest.mark.parametrize("net,loss", NET_LOSSES)
@pytest.mark.parametrize("what", ["x_nan", "x_inf", "x_-inf", "y_nan"])
def test_non_finite_data_gpu(device, net, loss, what):
    _non_finite(device, net, loss, what, (5, 6, 3, 1))


@gpu
@pytest.mark.parametrize("net", list(NETS))
def test_forward_gpu(device, net):
    _forward(device, net, (1, 263, 264, 265, 100_003))
