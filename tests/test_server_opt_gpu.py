"""Server optimizers (FedAvgM / FedAdagrad / FedAdam / FedYogi) fused into the FedAvg kernels on the GPU: ops.fedavg_apply,
the star round (verify_round) and the two-shot round, against the PyTorch definition (ops.reference.server_opt_step).

Tolerances as in test_server_opt.py: the kernels sum the average in their own fp32 order and use fmaf inside the step, a few
ulps of the average that m / (sqrt(v) + tau) turns into a relative error of the same order in the step."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.ops import reference

pytestmark = pytest.mark.gpu

OPT_KINDS = ["avgm", "adagrad", "adam", "yogi"]


def _opt(kind):
    return ServerOpt(kind, lr=0.05 if kind != "avgm" else 0.8)


def _tol(kind):
    return dict(rtol=1e-6, atol=1e-6) if kind == "avgm" else dict(rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("kind", ["sgd"] + OPT_KINDS)
@pytest.mark.parametrize("n", [4096 * 3, 1001])
def test_fedavg_apply_with_server_optimizer(kind, n):
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(n)
    opt = _opt(kind)
    st, ref = opt.init_state(n, dev), opt.init_state(n)
    theta = torch.randn(n, generator=g)
    th = theta.to(dev)
    w = torch.tensor([0.2, 0.3, 0.5])
    for _ in range(3):
        models = theta + 0.5 * torch.randn(3, n, generator=g)
        ops.fedavg_apply(th, models.to(dev), w.to(dev), opt=st)
        reference.server_opt_apply(theta, models, w, kind, opt.lr, ref.m, ref.v, opt.beta1, opt.beta2, opt.tau)
        torch.cuda.synchronize()
        torch.testing.assert_close(th.cpu(), theta, **_tol(kind))
        if ref.m is not None:
            torch.testing.assert_close(st.m.cpu(), ref.m, **_tol(kind))
        if ref.v is not None:
            torch.testing.assert_close(st.v.cpu(), ref.v, rtol=1e-5, atol=1e-8)
        theta = th.cpu()                                    # keep both sides on the same trajectory
        ref.m = st.m.cpu() if st.m is not None else None
        ref.v = st.v.cpu() if st.v is not None else None
    if kind == "sgd":                                       # plain FedAvg: the existing kernel, bit for bit
        a, b = th.clone(), th.clone()
        ops.fedavg_apply(a, models.to(dev), w.to(dev), opt=st)
        ops.fedavg_apply(b, models.to(dev), w.to(dev), opt.lr)
        assert torch.equal(a, b)


@pytest.mark.parametrize("kind", OPT_KINDS)
def test_star_engine_verify_round_with_server_optimizer(kind):
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=7, server_opt=_opt(kind))
    x, y = synthetic_unsw(200, seed=3)
    eng.set_local_data(x, y)
    for _ in range(3):
        m0 = eng.server_state()["m"].clone()
        res = eng.verify_round()
        assert res["ok"], res
        assert not torch.equal(eng.server_state()["m"], m0)     # the state is carried from round to round
    rep = eng.run_rounds(2)
    assert rep.extra["server_opt"] == kind and torch.isfinite(eng.global_flat()).all()


@pytest.mark.parametrize("kind", OPT_KINDS)
def test_twoshot_engine_with_server_optimizer(kind):
    """world 1: the average of a round is fit(theta), which a plain FedAvg engine (sgd, lr 1) yields as its new model."""
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    xs, ys = synthetic_unsw(256, seed=21)
    kw = dict(backend="fused", device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096, bf16_shadow=True, shuffle=False,
              model_kwargs={"width": 256, "depth": 3})
    opt = _opt(kind)

    def fit_of(theta):
        e = FederatedEngine("wide_mlp", **kw)
        e.set_local_data(xs, ys)
        e.load_global(theta)
        e.run_rounds(1)
        torch.cuda.synchronize()
        return e.global_flat().clone()

    eng = FederatedEngine("wide_mlp", server_opt=opt, **kw)
    eng.set_local_data(xs, ys)
    theta0 = eng.global_flat().clone()
    ref_theta, ref = theta0.clone(), opt.init_state(eng.P, dev)
    for rnd in range(2):
        avg = fit_of(ref_theta if rnd == 0 else eng.global_flat())
        start = eng.global_flat().clone()
        rep = eng.run_rounds(1)
        torch.cuda.synchronize()
        assert rep.extra["nvls"] is False and rep.extra["server_opt"] == kind
        want = start.clone()
        reference.server_opt_step(want, avg, kind, opt.lr, ref.m, ref.v, opt.beta1, opt.beta2, opt.tau)
        got = eng.global_flat()
        torch.testing.assert_close(got, want, **_tol(kind))
        st = eng.server_state()
        torch.testing.assert_close(st["m"], ref.m, **_tol(kind))
        if ref.v is not None:
            torch.testing.assert_close(st["v"], ref.v, rtol=1e-5, atol=1e-8)
        assert torch.equal(eng.arena.tensor("shadow")[: eng.P], got.to(torch.bfloat16))
        # follow the engine's own trajectory into the next round
        ref.m.copy_(st["m"])
        if ref.v is not None:
            ref.v.copy_(st["v"])
    assert not torch.equal(eng.global_flat(), theta0)


# ---- several GPUs ---------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, out_path, case):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from colearn_federated_learning_b200.data import shard_bounds, synthetic_unsw
        from colearn_federated_learning_b200.parallel import FederatedEngine
        dev = torch.device("cuda", rank)
        if case == "star":
            x, y = synthetic_unsw(80 * world, seed=4)
            lo, hi = list(shard_bounds(80 * world, world))[rank]
            eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=3, weighted=True,
                                  server_opt=ServerOpt("adam", lr=0.02))
            eng.set_local_data(x[lo:hi], y[lo:hi])
            oks = [eng.verify_round() for _ in range(3)]
            if rank == 0:
                torch.save({"oks": oks}, out_path)
            return
        # two-shot: the average of round 1 from a plain FedAvg engine (sgd, lr 1), then the adam engine's round 1 against the
        # reference step from the same start; every rank must hold the same model and only the moments of its own chunks
        xs, ys = synthetic_unsw(256 * world, seed=21)
        lo, hi = list(shard_bounds(256 * world, world))[rank]
        kw = dict(backend="fused", device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096, bf16_shadow=True, shuffle=False,
                  model_kwargs={"width": 256, "depth": 3})
        plain = FederatedEngine("wide_mlp", **kw)
        plain.set_local_data(xs[lo:hi], ys[lo:hi])
        theta0 = plain.global_flat().clone()
        plain.run_rounds(1)
        avg = plain.global_flat().clone()
        opt = ServerOpt("adam", lr=0.02)
        eng = FederatedEngine("wide_mlp", server_opt=opt, **kw)
        eng.set_local_data(xs[lo:hi], ys[lo:hi])
        eng.run_rounds(1)
        torch.cuda.synchronize()
        want, ref = theta0.clone(), opt.init_state(eng.P, dev)
        ops.reference.server_opt_step(want, avg, "adam", opt.lr, ref.m, ref.v, opt.beta1, opt.beta2, opt.tau)
        got = eng.global_flat().clone()
        err = float((got - want).abs().max())
        owned = (torch.arange(eng.P, device=dev) // eng.chunk_elems) % world == rank
        m = eng.server_state()["m"]
        m_err = float((m[owned] - ref.m[owned]).abs().max())
        untouched = bool((m[~owned] == 0).all())
        allg = [torch.zeros_like(got) for _ in range(world)]
        dist.all_gather(allg, got)
        if rank == 0:
            torch.save({"err": err, "m_err": m_err, "untouched": untouched, "same": all(torch.equal(allg[0], a) for a in allg),
                        "shadow_ok": bool(torch.equal(eng.arena.tensor("shadow")[: eng.P], got.to(torch.bfloat16)))}, out_path)
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("case", ["star", "twoshot"])
def test_server_optimizer_multi_rank(tmp_path, case):
    world = min(torch.cuda.device_count(), 8)
    out = str(tmp_path / "out.pt")
    mp.spawn(_rank_main, args=(world, _free_port(), out, case), nprocs=world, join=True)
    res = torch.load(out, weights_only=False)
    if case == "star":
        assert all(r["ok"] for r in res["oks"]), res
    else:
        assert res["err"] < 1e-5 and res["m_err"] < 1e-5 and res["untouched"] and res["same"] and res["shadow_ok"], res
