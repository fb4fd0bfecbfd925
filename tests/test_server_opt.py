"""Server optimizers (FedAvgM / FedAdagrad / FedAdam / FedYogi) without a GPU: the PyTorch definition against a float64
transcription of the update table, the kernel sources of comm.cu / elementwise.cu on the SIMT CPU build (star round,
two-shot, overlapped two-shot, fedavg_apply), the engine's CPU backend, the Coordinator's local mode and the CLI.

Tolerances: the kernels form the average with fp32 sums in their own order (per-rank fmaf chains, renormalisation by a
product) and use fmaf inside the step, so each element differs from the PyTorch reference by a few fp32 ulps of the
average (~1e-7 relative).  Through m / (sqrt(v) + tau) that becomes a relative error of the same order in the step, and
over 2-3 rounds of values O(1) an absolute 1e-5 / relative 1e-5 bound holds with a wide margin; plain momentum is one
fmaf away from the reference and holds to 1e-6."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.server_opt import KINDS, ServerOpt, default_server_lr
from colearn_federated_learning_b200.ops import reference

OPT_KINDS = ["avgm", "adagrad", "adam", "yogi"]
HYPER = dict(beta1=0.9, beta2=0.99, tau=1e-3)


def _tol(kind):
    return dict(rtol=1e-6, atol=1e-6) if kind == "avgm" else dict(rtol=1e-5, atol=1e-5)


@pytest.fixture(scope="module")
def simt():
    import importlib.util
    import shutil

    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _np_step(theta, avg, kind, lr, m, v, beta1=0.9, beta2=0.99, tau=1e-3):
    """float64 transcription of the table in fl/server_opt.py."""
    d = avg - theta
    if kind == "sgd":
        return theta + lr * d, m, v
    if kind == "avgm":
        m = beta1 * m + d
        return theta + lr * m, m, v
    m = beta1 * m + (1 - beta1) * d
    if kind == "adagrad":
        v = v + d * d
    elif kind == "adam":
        v = beta2 * v + (1 - beta2) * d * d
    else:
        v = v - (1 - beta2) * d * d * np.sign(v - d * d)
    return theta + lr * m / (np.sqrt(v) + tau), m, v


def _state(kind, n, lr=None):
    opt = ServerOpt(kind, lr=lr, **HYPER)
    return opt, opt.init_state(n)


# ---- the PyTorch definition ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", list(KINDS))
def test_reference_matches_float64_transcription(kind):
    g = torch.Generator().manual_seed(KINDS[kind])
    n, K = 257, 3
    opt, st = _state(kind, n, lr=0.05 if kind in ("adagrad", "adam", "yogi") else 0.7)
    theta = torch.randn(n, generator=g)
    t64 = theta.double().numpy()
    m64 = np.zeros(n)
    v64 = np.full(n, opt.tau ** 2)
    for _ in range(5):
        models = torch.randn(K, n, generator=g) + theta
        w = torch.tensor([0.5, 0.3, 0.2])
        before = theta.clone()
        reference.server_opt_apply(theta, models, w, kind, opt.lr, st.m, st.v, opt.beta1, opt.beta2, opt.tau)
        avg64 = (w.double().view(-1, 1) * models.double()).sum(0).numpy()
        t64, m64, v64 = _np_step(t64, avg64, kind, opt.lr, m64, v64, opt.beta1, opt.beta2, opt.tau)
        if kind == "sgd":
            want = reference.fedavg_apply(before.clone(), models, w, opt.lr)
            assert torch.equal(theta, want)                                   # bit for bit today's update
        np.testing.assert_allclose(theta.numpy(), t64, rtol=1e-5, atol=1e-5)
        if kind != "sgd":
            np.testing.assert_allclose(st.m.numpy(), m64, rtol=1e-5, atol=1e-6)
        if opt.has_v:
            np.testing.assert_allclose(st.v.numpy(), v64, rtol=1e-5, atol=1e-7)


def test_server_opt_settings_are_validated():
    assert ServerOpt("adam").lr == 0.01 and ServerOpt("avgm").lr == 1.0 and ServerOpt("sgd").lr == 1.0
    st = ServerOpt("adam", tau=0.01).init_state(5)
    assert torch.equal(st.m, torch.zeros(5)) and torch.allclose(st.v, torch.full((5,), 1e-4))
    assert ServerOpt("avgm").init_state(3).v is None and ServerOpt("sgd").init_state(3).m is None
    for bad in (dict(kind="lamb"), dict(kind="adam", beta1=1.0), dict(kind="adam", beta2=-0.1), dict(kind="yogi", tau=0.0),
                dict(kind="adagrad", tau=-1e-3), dict(kind="avgm", beta1=1.5)):
        with pytest.raises(ValueError):
            ServerOpt(**bad)
    theta, models, w = torch.zeros(4), torch.ones(2, 4), torch.tensor([0.5, 0.5])
    with pytest.raises(ValueError, match="carries its own lr"):
        ops.fedavg_apply(theta, models, w, 0.5, opt=ServerOpt("adam").init_state(4))


# ---- comm.cu / elementwise.cu on the SIMT CPU build -------------------------------------------------------------------------
@pytest.mark.parametrize("kind", OPT_KINDS)
def test_star_round_with_server_optimizer_on_cpu(simt, kind):
    torch.manual_seed(10 + KINDS[kind])
    W, P = 4, 1003                                            # P not a multiple of 4: float4 body + scalar tail
    opt, st = _state(kind, P, lr=0.1 if opt_is_adaptive(kind) else 0.8)
    ref_opt, ref = _state(kind, P, lr=opt.lr)
    theta = torch.randn(P)
    ref_theta = theta.clone()
    inboxes, bflags = torch.zeros(W, P), torch.zeros(W, dtype=torch.int32)
    arrive = torch.full((W,), 5, dtype=torch.int32)
    # round 1: everybody; round 2: ranks 0 and 2 selected; round 3: deadline, rank 3 never arrives (weight renormalised)
    rounds = [(0b1111, [0.4, 0.3, 0.2, 0.1], 0.0, arrive), (0b0101, [0.5, 0.0, 0.5, 0.0], 0.0, arrive),
              (0b1111, [0.4, 0.3, 0.2, 0.1], 20.0, torch.tensor([5, 5, 5, 4], dtype=torch.int32))]
    for i, (mask, weights, timeout, flags) in enumerate(rounds):
        models = [theta + 0.5 * torch.randn(P) for _ in range(W)]
        slots = torch.stack([w * m for w, m in zip(weights, models)])
        got = simt.star_round(theta, slots, flags, 5, inboxes, bflags, 6 + i, mask, opt.lr, True, True, 3, timeout, weights,
                              opt.code, opt.hyper, st.m, st.v)
        arrived = 0b0111 if timeout > 0 else mask
        assert got == arrived
        ws = [w if (arrived >> k) & 1 else 0.0 for k, w in enumerate(weights)]
        avg = sum(w * m for w, m in zip(ws, models)) / sum(ws)
        reference.server_opt_step(ref_theta, avg, kind, opt.lr, ref.m, ref.v, **HYPER)
        torch.testing.assert_close(theta, ref_theta, **_tol(kind))
        torch.testing.assert_close(st.m, ref.m, **_tol(kind))
        if st.v is not None:
            torch.testing.assert_close(st.v, ref.v, rtol=1e-5, atol=1e-7)
        for k in range(W):                                      # the broadcast carries the post-step model
            if (mask >> k) & 1:
                assert torch.equal(inboxes[k], theta)
    # nobody arrives in time: theta and both moments stay bit for bit
    keep = (theta.clone(), st.m.clone(), st.v.clone() if st.v is not None else None)
    got = simt.star_round(theta, slots, torch.zeros(W, dtype=torch.int32), 5, inboxes, bflags, 9, 0b1111, opt.lr, True, False, 2, 5.0,
                          [0.4, 0.3, 0.2, 0.1], opt.code, opt.hyper, st.m, st.v)
    assert got == 0 and torch.equal(theta, keep[0]) and torch.equal(st.m, keep[1])
    assert keep[2] is None or torch.equal(st.v, keep[2])


def opt_is_adaptive(kind):
    return kind in ("adagrad", "adam", "yogi")


def _twoshot_rounds(simt, kind, rounds, produced=False):
    torch.manual_seed(20 + KINDS[kind] + (100 if produced else 0))
    W, n, chunk = 3, 4 * 350, 64                              # 22 chunks (the last one short), owner of chunk c = c % W
    n_chunks = (n + chunk - 1) // chunk
    opt, _ = _state(kind, n, lr=0.1 if opt_is_adaptive(kind) else 0.8)
    states = [opt.init_state(n) for _ in range(W)]            # every rank's moment buffer (it touches the chunks it owns)
    _, ref = _state(kind, n, lr=opt.lr)
    weights = torch.tensor([0.2, 0.3, 0.5])
    theta = torch.randn(n)
    ref_theta = theta.clone()
    shadows = torch.zeros(W, n, dtype=torch.bfloat16)
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    works = torch.zeros(W, n)
    for i in range(rounds):
        epoch = 3 + i
        trained = theta + 0.5 * torch.randn(W, n)
        works.copy_(trained)                                    # the ranks trained in place on their arenas
        prevs = [theta.clone() for _ in range(W)]               # ... after keeping the round's starting model
        arrive = torch.full((W,), epoch, dtype=torch.int32)
        table = torch.full((W, W, n_chunks), epoch, dtype=torch.int32) if produced else None
        for r in range(W):
            simt.twoshot_fedavg(r, works, shadows, flags, arrive, weights, prevs[r], epoch, 0b111, opt.lr, chunk, 2, table,
                                5.0 if produced else 0.0, opt.code, opt.hyper, states[r].m, states[r].v)
        avg = (weights.view(-1, 1) * trained).sum(0)
        reference.server_opt_step(ref_theta, avg, kind, opt.lr, ref.m, ref.v, **HYPER)
        for k in range(W):
            torch.testing.assert_close(works[k], ref_theta, **_tol(kind))
            assert torch.equal(shadows[k], works[k].to(torch.bfloat16))
            assert torch.equal(works[k], works[0])
        assert int(flags.min()) == epoch
        theta = works[0].clone()
        # the moments, gathered by chunk owner, are the reference state; every other chunk of a rank's buffer is untouched
        owner = torch.arange(n) // chunk % W
        for name, init in (("m", 0.0), ("v", opt.tau ** 2)):
            bufs = [getattr(s, name) for s in states]
            if bufs[0] is None:
                continue
            gathered = torch.stack(bufs).gather(0, owner.view(1, -1)).view(-1)
            torch.testing.assert_close(gathered, getattr(ref, name), **(_tol(kind) if name == "m" else dict(rtol=1e-5, atol=1e-7)))
            for r in range(W):
                assert bool((bufs[r][owner != r] == init).all())


@pytest.mark.parametrize("kind", OPT_KINDS)
def test_twoshot_with_server_optimizer_on_cpu(simt, kind):
    _twoshot_rounds(simt, kind, rounds=2)


def test_overlapped_twoshot_with_adam_on_cpu(simt):
    """The overlapped form (fused wgrad -> reduce) shares twoshot_chunk: here every producer's chunks are already reported."""
    _twoshot_rounds(simt, "adam", rounds=2, produced=True)


@pytest.mark.parametrize("kind", ["sgd"] + OPT_KINDS)
def test_fedavg_apply_with_server_optimizer_on_cpu(simt, kind):
    torch.manual_seed(30 + KINDS[kind])
    n, K = 1001, 3                                            # n % 4 != 0: scalar tail
    opt, st = _state(kind, n, lr=0.1 if opt_is_adaptive(kind) else 0.8)
    _, ref = _state(kind, n, lr=opt.lr)
    theta = torch.randn(n)
    ref_theta = theta.clone()
    w = torch.tensor([0.2, 0.3, 0.5])
    for _ in range(3):
        models = theta + 0.5 * torch.randn(K, n)
        simt.fedavg_apply(theta, models, w, opt.lr, opt.code, opt.hyper, st.m, st.v)
        reference.server_opt_apply(ref_theta, models, w, kind, opt.lr, ref.m, ref.v, **HYPER)
        torch.testing.assert_close(theta, ref_theta, **_tol(kind))
        if st.m is not None:
            torch.testing.assert_close(st.m, ref.m, **_tol(kind))
    # ops.fedavg_apply on CPU tensors: the reference itself
    th, st2 = ref_theta.clone(), opt.init_state(n)
    ops.fedavg_apply(th, models, w, opt=st2)
    want, st3 = ref_theta.clone(), opt.init_state(n)
    reference.server_opt_apply(want, models, w, kind, opt.lr, st3.m, st3.v, **HYPER)
    assert torch.equal(th, want)


# ---- FederatedEngine, CPU backend -------------------------------------------------------------------------------------------
def _host_adam_rounds(theta0, shards, weights, eng, rounds, opt):
    from colearn_federated_learning_b200.fl.trainer import local_fit
    theta, st = theta0.clone(), opt.init_state(theta0.numel())
    for r in range(rounds):
        avg = torch.zeros_like(theta)
        for (x, y), w in zip(shards, weights):
            local = theta.clone()
            local_fit(local, eng.model, x, y, eng.cfg, r)
            avg += w * local
        reference.server_opt_step(theta, avg, opt.kind, opt.lr, st.m, st.v, opt.beta1, opt.beta2, opt.tau)
    return theta, st


def test_engine_cpu_single_process_adam_matches_host_loop():
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    opt = ServerOpt("adam", lr=0.02)
    eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), batch_size=4, lr=0.05, seed=3, server_opt=opt)
    x, y = synthetic_unsw(96, seed=0)
    eng.set_local_data(x, y)
    theta0 = eng.global_flat().clone()
    rep = eng.run_rounds(3)
    assert rep.extra["server_opt"] == "adam"
    want, st = _host_adam_rounds(theta0, [(x, y)], [1.0], eng, 3, opt)
    torch.testing.assert_close(eng.global_flat(), want, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(eng.server_state()["m"], st.m, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(eng.server_state()["v"], st.v, rtol=1e-5, atol=1e-9)
    # nobody selected: theta and the moments stay
    keep = (eng.global_flat().clone(), eng.server_state()["m"].clone(), eng.server_state()["v"].clone())
    eng.run_rounds(1, masks=0)
    assert torch.equal(eng.global_flat(), keep[0]) and torch.equal(eng.server_state()["m"], keep[1])
    assert torch.equal(eng.server_state()["v"], keep[2])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, out):
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), batch_size=2, lr=0.05, seed=5, weighted=True,
                              server_opt=ServerOpt("adam", lr=0.02))
        x, y = synthetic_unsw(90, seed=1)
        lo, hi = [(0, 60), (60, 90)][rank]
        eng.set_local_data(x[lo:hi], y[lo:hi])
        theta0 = eng.global_flat().clone()
        eng.run_rounds(2)
        if rank == 0:
            torch.save({"theta0": theta0, "theta": eng.global_flat().clone(), "m": eng.server_state()["m"].clone()}, out)
        else:
            assert eng.server_state()["m"] is None          # star / CPU: the state lives on the coordinator only
    finally:
        dist.destroy_process_group()


def test_engine_cpu_two_process_gloo_adam_matches_host_loop(tmp_path):
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    out = str(tmp_path / "res.pt")
    mp.spawn(_gloo_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    res = torch.load(out, weights_only=False)
    x, y = synthetic_unsw(90, seed=1)
    eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), batch_size=2, lr=0.05, seed=5)
    want, st = _host_adam_rounds(res["theta0"], [(x[:60], y[:60]), (x[60:], y[60:])], [2 / 3, 1 / 3], eng, 2, ServerOpt("adam", lr=0.02))
    torch.testing.assert_close(res["theta"], want, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(res["m"], st.m, rtol=1e-4, atol=1e-6)


def test_engine_rejects_bad_combinations():
    from colearn_federated_learning_b200.parallel import FederatedEngine
    with pytest.raises(ValueError, match="chunk ownership moves"):
        FederatedEngine("wide_mlp", backend="cpu", device=torch.device("cpu"), algo="twoshot", round_deadline_ms=50.0,
                        model_kwargs={"width": 64, "depth": 1}, server_opt=ServerOpt("adam"))
    with pytest.raises(ValueError, match="carries its own lr"):
        FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), server_lr=0.5, server_opt=ServerOpt("avgm"))
    # sgd stays allowed with a deadline; server_lr alone is plain FedAvg as before
    eng = FederatedEngine("wide_mlp", backend="cpu", device=torch.device("cpu"), algo="twoshot", round_deadline_ms=50.0,
                          model_kwargs={"width": 64, "depth": 1}, server_opt=ServerOpt("sgd", lr=0.5))
    assert eng.server_lr == 0.5 and eng.opt_state is None
    assert FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), server_lr=0.3).server_opt.kind == "sgd"


# ---- CLI and the classic Coordinator ---------------------------------------------------------------------------------------
def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_cli_server_opt_flags_and_defaults():
    a = _cli()
    assert a.server_opt == "sgd" and a.server_lr == 1.0
    assert _cli("--server-opt", "avgm").server_lr == 1.0
    for kind in ("adagrad", "adam", "yogi"):
        assert _cli("--server-opt", kind).server_lr == default_server_lr(kind) == 0.01
    a = _cli("--server-opt", "yogi", "--server-lr", "0.05", "--server-beta1", "0.5", "--server-beta2", "0.9", "--server-tau", "0.01")
    opt = a.server_optimizer()
    assert (opt.kind, opt.lr, opt.beta1, opt.beta2, opt.tau) == ("yogi", 0.05, 0.5, 0.9, 0.01)
    for bad in (["--server-beta1", "1.0"], ["--server-beta2", "-0.5"], ["--server-tau", "0"], ["--server-opt", "lamb"]):
        with pytest.raises(SystemExit):
            _cli("--server-opt", "adam", *bad)


def test_local_mode_coordinator_two_rounds_with_adam(tmp_path):
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator, train_virtual_workers
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.data import BaseDataset, federate, synthetic_unsw
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    cpu = torch.device("cpu")
    args = _cli("--server-opt", "adam", "--synthetic", "60", "--lr", "0.05")
    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, False, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "test.pth"), device=cpu)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    torch.manual_seed(0)
    init = FFNN()
    save_model(init, c.path)
    ips = ["10.0.0.1", "10.0.0.2"]
    for ip in ips:
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert c.windower.last_result is not None and c.windower.last_result["rounds"] == 2
    x, y = synthetic_unsw(60, seed=args.seed)
    fed = federate(BaseDataset(x, y), ips, cpu)
    theta = flatten_params(init).clone()
    st = ServerOpt("adam", lr=0.01).init_state(theta.numel())
    for r in range(2):
        flats, _, counts = train_virtual_workers(theta, FFNN(), fed, c._fit_config("local"), r)
        reference.server_opt_apply(theta, flats, torch.full((len(ips),), 1.0 / len(ips)), "adam", 0.01, st.m, st.v, **HYPER)
    m = FFNN()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    torch.testing.assert_close(flatten_params(m), theta, rtol=1e-5, atol=1e-6)
    # the state stays with the Coordinator (carried into the next window)
    assert c._server_opt_state is not None and torch.allclose(c._server_opt_state.m, st.m, rtol=1e-4, atol=1e-7)
