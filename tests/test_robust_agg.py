"""Byzantine-robust aggregation (coordinate-wise median / trimmed mean) without a GPU: the PyTorch definition against a
float64 transcription, and the kernel sources of comm.cu / elementwise.cu on the SIMT CPU build (star round, two-shot with
and without a deadline, overlapped two-shot, fedavg_apply on both of its paths) bit for bit against the definition.

Bit-exact comparisons hold because the definition fixes every rounding: ranks are integer counts, the kept values are summed
in slot order starting from +0 and divided once (IEEE), and the server step with lr = 1 is fmaf(1, a - t, t) = (a - t) + t
on both sides.  Only the FedAdam composition compares with a tolerance (the kernels' fmaf chains in the optimizer step,
see tests/test_server_opt.py).  "Bit for bit" is for every value but NaN: IEEE does not fix the sign or payload of a NaN
that arithmetic produces (x86 passes one operand's payload through, the GPU writes its canonical NaN), so a NaN must meet a
NaN and every other value must carry the same 32 bits."""
import math
import os

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.aggregate import KINDS, Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.ops import reference

ROBUST = [Aggregator("median"), Aggregator("trimmed_mean", 0.2), Aggregator("trimmed_mean", 0.0), Aggregator("trimmed_mean", 0.49)]


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


def same_bits(a, b):
    """a and b hold the same float32 (bfloat16) bit patterns, any NaN matching any NaN"""
    nan, bits = a.isnan(), torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(bits), b[~nan].view(bits)))


def models_with_outliers(K, P, seed):
    """Client models around a common point, with planted trouble: huge outliers, NaN, +-Inf, +-0 and exact ties."""
    g = torch.Generator().manual_seed(seed)
    m = torch.randn(K, P, generator=g)
    r = torch.rand(K, P, generator=g)
    m[r < 0.04] = 1e6
    m[(r >= 0.04) & (r < 0.06)] = float("nan")
    m[(r >= 0.06) & (r < 0.08)] = float("inf")
    m[(r >= 0.08) & (r < 0.10)] = -float("inf")
    m[(r >= 0.10) & (r < 0.13)] = 0.0
    m[(r >= 0.13) & (r < 0.16)] = -0.0
    tie = (r >= 0.16) & (r < 0.22)
    m[tie] = 0.5
    if K > 1:
        m[1, : P // 8] = -float("nan")               # a negative NaN
    return m


def _np_aggregate(models, kind, beta, rows=None):
    """float64 transcription: sort the values of each column by the IEEE total order (stable, so ties keep slot order),
    drop b at each end, average the rest."""
    v = models.numpy() if rows is None else models.numpy()[rows]
    n = v.shape[0]
    bits = v.astype(np.float32).view(np.int32)
    key = bits ^ ((bits >> 31) & 0x7FFFFFFF)
    half = (n - 1) // 2
    b = half if kind == "median" else min(int(math.floor(np.float32(beta) * np.float32(n))), half)
    order = np.argsort(key, axis=0, kind="stable")
    kept = np.take_along_axis(v.astype(np.float64), order, axis=0)[b: n - b]
    with np.errstate(invalid="ignore"):
        return kept.sum(0) / (n - 2 * b)


# ---- the PyTorch definition ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", range(1, 18))
def test_reference_matches_float64_transcription(n):
    models = models_with_outliers(n, 513, seed=n)
    for agg in ROBUST + [Aggregator("trimmed_mean", 0.25), Aggregator("trimmed_mean", 1.0 / 3.0)]:
        got = reference.robust_aggregate(models, None, agg.kind, agg.trim)
        want = _np_aggregate(models, agg.kind, agg.trim)
        np.testing.assert_allclose(got.numpy(), want, rtol=1e-6, atol=1e-5, equal_nan=True)
        assert not (got.isinf() & (got > 0) & torch.from_numpy(want < 0)).any()
    # a subset mask is the same as the selected rows
    if n >= 3:
        mask = 0b101 | (1 << (n - 1))
        rows = [k for k in range(n) if (mask >> k) & 1]
        np.testing.assert_allclose(reference.robust_aggregate(models, mask, "median").numpy(), _np_aggregate(models, "median", 0, rows),
                                   rtol=1e-6, atol=1e-5, equal_nan=True)


def test_median_and_trim_semantics():
    col = torch.tensor([[3.0], [1.0], [2.0], [100.0]])
    assert reference.robust_aggregate(col, None, "median").item() == 2.5                     # even n: mean of the middle two
    assert reference.robust_aggregate(col[:3], None, "median").item() == 2.0                 # odd n: the middle value
    assert reference.robust_aggregate(col, None, "trimmed_mean", 0.25).item() == 2.5         # b = 1
    assert reference.robust_aggregate(col, None, "trimmed_mean", 0.24).item() == 26.5        # b = 0: the plain mean
    # a minority of NaN / Inf senders is trimmed like any outlier
    bad = torch.tensor([[1.0], [float("nan")], [2.0], [-float("inf")], [3.0]])
    assert reference.robust_aggregate(bad, None, "median").item() == 2.0
    assert reference.robust_aggregate(bad, None, "trimmed_mean", 0.2).item() == 2.0
    # trim count: beta * n in float32, capped at floor((n - 1) / 2)
    assert reference.agg_trim_count("trimmed_mean", 0.1, 10) == 1 and reference.agg_trim_count("trimmed_mean", 0.49, 4) == 1
    assert reference.agg_trim_count("trimmed_mean", 0.3, 10) == int(np.floor(np.float32(0.3) * np.float32(10)))
    assert reference.agg_trim_count("median", 0.0, 1) == 0 and reference.agg_trim_count("median", 0.0, 8) == 3


def test_aggregator_settings_are_validated():
    assert Aggregator().kind == "mean" and not Aggregator().robust
    assert Aggregator("median").code == KINDS["median"] == 1 and Aggregator("trimmed_mean").code == 2
    assert Aggregator("median", 0.3).trim == 0.0 and Aggregator("trimmed_mean", 0.3).trim == 0.3
    for bad in (dict(kind="krum"), dict(kind="trimmed_mean", trim_fraction=0.5), dict(kind="trimmed_mean", trim_fraction=-0.1),
                dict(kind="median", trim_fraction=float("nan"))):
        with pytest.raises(ValueError):
            Aggregator(**bad)


def test_ops_fedavg_apply_on_cpu_is_the_reference():
    models = models_with_outliers(5, 300, seed=3)
    theta = torch.randn(300)
    w = torch.full((5,), 0.2)
    for agg in ROBUST:
        got = ops.fedavg_apply(theta.clone(), models, w, 0.5, aggregator=agg)
        avg = reference.robust_aggregate(models, None, agg.kind, agg.trim)
        assert same_bits(got, theta.clone().add_(0.5 * (avg - theta)))
    # mean (or no aggregator) is today's weighted FedAvg
    assert torch.equal(ops.fedavg_apply(theta.clone(), models.nan_to_num(), w, aggregator=Aggregator()),
                       reference.fedavg_apply(theta.clone(), models.nan_to_num(), w))


# ---- elementwise.cu on the SIMT CPU build ------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 3, 16, 33, 100])
def test_fedavg_apply_robust_on_cpu_bit_exact(simt, K):
    """register path (K <= 32: KMAX 4 / 16 / 32 here) and the general path (K > 32); n = 1001 is not a multiple of 4"""
    n = 1001 if K < 100 else 203
    models = models_with_outliers(K, n, seed=40 + K)
    w = torch.full((K,), 1.0 / K)
    for agg in ROBUST:
        theta = torch.randn(n, generator=torch.Generator().manual_seed(K))
        want = reference.fedavg_apply(theta.clone(), models, w, 1.0, aggregator=agg)
        simt.fedavg_apply(theta, models, w, 1.0, 0, [], None, None, agg.code, agg.trim)
        assert same_bits(theta, want), agg


def test_fedavg_apply_robust_with_adam_on_cpu(simt):
    n, K = 1001, 7
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(n), opt.init_state(n)
    theta = torch.randn(n)
    ref_theta = theta.clone()
    agg = Aggregator("trimmed_mean", 0.2)
    for i in range(3):
        models = theta + 0.5 * torch.randn(K, n)
        models[i] = 1e5                                       # one poisoned client per round
        simt.fedavg_apply(theta, models, torch.full((K,), 1.0 / K), opt.lr, opt.code, opt.hyper, st.m, st.v, agg.code, agg.trim)
        reference.server_opt_apply(ref_theta, models, None, "adam", opt.lr, ref.m, ref.v, *opt.hyper, aggregator=agg)
        torch.testing.assert_close(theta, ref_theta, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.m, ref.m, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.v, ref.v, rtol=1e-5, atol=1e-7)
    assert float(theta.abs().max()) < 10.0                    # the poisoned client did not move the model


# ---- comm.cu on the SIMT CPU build -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("agg", ROBUST[:2], ids=lambda a: a.kind)
def test_star_round_robust_on_cpu_bit_exact(simt, agg):
    W, P = 6, 1003                                            # float4 body + scalar tail
    theta = torch.randn(P)
    inboxes, bflags = torch.zeros(W, P), torch.zeros(W, dtype=torch.int32)
    full = torch.full((W,), 5, dtype=torch.int32)
    late = full.clone()
    late[4] = 4
    weights = [1.0 / W] * W                                   # (not used by a robust kind)
    # all six; a subset of four; a deadline at which worker 4 is late
    for i, (mask, timeout, flags, arrived) in enumerate([(0b111111, 0.0, full, 0b111111), (0b101101, 0.0, full, 0b101101),
                                                         (0b111111, 20.0, late, 0b101111)]):
        slots = models_with_outliers(W, P, seed=60 + i)       # raw models: the producers push theta_k unscaled
        want = theta.clone()
        reference.fedavg_apply(want, slots[[k for k in range(W) if (arrived >> k) & 1]], None, 1.0, aggregator=agg)
        got = simt.star_round(theta, slots, flags, 5, inboxes, bflags, 6 + i, mask, 1.0, True, True, 3, timeout, weights,
                              0, [], None, None, agg.code, agg.trim)
        assert got == arrived
        assert same_bits(theta, want)
        for k in range(W):
            if (mask >> k) & 1:
                assert same_bits(inboxes[k], theta)
    # nobody arrives in time: theta stays bit for bit
    theta = torch.randn(P)
    keep = theta.clone()
    got = simt.star_round(theta, slots, torch.zeros(W, dtype=torch.int32), 5, inboxes, bflags, 9, 0b111111, 1.0, True, False, 2, 5.0,
                          weights, 0, [], None, None, agg.code, agg.trim)
    assert got == 0 and same_bits(theta, keep)


def _twoshot_round(simt, W, agg, produced=False, seed=0):
    n, chunk = 4 * 300, 64
    n_chunks = (n + chunk - 1) // chunk
    trained = models_with_outliers(W, n, seed=seed)
    works = trained.clone()
    shadows = torch.zeros(W, n, dtype=torch.bfloat16)
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    mask = (1 << W) - 1 if produced else ((1 << W) - 1) & ~0b10          # rank 1 not selected (it still owns chunks)
    epoch = 3
    arrive = torch.full((W,), epoch, dtype=torch.int32)
    table = torch.full((W, W, n_chunks), epoch, dtype=torch.int32) if produced else None
    weights = torch.full((W,), 1.0 / W)
    for r in range(W):
        simt.twoshot_fedavg(r, works, shadows, flags, arrive, weights, None, epoch, mask, 1.0, chunk, 2, table,
                            5.0 if produced else 0.0, 0, [], None, None, agg.code, agg.trim)
    want = reference.robust_aggregate(trained, mask, agg.kind, agg.trim)
    for k in range(W):
        assert same_bits(works[k], want), k
        assert same_bits(shadows[k], works[k].to(torch.bfloat16))
    assert int(flags.min()) == epoch


@pytest.mark.parametrize("W", range(3, 9))
def test_twoshot_robust_on_cpu_bit_exact(simt, W):
    _twoshot_round(simt, W, ROBUST[W % 2], seed=70 + W)


def test_overlapped_twoshot_robust_on_cpu_bit_exact(simt):
    _twoshot_round(simt, 5, Aggregator("median"), produced=True, seed=80)


@pytest.mark.parametrize("W", [3, 5, 8])
def test_twoshot_robust_with_deadline_on_cpu_bit_exact(simt, W):
    """rank W-1 misses the deadline: ownership is dealt among the others, the aggregate is over the arrived ranks only"""
    agg = Aggregator("median") if W != 5 else Aggregator("trimmed_mean", 0.25)
    n, chunk = 4 * 256, 128
    n_chunks = n // chunk
    trained = models_with_outliers(W, n, seed=90 + W)
    works = trained.clone()
    globals_ = torch.zeros(W, n)
    flags = torch.zeros(W, n_chunks, dtype=torch.int32)
    decisions = torch.zeros(W, 16, dtype=torch.int32)
    weights = torch.zeros(16)
    weights[:W] = 1.0 / W
    epoch = 5
    arrive = [torch.zeros(W, dtype=torch.int32) for _ in range(W)]
    for a in arrive:
        a[: W - 1] = epoch
    full = (1 << W) - 1
    for r in range(W - 1):                                    # the coordinator (which decides) first
        simt.twoshot_fedavg_deadline(r, works, globals_, flags, arrive[r], weights, epoch, full, chunk, 2, 2.0, decisions,
                                     agg.code, agg.trim)
    arrived = full & ~(1 << (W - 1))
    assert decisions[0, 2 * (epoch % 8) + 1].item() == arrived
    want = reference.robust_aggregate(trained, arrived, agg.kind, agg.trim)
    for k in range(W):
        assert same_bits(globals_[k], want), k
    for k in range(W - 1):
        assert same_bits(works[k], want), k


# ---- FederatedEngine, CPU backend over gloo ---------------------------------------------------------------------------------
def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _shards():
    from colearn_federated_learning_b200.data import synthetic_unsw
    x, y = synthetic_unsw(90, seed=1)
    shards = [(x[0:30], y[0:30]), (x[30:60], y[30:60]), (x[60:90] * 1e3, 1.0 - y[60:90])]   # rank 2 trains on poisoned data
    return shards


def _gloo_worker(rank, world, port, out, kind):
    import torch.distributed as dist

    from colearn_federated_learning_b200.parallel import FederatedEngine
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), batch_size=2, lr=0.05, seed=5,
                              aggregator=Aggregator(kind, 0.34))
        x, y = _shards()[rank]
        eng.set_local_data(x, y)
        theta0 = eng.global_flat().clone()
        reps = [eng.run_rounds(1), eng.run_rounds(1, masks=0b011)]
        if rank == 0:
            torch.save({"theta0": theta0, "theta": eng.global_flat().clone(), "agg": reps[0].extra["aggregator"]}, out)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["median", "trimmed_mean"])
def test_engine_cpu_three_process_gloo_robust_matches_reference(tmp_path, kind):
    import torch.multiprocessing as mp

    from colearn_federated_learning_b200.fl.trainer import local_fit
    from colearn_federated_learning_b200.parallel import FederatedEngine
    out = str(tmp_path / "res.pt")
    mp.spawn(_gloo_worker, args=(3, _free_port(), out, kind), nprocs=3, join=True)
    res = torch.load(out, weights_only=False)
    assert res["agg"] == kind
    eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), batch_size=2, lr=0.05, seed=5)
    theta = res["theta0"].clone()
    for r, mask in enumerate([0b111, 0b011]):
        locals_ = []
        for x, y in _shards():
            local = theta.clone()
            local_fit(local, eng.model, x, y, eng.cfg, r)
            locals_.append(local)
        avg = reference.robust_aggregate(torch.stack(locals_), mask, kind, 0.34)
        theta.add_(1.0 * (avg - theta))
    assert torch.equal(res["theta"], theta)


def test_engine_refuses_robust_aggregator_with_many_clients_per_rank():
    from colearn_federated_learning_b200.parallel import FederatedEngine
    with pytest.raises(ValueError, match="clients_per_rank=1"):
        FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), clients_per_rank=4, aggregator=Aggregator("median"))
    eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), clients_per_rank=4)
    assert eng.aggregator.kind == "mean"


def test_engine_cpu_single_process_robust_with_nobody_selected_keeps_theta():
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    eng = FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), batch_size=4, lr=0.05, seed=3,
                          aggregator=Aggregator("median"))
    x, y = synthetic_unsw(64, seed=0)
    eng.set_local_data(x, y)
    theta0 = eng.global_flat().clone()
    assert eng.run_rounds(1).extra["aggregator"] == "median"
    moved = eng.global_flat().clone()
    assert not torch.equal(moved, theta0)
    eng.run_rounds(1, masks=0)
    assert torch.equal(eng.global_flat(), moved)


# ---- CLI and the classic Coordinator ---------------------------------------------------------------------------------------
def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_cli_aggregator_flags():
    a = _cli()
    assert a.aggregator == "mean" and a.trim_fraction == 0.1 and not a.client_aggregator().robust
    agg = _cli("--aggregator", "trimmed_mean", "--trim-fraction", "0.25").client_aggregator()
    assert (agg.kind, agg.trim) == ("trimmed_mean", 0.25)
    assert _cli("--aggregator", "median").client_aggregator().code == 1
    assert _cli("--weighted").weighted                                         # the weighted mean stays allowed
    for bad in (["--aggregator", "median", "--weighted"], ["--aggregator", "trimmed_mean", "--weighted"],
                ["--aggregator", "trimmed_mean", "--trim-fraction", "0.5"], ["--trim-fraction", "-0.1"], ["--aggregator", "krum"]):
        with pytest.raises(SystemExit):
            _cli(*bad)


def test_local_mode_coordinator_two_rounds_with_median(tmp_path):
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator, train_virtual_workers
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.data import BaseDataset, federate, synthetic_unsw
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    cpu = torch.device("cpu")
    args = _cli("--aggregator", "median", "--synthetic", "90", "--lr", "0.05")
    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, False, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "test.pth"), device=cpu)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    torch.manual_seed(0)
    init = FFNN()
    save_model(init, c.path)
    ips = ["10.0.0.1", "10.0.0.2", "10.0.0.3"]
    for ip in ips:
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert c.windower.last_result is not None and c.windower.last_result["rounds"] == 2
    x, y = synthetic_unsw(90, seed=args.seed)
    fed = federate(BaseDataset(x, y), ips, cpu)
    theta = flatten_params(init).clone()
    for r in range(2):
        flats, _, counts = train_virtual_workers(theta, FFNN(), fed, c._fit_config("local"), r)
        reference.fedavg_apply(theta, flats, None, 1.0, aggregator=Aggregator("median"))
    m = FFNN()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    assert torch.equal(flatten_params(m), theta)
