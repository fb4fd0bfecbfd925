"""Secure aggregation kernels on the H100: secagg_mask_kernel bit for bit against the reference at P = 1 M + 37 with S = 2 /
17 / 100 streams, fedavg_secagg_kernel bit for bit against the reference at K up to 100 with 0 / 1 / 10 dropped devices (plain
and FedAdam) and identical between two runs, the FFNN shape with thousands of streams (the split path), and one remote round
with CUDA workers and a CUDA coordinator over localhost."""
import socket

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.ops import reference

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    return [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n)]


def _same(a, b):
    return torch.equal(a.cpu().contiguous().view(torch.int32), b.cpu().contiguous().view(torch.int32))


@pytest.mark.parametrize("S", [2, 17, 100])
def test_mask_bit_exact(S):
    P = (1 << 20) + 37
    g = torch.Generator().manual_seed(S)
    theta = torch.randn(P, generator=g)
    model = theta + 0.3 * torch.randn(P, generator=g)
    model[5], model[6], model[7], model[8] = float("nan"), float("inf"), float("-inf"), theta[8] + 0.25
    keys, signs = _keys(S, S), [1 if i % 2 else -1 for i in range(S)]
    y, clipped, nonfinite = ops.secagg_mask(model.to(DEV), theta.to(DEV), keys, signs, 0.25, 22)
    want, wc, wn = reference.secagg_mask(model, theta, keys, signs, 0.25, 22)
    assert y.is_cuda and y.dtype == torch.uint32 and _same(y, want) and (clipped, nonfinite) == (wc, wn)
    # an odd length (scalar column at the end) and a misaligned row (scalar path throughout)
    y2, _, _ = ops.secagg_mask(model[1:1001].to(DEV), theta[1:1001].to(DEV), keys, signs, 0.25, 22)
    assert _same(y2, reference.secagg_mask(model[1:1001], theta[1:1001], keys, signs, 0.25, 22)[0])


@pytest.mark.parametrize("K", [2, 10, 33, 100])
@pytest.mark.parametrize("ndrop", [0, 1, 10])
def test_apply_bit_exact(K, ndrop):
    P = 100_003
    g = torch.Generator().manual_seed(K * 16 + ndrop)
    theta = torch.randn(P, generator=g)
    masked = torch.randint(-2 ** 31, 2 ** 31, (K, P), generator=g, dtype=torch.int64).to(torch.int32)
    S = K * (1 + ndrop)
    keys, signs = _keys(S, K + 1000 * ndrop), [1 if i % 3 else -1 for i in range(S)]
    want = reference.fedavg_apply_secagg(theta.clone(), masked, keys, signs, 20, K, 0.7)
    got = theta.to(DEV)
    ops.fedavg_apply_secagg(got, masked.to(DEV), keys, signs, 20, K, 0.7)
    assert _same(got, want)
    again = theta.to(DEV)
    ops.fedavg_apply_secagg(again, masked.to(DEV), keys, signs, 20, K, 0.7)
    assert _same(got, again)
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(P, DEV), opt.init_state(P)
    want = reference.fedavg_apply_secagg(theta.clone(), masked, keys, signs, 20, K, opt=ref)
    got = theta.to(DEV)
    ops.fedavg_apply_secagg(got, masked.to(DEV), keys, signs, 20, K, opt=st)
    assert _same(got, want) and _same(st.m, ref.m) and _same(st.v, ref.v)


@pytest.mark.parametrize("S", [300, 2000])
def test_ffnn_shape_with_thousands_of_streams_takes_the_split_path(S):
    P, K = 2401, 90
    g = torch.Generator().manual_seed(S)
    theta = torch.randn(P, generator=g)
    masked = torch.randint(-2 ** 31, 2 ** 31, (K, P), generator=g, dtype=torch.int64).to(torch.int32)
    keys, signs = _keys(S, S), [1 if i % 2 else -1 for i in range(S)]
    want = reference.fedavg_apply_secagg(theta.clone(), masked, keys, signs, 24, K)
    got = theta.to(DEV)
    ops.fedavg_apply_secagg(got, masked.to(DEV), keys, signs, 24, K)
    assert _same(got, want)


def test_remote_round_cuda_workers_and_coordinator(tmp_path):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw

    workers = []
    for seed in (1, 2, 3):
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=DEV)
        w.add_dataset(BaseDataset(*synthetic_unsw(256, seed=seed)))
        w.start(block=False)
        workers.append(w)
    try:
        args = Arguments(model="mlp", lr=0.05, batch_size=16, federate_after_n_batches=10, synthetic=64, secure_agg=True)
        broker, clock = InProcessBroker(), FakeClock()
        c = Coordinator(1, True, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "r.pth"),
                        device=DEV, evaluate_after=False)
        c.connect()
        c.subscribe("topic/state")
        pub = BusClient("pub", broker=broker)
        pub.connect()
        for w in workers:
            pub.publish("topic/state", f"(127.0.0.1, {w.port}, TRAINING)")
        c.drain()
        clock.advance(1.0)
        res = c.windower.last_result
        recs = [r for r in c.metrics.records if "secagg_u2" in r]
        assert res["dropped"] == [] and all(w.fits_served == 2 for w in workers)
        assert len(recs) == 2 and all(r["secagg_u2"] == 3 and not r["secagg_abandoned"] for r in recs)
    finally:
        for w in workers:
            w.stop()
        settings.training_devices.clear()
