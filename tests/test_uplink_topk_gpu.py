"""Top-k uplink kernels on the H100: topk_delta_kernel bit for bit against the reference at P = 1 M + 37 (indices, values
and the residual written back, NaN meeting NaN), fedavg_topk_kernel against the reference at K up to 100 (weighted,
server_lr != 1, FedAdam) and bit-identical between two runs, a local-mode Coordinator window on CUDA against the same
window on CPU, and one remote-mode round with a CUDA worker and a CUDA coordinator over localhost."""
import socket

import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec
from colearn_federated_learning_b200.ops import reference

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    nan = a.isnan()
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


@pytest.mark.parametrize("k", [1, 8, 32])
def test_encode_topk_delta_bit_exact(k):
    P, K = (1 << 20) + 37, 3
    g = torch.Generator().manual_seed(k)
    theta = torch.randn(P, generator=g)
    models = theta + torch.randn(K, P, generator=g) * 0.01
    res = 0.005 * torch.randn(K, P, generator=g)
    models[1, 5000] = float("nan")
    models[1, 5003] = float("-inf")
    models[2, :256] = theta[:256]                                  # an all-zero block
    res[2, :256] = 0.0
    codec = UplinkCodec("topk", k)
    r_gpu, r_ref = res.to(DEV), res.clone()
    idx, val = ops.encode_topk_delta(models.to(DEV), theta.to(DEV), r_gpu, codec)
    want_i, want_v = reference.encode_topk_delta(models, theta, r_ref, k)
    assert idx.is_cuda and idx.shape == want_i.shape == (K, codec.entries(P))
    assert torch.equal(idx.cpu(), want_i) and same_bits(val, want_v) and same_bits(r_gpu, r_ref)
    # P % 4 != 0 (scalar path), a last block shorter than k
    P2 = 999 if k < 32 else 768 + 5
    r2, r2_ref = res[:, :P2].contiguous().to(DEV), res[:, :P2].contiguous()
    i2, v2 = ops.encode_topk_delta(models[:, :P2].contiguous().to(DEV), theta[:P2].to(DEV), r2, codec)
    w2, wv2 = reference.encode_topk_delta(models[:, :P2], theta[:P2], r2_ref, k)
    assert torch.equal(i2.cpu(), w2) and same_bits(v2, wv2) and same_bits(r2, r2_ref)


@pytest.mark.parametrize("K", [1, 3, 16, 33, 100])
@pytest.mark.parametrize("k", [1, 8, 32])
def test_fedavg_apply_topk_matches_reference(K, k):
    P = 100_003
    g = torch.Generator().manual_seed(K * 40 + k)
    theta = torch.randn(P, generator=g)
    models = theta + torch.randn(K, P, generator=g) * torch.rand(K, 1, generator=g)
    if K > 2:
        models[1] = theta + 1e4
    res = torch.zeros(K, P)
    idx, val = reference.encode_topk_delta(models, theta, res, k)
    codec = UplinkCodec("topk", k)
    w = torch.rand(K, generator=g) + 0.1
    w /= w.sum()
    got = theta.to(DEV)
    ops.fedavg_apply_topk(got, idx.to(DEV), val.to(DEV), w.to(DEV), codec, 0.7)
    want = reference.fedavg_apply_topk(theta.clone(), idx, val, w, k, 0.7)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-5)
    again = theta.to(DEV)
    ops.fedavg_apply_topk(again, idx.to(DEV), val.to(DEV), w.to(DEV), codec, 0.7)
    assert torch.equal(got.view(torch.int32), again.view(torch.int32))   # deterministic: the same bits twice
    # FedAdam on the same deltas
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(P, DEV), opt.init_state(P)
    got = theta.to(DEV)
    ops.fedavg_apply_topk(got, idx.to(DEV), val.to(DEV), w.to(DEV), codec, opt=st)
    want = reference.fedavg_apply_topk(theta.clone(), idx, val, w, k, opt=ref)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(st.m.cpu(), ref.m, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(st.v.cpu(), ref.v, rtol=1e-5, atol=1e-7)


def _window(tmp_path, device, uplink):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.models import MLP, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    args = Arguments(model="mlp", synthetic=512, lr=0.05, batch_size=8, federate_after_n_batches=5, uplink=uplink, uplink_topk=8)
    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, False, 3, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / f"{device.type}{uplink}.pth"),
                    device=device)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    torch.manual_seed(0)
    save_model(MLP(), c.path)
    for ip in ("10.0.0.1", "10.0.0.2", "10.0.0.3"):
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert c.windower.last_result["uplink"] == uplink
    m = MLP()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    settings.training_devices.clear()
    return flatten_params(m)


def test_local_mode_window_on_cuda_matches_cpu(tmp_path):
    gpu, cpu = _window(tmp_path, DEV, "topk"), _window(tmp_path, torch.device("cpu"), "topk")
    gpu32, cpu32 = _window(tmp_path, DEV, "fp32"), _window(tmp_path, torch.device("cpu"), "fp32")
    # the local fits differ in the last bits between the fused CUDA trainer and the CPU executor (the fp32 windows show how
    # far); the selection can then differ where two magnitudes of a block are within those bits, and such a flip sends one
    # entry a round early or late: the top-k windows agree to the fp32 windows' divergence except at a few parameters
    diff, diff32 = (gpu - cpu).abs(), (gpu32 - cpu32).abs()
    assert float(diff.mean()) < float(diff32.mean()) + 1e-4, (float(diff.mean()), float(diff32.mean()))
    assert float((diff > float(diff32.max()) + 1e-6).float().mean()) < 0.01
    assert not torch.equal(gpu, gpu32)


def test_remote_round_cuda_worker_and_coordinator(tmp_path):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=DEV)
    w.add_dataset(BaseDataset(*synthetic_unsw(256, seed=1)))
    w.start(block=False)
    try:
        args = Arguments(model="mlp", lr=0.05, batch_size=16, federate_after_n_batches=10, uplink="topk", uplink_topk=8, synthetic=64)
        broker, clock = InProcessBroker(), FakeClock()
        c = Coordinator(1, True, 1, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "r.pth"),
                        device=DEV, evaluate_after=False)
        c.connect()
        c.subscribe("topic/state")
        pub = BusClient("pub", broker=broker)
        pub.connect()
        pub.publish("topic/state", f"(127.0.0.1, {port}, TRAINING)")
        c.drain()
        clock.advance(1.0)
        res = c.windower.last_result
        assert res["uplink"] == "topk" and res["dropped"] == [] and w.fits_served == 1
        assert w._residuals["mlp"].is_cuda and bool(w._residuals["mlp"].any())
        rec = [r for r in c.metrics.records if "bytes_in" in r][0]
        assert rec["bytes_in"] < UplinkCodec("fp32").payload_bytes(4994) / 15
    finally:
        w.stop()
        settings.training_devices.clear()
