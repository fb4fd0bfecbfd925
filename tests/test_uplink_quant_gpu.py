"""Uplink codec kernels on the H100: quantize_delta_kernel bit for bit against the reference at P = 1 M + 37,
fedavg_q_kernel / fedavg_q_robust_kernel against the reference at K up to 100 (mean with the fedavg_apply tolerance, robust
kinds bit for bit, NaN meeting NaN), a local-mode Coordinator window on CUDA against the same window on CPU, and one
remote-mode round with a CUDA worker and a CUDA coordinator over localhost."""
import socket

import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec
from colearn_federated_learning_b200.ops import reference

pytestmark = pytest.mark.gpu
CODECS = [UplinkCodec("int8"), UplinkCodec("int4")]
DEV = torch.device("cuda", 0)


def same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    nan = a.isnan()
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_encode_delta_bit_exact(codec):
    P, K = (1 << 20) + 37, 3
    g = torch.Generator().manual_seed(1)
    theta = torch.randn(P, generator=g)
    models = theta + torch.randn(K, P, generator=g) * 0.01
    models[1, 5000] = float("nan")
    models[2, :256] = theta[:256]                                  # an all-zero block
    keys = [123, 0xFFFFFFFF, 2 ** 31 + 5]
    payload, scales = ops.encode_delta(models.to(DEV), theta.to(DEV), codec, keys)
    want_p, want_s = reference.encode_delta(models, theta, codec.bits, keys)
    assert payload.is_cuda and payload.shape == want_p.shape
    assert torch.equal(payload.cpu(), want_p) and same_bits(scales, want_s)
    # P % 4 != 0 (scalar path)
    p2, s2 = ops.encode_delta(models[:, :999].contiguous().to(DEV), theta[:999].to(DEV), codec, keys)
    w2, ws2 = reference.encode_delta(models[:, :999], theta[:999], codec.bits, keys)
    assert torch.equal(p2.cpu(), w2) and same_bits(s2, ws2)


@pytest.mark.parametrize("K", [1, 3, 16, 33, 100])
@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_fedavg_apply_quantized_matches_reference(K, codec):
    P = 100_003
    g = torch.Generator().manual_seed(K)
    theta = torch.randn(P, generator=g)
    models = theta + torch.randn(K, P, generator=g) * torch.rand(K, 1, generator=g)
    if K > 2:
        models[1] = theta + 1e4
    payload, scales = reference.encode_delta(models, theta, codec.bits, list(range(K)))
    w = torch.rand(K, generator=g) + 0.1
    w /= w.sum()
    got = theta.to(DEV)
    ops.fedavg_apply_quantized(got, payload.to(DEV), scales.to(DEV), w.to(DEV), codec, 0.7)
    want = reference.fedavg_apply_quantized(theta.clone(), payload, scales, w, codec.bits, 0.7)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-5)
    for agg in (Aggregator("median"), Aggregator("trimmed_mean", 0.2)):
        got = theta.to(DEV)
        ops.fedavg_apply_quantized(got, payload.to(DEV), scales.to(DEV), w.to(DEV), codec, aggregator=agg)
        want = reference.fedavg_apply_quantized(theta.clone(), payload, scales, None, codec.bits, aggregator=agg)
        assert same_bits(got, want), agg
    # FedAdam on the same deltas
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(P, DEV), opt.init_state(P)
    got = theta.to(DEV)
    ops.fedavg_apply_quantized(got, payload.to(DEV), scales.to(DEV), w.to(DEV), codec, opt=st)
    want = reference.fedavg_apply_quantized(theta.clone(), payload, scales, w, codec.bits, opt=ref)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(st.m.cpu(), ref.m, rtol=1e-5, atol=1e-5)


def _window(tmp_path, device, uplink):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.models import MLP, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    args = Arguments(model="mlp", synthetic=512, lr=0.05, batch_size=8, federate_after_n_batches=5, uplink=uplink)
    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, False, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / f"{device.type}.pth"),
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
    gpu = _window(tmp_path, DEV, "int8")
    cpu = _window(tmp_path, torch.device("cpu"), "int8")
    gpu32, cpu32 = _window(tmp_path, DEV, "fp32"), _window(tmp_path, torch.device("cpu"), "fp32")
    # the local fits differ in the last bits between the fused CUDA trainer and the CPU executor (the fp32 windows show how
    # far), and a code can flip where a value sits on a rounding boundary: such a flip moves one parameter by one step
    # (~|delta| / 127), so the int8 windows agree to the fp32 windows' divergence plus a few steps
    diff, diff32 = (gpu - cpu).abs(), (gpu32 - cpu32).abs()
    assert float(diff.max()) < float(diff32.max()) + 5e-3, (float(diff.max()), float(diff32.max()))
    assert float(diff.mean()) < float(diff32.mean()) + 1e-4, (float(diff.mean()), float(diff32.mean()))
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
        args = Arguments(model="mlp", lr=0.05, batch_size=16, federate_after_n_batches=10, uplink="int4", synthetic=64)
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
        assert res["uplink"] == "int4" and res["dropped"] == [] and w.fits_served == 1
        rec = [r for r in c.metrics.records if "bytes_in" in r][0]
        assert rec["bytes_in"] < UplinkCodec("fp32").payload_bytes(4994) / 6
    finally:
        w.stop()
        settings.training_devices.clear()
