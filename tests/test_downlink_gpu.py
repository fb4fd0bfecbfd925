"""Compressed downlink kernels on the H100: downlink_quant_kernel / downlink_topk_kernel bit for bit against the reference at
P = 1 M + 37 (wire bytes and the advanced replica, NaN meeting NaN), replica_apply_q_kernel / replica_apply_topk_kernel bit
for bit, 20 rounds of a CUDA coordinator replica against a CPU-reference device replica (equal crcs every round) with
identical bits on a second run, and a remote training with a CUDA worker and a CUDA coordinator over localhost."""
import socket
import zlib

import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl.uplink import UplinkCodec, downlink_key
from colearn_federated_learning_b200.ops import reference

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
CODECS = [UplinkCodec("int8"), UplinkCodec("int4"), UplinkCodec("topk", 1), UplinkCodec("topk", 8), UplinkCodec("topk", 32)]
IDS = ["int8", "int4", "topk1", "topk8", "topk32"]


def same_bits(a, b):
    a, b = a.cpu().reshape(-1), b.cpu().reshape(-1)
    nan = a.isnan()
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


def _pair(P, seed):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    rep = theta + 0.01 * torch.randn(P, generator=g)
    rep[:256] = theta[:256]                                        # a block with nothing to send
    theta[5000], theta[5003] = float("nan"), float("-inf")
    return theta, rep


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_encode_and_advance_bit_exact(codec):
    P = (1 << 20) + 37
    theta, rep = _pair(P, seed=codec.k + codec.bits)
    key = downlink_key(11)
    r_gpu, r_ref = rep.to(DEV), rep.clone()
    a, b = ops.encode_downlink(theta.to(DEV), r_gpu, codec, key)
    want_a, want_b = reference.encode_downlink(theta, r_ref, codec, key)
    assert a.is_cuda and a.shape == want_a.shape and b.shape == want_b.shape
    assert torch.equal(a.cpu(), want_a) and same_bits(b, want_b) and same_bits(r_gpu, r_ref)
    # the device side: the same wire applied by replica_apply_*_kernel
    dev_gpu, dev_ref = rep.to(DEV), rep.clone()
    ops.apply_downlink(dev_gpu, want_a.to(DEV), want_b.to(DEV), codec)
    reference.apply_downlink(dev_ref, want_a, want_b, codec)
    assert same_bits(dev_gpu, dev_ref) and same_bits(dev_ref, r_ref)


def _rounds(codec, P=4994, rounds=20):
    """a CUDA coordinator replica and a CPU-reference device replica over `rounds` rounds of a moving theta: their crcs"""
    g = torch.Generator().manual_seed(3)
    theta = torch.randn(P, generator=g)
    coord, dev = theta.to(DEV), theta.clone()
    crcs = []
    for t in range(1, rounds + 1):
        theta += 0.01 * torch.randn(P, generator=g)
        a, b = ops.encode_downlink(theta.to(DEV), coord, codec, downlink_key(t))
        reference.apply_downlink(dev, a.cpu(), b.cpu(), codec)
        crcs.append((zlib.crc32(coord.cpu().numpy().tobytes()), zlib.crc32(dev.numpy().tobytes())))
    return crcs


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_cuda_coordinator_and_cpu_device_agree_every_round(codec):
    first = _rounds(codec)
    assert all(c == d for c, d in first)
    assert _rounds(codec) == first                                 # a second run gives identical bits


def test_remote_rounds_cuda_worker_and_coordinator(tmp_path):
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
        args = Arguments(model="mlp", lr=0.05, batch_size=16, federate_after_n_batches=10, uplink="int8", downlink="topk",
                         downlink_topk=8, synthetic=64)
        broker, clock = InProcessBroker(), FakeClock()
        c = Coordinator(1, True, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "r.pth"),
                        device=DEV, evaluate_after=False)
        c.connect()
        c.subscribe("topic/state")
        pub = BusClient("pub", broker=broker)
        pub.connect()
        pub.publish("topic/state", f"(127.0.0.1, {port}, TRAINING)")
        c.drain()
        clock.advance(1.0)
        res = c.windower.last_result
        # round 1 went out as a top-k wire to the replica, and the device's replica crc matched the coordinator's
        assert res["downlink"] == "topk" and res["dropped"] == [] and w.fits_served == 2
        tag, replica = w._replicas["mlp"]
        assert replica.is_cuda and tag.endswith(":1")
        out = [r["bytes_out"] for r in c.metrics.records if "bytes_out" in r]
        assert out[1] < UplinkCodec("fp32").payload_bytes(4994) / 5
    finally:
        w.stop()
        settings.training_devices.clear()
