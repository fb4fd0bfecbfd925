"""Compressed downlink without a GPU: the numpy definition against an independent scalar transcription (edge blocks
included), coordinator / device lockstep, how fast the replica tracks a frozen model, the kernel sources of elementwise.cu on
the SIMT CPU build, remote mode over TCP (traffic, replica crcs, refused requests, a device with a wrong replica), local
mode and the CLI.

Everything here is bit-exact: the encode and the replica update are fixed fp32 roundings, and a NaN compares as NaN
because the GPU writes its canonical NaN."""
import os
import socket

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.control.coordinator import check_quantized_reply, check_topk_reply
from colearn_federated_learning_b200.fl.uplink import UplinkCodec, downlink_key
from colearn_federated_learning_b200.ops import reference

f32 = np.float32
M32 = 0xFFFFFFFF
CODECS = [UplinkCodec("int8"), UplinkCodec("int4"), UplinkCodec("topk", 1), UplinkCodec("topk", 8), UplinkCodec("topk", 32)]
IDS = ["int8", "int4", "topk1", "topk8", "topk32"]


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
    a, b = a.cpu().reshape(-1), b.cpu().reshape(-1)
    nan = a.isnan()
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


def _bits(x):
    return int(np.array(x, dtype=f32).view(np.uint32))


def _float(b):
    return np.array(b, dtype=np.uint32).view(f32)[()]


# ---- an independent scalar transcription of downlink.cuh -------------------------------------------------------------------
def _fmix(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    return h ^ (h >> 16)


def _uniform(key, j):
    return f32(_fmix(key ^ ((j * 0x9E3779B9) & M32)) >> 8) * f32(2.0 ** -24)


def _scalar_quant(theta, replica, bits, key):
    L = 127 if bits == 8 else 7
    t, r = theta.numpy(), replica.numpy().copy()
    P = t.size
    codes, steps = [], []
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        for b0 in range(0, P, 256):
            js = range(b0, min(P, b0 + 256))
            d = {j: f32(t[j]) - f32(r[j]) for j in js}
            smax = max(_bits(d[j]) & 0x7FFFFFFF for j in js)
            if smax >= 0x7F800000:
                step, inv = _float(0x7FC00000), f32(0.0)
            else:
                inv = f32(L) / _float(smax)
                step = _float(smax) / f32(L)
                if not inv <= np.finfo(f32).max:
                    step, inv = f32(0.0), f32(0.0)
            steps.append(step)
            for j in js:
                q = 0
                if inv != 0:
                    u = f32(d[j] * inv)
                    fl = np.floor(u)
                    q = min(L, max(-L, int(fl) + (1 if _uniform(key, j) < f32(u - fl) else 0)))
                codes.append(q)
                r[j] = f32(r[j] + f32(f32(q) * step))
    q = np.array(codes, dtype=np.int8)
    if bits == 8:
        payload = q.view(np.uint8)
    else:
        nib = np.concatenate([q.astype(np.uint8) & 0xF, np.zeros(P % 2, dtype=np.uint8)])
        payload = nib[0::2] | (nib[1::2] << 4)
    return torch.from_numpy(payload.copy()), torch.from_numpy(np.array(steps, dtype=f32)), torch.from_numpy(r)


def _key(x):
    a = _bits(x) & 0x7FFFFFFF
    return 0x7F800001 if a > 0x7F800000 else a


def _scalar_topk(theta, replica, k):
    t, r = theta.numpy(), replica.numpy().copy()
    P = t.size
    ids, vals = [], []
    with np.errstate(invalid="ignore", over="ignore"):
        for b0 in range(0, P, 256):
            js = list(range(b0, min(P, b0 + 256)))
            v = {j: f32(t[j]) - f32(r[j]) for j in js}
            kept = sorted(sorted(js, key=lambda j: (-_key(v[j]), j))[:min(k, len(js))])
            ids += [j - b0 for j in kept]
            vals += [v[j] for j in kept]
            for j in kept:
                r[j] = f32(r[j] + v[j])
    return torch.tensor(ids, dtype=torch.uint8), torch.from_numpy(np.array(vals, dtype=f32)), torch.from_numpy(r)


def _scalar(theta, replica, codec, key):
    return _scalar_quant(theta, replica, codec.bits, key) if codec.quantized else _scalar_topk(theta, replica, codec.k)


def _pair(P, seed, scale=0.01):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    return theta, theta + scale * torch.randn(P, generator=g) * torch.rand(1, generator=g)


@pytest.mark.parametrize("P", [1, 255, 256, 257, 4994])
@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_reference_matches_scalar_transcription(P, codec):
    theta, rep = _pair(P, seed=P)
    key = downlink_key(P)
    want_a, want_b, want_r = _scalar(theta, rep, codec, key)
    r = rep.clone()
    a, b = reference.encode_downlink(theta, r, codec, key)
    if codec.quantized:
        assert a.shape == (codec.payload_bytes(P),) and b.shape == (codec.scale_count(P),)
    else:
        assert a.shape == b.shape == (codec.entries(P),) and a.dtype == torch.uint8
    assert torch.equal(a, want_a) and same_bits(b, want_b) and same_bits(r, want_r)
    # CPU tensors through ops: the reference itself
    r2 = rep.clone()
    a2, b2 = ops.encode_downlink(theta, r2, codec, key)
    assert torch.equal(a2, a) and same_bits(b2, b) and same_bits(r2, r)


def _edge_pair(P=5 * 256 + 3):
    """block 0: theta == replica; block 1: +-0 in both; block 2: a difference that underflows the codec's scale (and a
    subnormal); block 3: equal magnitudes (ties go to the lower index); block 4: random; last block 3 long"""
    g = torch.Generator().manual_seed(7)
    theta = torch.randn(P, generator=g)
    rep = theta + 0.01 * torch.randn(P, generator=g)
    rep[:256] = theta[:256]
    theta[256:512] = torch.tensor([0.0, -0.0]).repeat(128)
    rep[256:512] = torch.tensor([-0.0, 0.0, 0.0, -0.0]).repeat(64)
    theta[512:768] = 1e-38
    rep[512:768] = 1e-38
    theta[512 + 5] = 1e-38 + 1e-44                                 # d = one subnormal step: L / s overflows, step 0
    theta[768:1024] = 0.5
    rep[768:1024] = 0.5 + 0.25 * torch.tensor([1.0, -1.0]).repeat(128)
    return theta, rep


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_edge_blocks(codec):
    theta, rep = _edge_pair()
    key = downlink_key(3)
    r = rep.clone()
    a, b = reference.encode_downlink(theta, r, codec, key)
    want_a, want_b, want_r = _scalar(theta, rep, codec, key)
    assert torch.equal(a, want_a) and same_bits(b, want_b) and same_bits(r, want_r)
    assert torch.equal(r[:256], rep[:256])                         # theta == replica: the replica keeps its values
    assert (r[256:512] == 0).all()                                 # +-0: still zeros
    if codec.quantized:
        assert float(b[0]) == 0.0 and float(b[1]) == 0.0 and float(b[2]) == 0.0     # all-zero and underflowing blocks: step 0
        codes = reference.decode_codes(a.view(1, -1), codec.bits, theta.numel())[0]
        assert (codes[:768] == 0).all()
        assert torch.equal(r[512:768], rep[512:768])               # nothing delivered below the codec's resolution
    else:
        k = codec.k
        assert a[:k].tolist() == list(range(k))                    # theta == replica: the lowest offsets, value 0
        assert (b[:k] == 0).all()
        assert 5 in a[2 * k:3 * k].tolist()                        # the only non-zero difference of the block is sent
        assert a[3 * k:4 * k].tolist() == list(range(k))           # equal magnitudes: ties go to the lower index
        assert torch.equal(r[768:768 + k], theta[768:768 + k])


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_device_replica_follows_the_coordinator_in_lockstep(codec):
    """30 rounds of a moving theta: the coordinator encodes and advances its replica, the device checks the wire bytes as a
    worker does and applies them to its own replica; the two are bit-identical every round"""
    P = 1001
    g = torch.Generator().manual_seed(1)
    theta = torch.randn(P, generator=g)
    coord, dev = theta.clone(), theta.clone()
    for t in range(1, 31):
        theta += (0.01 if t % 7 else 1.0) * torch.randn(P, generator=g)
        a, b = ops.encode_downlink(theta, coord, codec, downlink_key(100 + t))
        if codec.quantized:
            wire = check_quantized_reply({"uplink": codec.kind, "payload": a.numpy().tobytes(), "scales": b.numpy().tobytes()}, codec, P)
        else:
            wire = check_topk_reply({"uplink": "topk", "topk": codec.k, "indices": a.numpy().tobytes(), "values": b.numpy().tobytes()},
                                    codec, P)
        ops.apply_downlink(dev, *wire, codec)
        assert same_bits(dev, coord), t
    assert not torch.equal(coord, theta)                           # the replica lags: something is still to be delivered


def test_int8_replica_tracks_a_frozen_model_by_a_factor_of_L_per_round():
    """each round shrinks max|theta - r| by at least L = 127 (|q step - d| <= step = max|d| / L) until the fp32 rounding of
    r + q step, at most 2 ulps of max|theta| here"""
    P = 4994
    g = torch.Generator().manual_seed(2)
    theta = torch.randn(P, generator=g)
    r = torch.zeros(P)
    ulp = float(np.spacing(f32(theta.abs().max())))
    err = float((theta - r).abs().max())
    floor_rounds = 0
    for t in range(12):
        reference.encode_downlink(theta, r, UplinkCodec("int8"), downlink_key(t))
        new = float((theta - r).abs().max())
        assert new <= max(err / 127 * (1 + 1e-6), 2 * ulp), (t, err, new)
        floor_rounds += new <= 2 * ulp
        err = new
    assert floor_rounds >= 8                                       # 4 rounds reach the floor from |theta| ~ 4


@pytest.mark.parametrize("k", [1, 8, 32])
def test_topk_replica_reaches_a_frozen_model(k):
    """every round delivers the k largest differences of every block: after ceil(256 / k) + 2 rounds the replica is within
    1 ulp of theta everywhere (r + (theta - r) is one rounding away from theta)"""
    P = 1001
    g = torch.Generator().manual_seed(k)
    theta = torch.randn(P, generator=g)
    r = theta * (1 + 0.01 * torch.randn(P, generator=g))
    for t in range(-(-256 // k) + 2):
        reference.encode_downlink(theta, r, UplinkCodec("topk", k), 0)
    ulps = np.spacing(np.abs(theta.numpy()))
    assert (np.abs(theta.numpy() - r.numpy()) <= ulps).all()


def test_ops_refuse_what_they_cannot_do():
    theta = torch.randn(300)
    with pytest.raises(ValueError):
        ops.encode_downlink(theta, theta.clone(), UplinkCodec("fp32"), 0)
    with pytest.raises(ValueError):
        ops.encode_downlink(theta, theta.double(), UplinkCodec("int8"), 0)
    with pytest.raises(ValueError):
        ops.encode_downlink(theta, torch.zeros(301), UplinkCodec("topk"), 0)
    with pytest.raises(ValueError):
        ops.apply_downlink(theta.clone(), torch.zeros(300, dtype=torch.uint8), torch.zeros(2), UplinkCodec("fp32"))


# ---- elementwise.cu on the SIMT CPU build ------------------------------------------------------------------------------------
def _simt_encode(simt, theta, r, codec, key):
    if codec.quantized:
        payload, scales = simt.downlink_quant(theta, r, key, codec.bits)
        assert payload.numel() % 16 == 0
        return payload[:codec.payload_bytes(theta.numel())], scales
    return simt.downlink_topk(theta, r, codec.k)


def _simt_apply(simt, r, a, b, codec):
    if codec.quantized:
        pad = torch.zeros((a.numel() + 15) // 16 * 16, dtype=torch.uint8)
        pad[:a.numel()] = a
        simt.replica_apply_quant(r, pad, b, codec.bits)
    else:
        simt.replica_apply_topk(r, a, b, codec.k)


@pytest.mark.parametrize("codec", CODECS, ids=IDS)
def test_downlink_kernels_on_cpu_bit_exact(simt, codec):
    key = downlink_key(9)
    for P in (1, 5, 255, 256, 257, 1000, 1001, 1024, 4994):        # 16-byte path when P % 4 == 0, scalar path otherwise
        theta, rep = _pair(P, seed=P + codec.k)
        if P >= 1000:
            theta[260], theta[300] = float("nan"), float("-inf")   # non-finite differences: NaN step / always sent
            rep[:256] = theta[:256]                                # a block with nothing to send
        r_ref, r_sim, dev_ref, dev_sim = rep.clone(), rep.clone(), rep.clone(), rep.clone()
        a, b = reference.encode_downlink(theta, r_ref, codec, key)
        a2, b2 = _simt_encode(simt, theta, r_sim, codec, key)
        assert torch.equal(a2, a) and same_bits(b2, b) and same_bits(r_sim, r_ref), P
        reference.apply_downlink(dev_ref, a, b, codec)
        _simt_apply(simt, dev_sim, a, b, codec)
        assert same_bits(dev_sim, dev_ref) and same_bits(dev_ref, r_ref), P
    # replica and theta not 16-byte aligned (views one float into a buffer): the scalar path, same bits
    buf, tbuf = torch.randn(1001), torch.randn(1001)
    theta, rep = tbuf[1:], buf[1:]
    r_ref = rep.clone()
    a, b = reference.encode_downlink(theta, r_ref, codec, key)
    a2, b2 = _simt_encode(simt, theta, rep, codec, key)
    assert torch.equal(a2, a) and same_bits(b2, b) and same_bits(rep, r_ref)
    dev, dev2 = torch.zeros(1001)[1:], torch.zeros(1001)[1:]
    dev.copy_(tbuf[1:] + 0.5)
    dev2.copy_(dev)
    reference.apply_downlink(dev, a, b, codec)
    _simt_apply(simt, dev2, a, b, codec)
    assert same_bits(dev2, dev)


# ---- remote mode over TCP ---------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _coordinator(tmp_path, args, rounds, remote=True):
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.utils.metrics import RoundLogger

    class Losses(RoundLogger):
        def __init__(self):
            super().__init__()
            self.per_round = [[]]

        def worker_loss(self, worker_id, loss):
            self.per_round[-1].append(loss)

        def end_round(self, round_idx, seconds, **fields):
            self.per_round.append([])
            return super().end_round(round_idx, seconds, **fields)

    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, remote, rounds, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "test.pth"),
                    device=torch.device("cpu"), metrics=Losses(), evaluate_after=False)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    return c, pub, clock


def _worker(seed, cls=None):
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw
    port = _free_port()
    w = (cls or WorkerServer)(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
    w.add_dataset(BaseDataset(*synthetic_unsw(256, seed=seed)))
    w.start(block=False)
    return w, port


def _args(uplink, downlink, model="ffnn"):
    from colearn_federated_learning_b200.control.arguments import Arguments
    return Arguments(model=model, lr=0.1, batch_size=16, federate_after_n_batches=30, uplink=uplink, uplink_topk=8, downlink=downlink,
                     downlink_topk=8, synthetic=64)


def _train(tmp_path, args, workers, rounds):
    torch.manual_seed(0)
    c, pub, clock = _coordinator(tmp_path, args, rounds)
    for w in workers:
        pub.publish("topic/state", f"(127.0.0.1, {w.port}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    return c, c.windower.last_result


def _remote_run(tmp_path, uplink, downlink, rounds=3, stub=None, model="ffnn"):
    workers = [_worker(1)[0], _worker(2)[0]] + ([_worker(3, stub)[0]] if stub is not None else [])
    try:
        c, res = _train(tmp_path / f"{uplink}-{downlink}", _args(uplink, downlink, model), workers, rounds)
        return c, res, workers
    finally:
        for w in workers:
            w.stop()


# downlink wire bytes of the FFNN's 2,401 parameters (10 blocks, the last one 97 long)
WIRE = {"int8": 2401 + 40, "int4": 1201 + 40, "topk": 400}
# msgpack framing of the wire fields, the two replica tags and the codec fields, less the fp32 params' own framing
OVERHEAD = 120


@pytest.mark.parametrize("uplink,downlink", [("int8", "int8"), ("int8", "int4"), ("topk", "topk"), ("topk", "int8")])
def test_remote_rounds_with_a_compressed_downlink(tmp_path, uplink, downlink):
    fp32, res32, _ = _remote_run(tmp_path / "a", uplink, "fp32")
    out32 = [r["bytes_out"] for r in fp32.metrics.records if "bytes_out" in r]
    c, res, workers = _remote_run(tmp_path / "b", uplink, downlink)
    out = [r["bytes_out"] for r in c.metrics.records if "bytes_out" in r]
    # every device kept the coordinator's replica (a crc mismatch would have dropped it) and trained every round
    assert res["downlink"] == downlink and res["dropped"] == [] and all(w.fits_served == 3 for w in workers)
    assert len(out) == len(out32) == 3 and res32["downlink"] == "fp32"
    assert abs(out[0] - out32[0]) <= 2 * 80                        # round 0 carries the fp32 model plus codec fields and a tag
    for r in (1, 2):
        saved = (out32[r] - out[r]) / 2                            # per device
        assert 9604 - WIRE[downlink] - OVERHEAD <= saved <= 9604 - WIRE[downlink], (r, saved, out32, out)
    held = [w._replicas["ffnn"] for w in workers]
    assert held[0][0] == held[1][0] and held[0][0].endswith(":2") and same_bits(held[0][1], held[1][1])


def test_remote_loss_falls_with_a_compressed_downlink(tmp_path):
    c, res, _ = _remote_run(tmp_path, "int8", "int8", model="mlp")
    losses = [np.mean(l) for l in c.metrics.per_round if l]
    assert res["dropped"] == [] and len(losses) == 3 and losses[2] < losses[0], losses


def test_without_the_flag_requests_and_replies_are_unchanged(tmp_path):
    from colearn_federated_learning_b200.control.workers import WorkerServer
    seen = []

    class Recording(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            if req.get("op") == "fit":
                seen.append((list(req), list(resp)))
            return resp

    _remote_run(tmp_path, "int8", "fp32", rounds=2, stub=Recording)
    assert seen and all(r == ["op", "config", "params", "dataset_key", "uplink"] for r, _ in seen)
    assert all(r == ["ok", "uplink", "payload", "scales", "loss", "n", "path"] for _, r in seen)


def test_a_device_with_a_wrong_replica_crc_is_dropped(tmp_path):
    from colearn_federated_learning_b200.control.workers import WorkerServer

    class WrongCrc(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            if req.get("op") == "fit" and resp.get("ok") and "replica_base" in req:
                resp["replica_crc"] ^= 1
            return resp

    c, res, workers = _remote_run(tmp_path, "topk", "int4", rounds=3, stub=WrongCrc)
    bad = f"127.0.0.1:{workers[2].port}"
    # round 0 (fp32 model, matching crc) is taken; its round-1 reply is dropped and it leaves the training
    assert res["dropped"] == [bad] and workers[2].fits_served == 2
    assert all(w.fits_served == 3 for w in workers[:2])


def test_a_worker_resynchronises_at_the_next_training(tmp_path):
    workers = [_worker(1)[0], _worker(2)[0]]
    try:
        _, first = _train(tmp_path / "1", _args("int8", "topk"), workers, 2)
        tag1 = workers[0]._replicas["ffnn"][0]
        _, second = _train(tmp_path / "2", _args("int8", "topk"), workers, 2)
        tag2 = workers[0]._replicas["ffnn"][0]
    finally:
        for w in workers:
            w.stop()
    assert first["dropped"] == second["dropped"] == [] and all(w.fits_served == 4 for w in workers)
    assert tag1.endswith(":1") and tag2.endswith(":1") and tag1.split(":")[0] != tag2.split(":")[0]


@pytest.fixture()
def round0():
    """a worker that took a round-0 request (int8 uplink, downlink `codec`), a client to it and the coordinator's replica"""
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    from colearn_federated_learning_b200.models import FFNN, flatten_params

    w, port = _worker(1)
    client = RemoteWorkerClient(w.id, "127.0.0.1", port)
    torch.manual_seed(0)
    theta = flatten_params(FFNN()).detach().clone()
    cfg = FitConfig(model="ffnn", loss="bce", batch_size=16, epochs=1, max_nr_batches=5, lr=0.1, shuffle=True, seed=1).to_dict()

    def start(codec):
        base = {"op": "fit", "config": cfg, "dataset_key": "training", "uplink": "int8", "downlink": codec.kind, "downlink_topk": codec.k}
        resp = client._call({**base, "params": theta.numpy().tobytes(), "replica": "n:0"})
        assert resp["replica_crc"] == __import__("zlib").crc32(theta.numpy().tobytes())
        return base
    yield w, client, theta, start
    client.close()
    w.stop()


def _wire_fields(codec, a, b):
    names = ("dpayload", "dscales") if codec.quantized else ("dindices", "dvalues")
    return {names[0]: a.numpy().tobytes(), names[1]: b.numpy().astype("<f4").tobytes()}


def _scales_with(value):
    def f(fields):
        s = np.frombuffer(fields["dscales"], dtype="<f4").copy()
        s[1] = value
        fields["dscales"] = s.tobytes()
    return f


def _offsets_with(fn):
    def f(fields):
        i = np.frombuffer(fields["dindices"], dtype=np.uint8).copy()
        fn(i)
        fields["dindices"] = i.tobytes()
    return f


TAMPER = {
    "wrong_replica_base": (UplinkCodec("int8"), lambda f: f.update(replica_base="n:5")),
    "previous_training_tag": (UplinkCodec("int8"), lambda f: f.update(replica_base="m:0")),
    "short_payload": (UplinkCodec("int8"), lambda f: f.update(dpayload=f["dpayload"][:-1])),
    "missing_scales": (UplinkCodec("int4"), lambda f: f.pop("dscales")),
    "nan_scale": (UplinkCodec("int8"), _scales_with(np.nan)),
    "oversize_scale": (UplinkCodec("int4"), _scales_with(np.finfo(np.float32).max / 6)),
    "short_indices": (UplinkCodec("topk", 8), lambda f: f.update(dindices=f["dindices"][:-1])),
    "descending_offsets": (UplinkCodec("topk", 8), _offsets_with(lambda i: i.__setitem__(slice(8, 10), i[8:10][::-1].copy()))),
    "offset_past_last_block": (UplinkCodec("topk", 8), _offsets_with(lambda i: i.__setitem__(-1, 97))),
    "inf_value": (UplinkCodec("topk", 8), lambda f: f.update(dvalues=np.full(80, np.inf, dtype="<f4").tobytes())),
    "wrong_downlink_topk": (UplinkCodec("topk", 8), lambda f: f.update(downlink_topk=33)),
    "no_replica_tag": (UplinkCodec("topk", 8), lambda f: f.pop("replica")),
}


@pytest.mark.parametrize("case", sorted(TAMPER))
def test_a_tampered_downlink_is_refused_and_the_replica_kept(round0, case):
    w, client, theta, start = round0
    codec, mutate = TAMPER[case]
    base = start(codec)
    before_tag, before = w._replicas["ffnn"][0], w._replicas["ffnn"][1].clone()
    coord = theta.clone()
    a, b = reference.encode_downlink(theta + 0.01 * torch.randn(theta.numel()), coord, codec, downlink_key(2))
    fields = {**_wire_fields(codec, a, b), "replica_base": "n:0", "replica": "n:1"}
    mutate(fields)
    served = w.fits_served
    with pytest.raises(RuntimeError):
        client._call({**base, **fields})
    assert w.fits_served == served and w._replicas["ffnn"][0] == before_tag and torch.equal(w._replicas["ffnn"][1], before)
    # the untampered wire is taken: the device's replica is the coordinator's
    resp = client._call({**base, **_wire_fields(codec, a, b), "replica_base": "n:0", "replica": "n:1"})
    assert w._replicas["ffnn"][0] == "n:1" and same_bits(w._replicas["ffnn"][1], coord)
    assert resp["replica_crc"] == __import__("zlib").crc32(coord.numpy().tobytes())


def test_a_round0_request_without_params_is_refused(round0):
    w, client, theta, start = round0
    base = start(UplinkCodec("int8"))
    before = w._replicas["ffnn"][1].clone()
    with pytest.raises(RuntimeError):
        client._call({**base, "replica": "k:0"})
    assert w._replicas["ffnn"][0] == "n:0" and torch.equal(w._replicas["ffnn"][1], before)


# ---- local mode and the CLI -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("uplink,downlink", [("int8", "int4"), ("topk", "topk")])
def test_local_mode_with_a_compressed_downlink(tmp_path, uplink, downlink):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.coordinator import train_virtual_workers
    from colearn_federated_learning_b200.data import BaseDataset, federate, synthetic_unsw
    from colearn_federated_learning_b200.fl.uplink import uplink_key
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    args = Arguments(synthetic=90, lr=0.05, uplink=uplink, uplink_topk=4, downlink=downlink, downlink_topk=4)
    c, pub, clock = _coordinator(tmp_path, args, rounds=3, remote=False)
    torch.manual_seed(0)
    init = FFNN()
    save_model(init, c.path)
    ips = ["10.0.0.1", "10.0.0.2", "10.0.0.3"]
    for ip in ips:
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert c.windower.last_result["downlink"] == downlink
    x, y = synthetic_unsw(90, seed=args.seed)
    fed = federate(BaseDataset(x, y), ips, torch.device("cpu"))
    cfg = c._fit_config("local")
    up, down = args.uplink_codec(), args.downlink_codec()
    theta = flatten_params(init).clone()
    replica = theta.clone()
    res = torch.zeros(3, theta.numel())
    w = torch.full((3,), 1.0 / 3)
    for r in range(3):
        if r:
            reference.encode_downlink(theta, replica, down, downlink_key(cfg.seed + r))
        flats, _, _ = train_virtual_workers(replica, FFNN(), fed, cfg, r)
        if up.quantized:
            payload, scales = reference.encode_delta(flats, replica, up.bits, [uplink_key(ip, cfg.seed + r) for ip in ips])
            reference.fedavg_apply_quantized(theta, payload, scales, w, up.bits)
        else:
            idx, val = reference.encode_topk_delta(flats, replica, res, up.k)
            reference.fedavg_apply_topk(theta, idx, val, w, up.k)
    assert not torch.equal(replica, theta)
    m = FFNN()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    assert torch.equal(flatten_params(m), theta)
    settings.training_devices.clear()


def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_cli_downlink_flags():
    a = _cli()
    assert a.downlink == "fp32" and a.downlink_topk == 8 and a.downlink_codec().kind == "fp32"
    assert _cli("--uplink-codec", "int8", "--downlink-codec", "int4").downlink_codec().bits == 4
    c = _cli("--uplink-codec", "int4", "--downlink-codec", "topk", "--downlink-topk", "32", "-r").downlink_codec()
    assert c.sparse and c.k == 32
    assert _cli("--uplink-codec", "topk", "--downlink-codec", "topk").downlink_codec().k == 8
    assert _cli("--uplink-codec", "int8", "--downlink-codec", "int8", "--aggregator", "median").downlink_codec().quantized
    for bad in (["--uplink-codec", "int8", "--downlink-codec", "int8", "--box"], ["--uplink-codec", "int8", "--downlink-codec", "topk", "-e"],
                ["--downlink-codec", "int8"], ["--uplink-codec", "fp32", "--downlink-codec", "topk"],
                ["--uplink-codec", "int8", "--downlink-codec", "topk", "--downlink-topk", "0"],
                ["--uplink-codec", "int8", "--downlink-codec", "topk", "--downlink-topk", "33"]):
        with pytest.raises(SystemExit):
            _cli(*bad)
