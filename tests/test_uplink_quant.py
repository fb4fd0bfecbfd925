"""Uplink compression (int8 / int4 stochastic codec of the client deltas) without a GPU: the PyTorch/numpy definition against
an independent scalar transcription, its statistical properties, the kernel sources of elementwise.cu on the SIMT CPU
build, remote mode over TCP (traffic, validation of untrusted replies), local mode and the CLI.

The encode is bit-exact everywhere (every rounding is fixed by the definition in ops/csrc/uplink_quant.cuh).  The fused
decode + FedAvg compares with the tolerance of the fp32 fedavg_apply tests for the weighted mean (the kernel's fmaf chain
against the reference's torch sum), bit for bit for the robust kinds (ranks are integer counts, the kept values are summed
in slot order from +0, theta + x and the lr = 1 step are single roundings on both sides), and with the tests/test_server_opt.py
tolerance for a FedAdam composition."""
import math
import os
import socket

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec, uplink_key
from colearn_federated_learning_b200.ops import reference

CODECS = [UplinkCodec("int8"), UplinkCodec("int4")]
ROBUST = [Aggregator("median"), Aggregator("trimmed_mean", 0.2)]


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
    nan = a.isnan()
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


def keys_i32(keys):
    return torch.from_numpy(np.array(keys, dtype=np.int64).astype(np.uint32).view(np.int32).copy())


# ---- an independent scalar transcription of uplink_quant.cuh ---------------------------------------------------------------
def _fmix32(h):
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    return h ^ (h >> 16)


def _scalar_encode(models, theta, bits, keys):
    """element by element in Python integers and numpy float32 scalars"""
    L = 127 if bits == 8 else 7
    f32 = np.float32
    m, t = models.numpy().astype(np.float32), theta.numpy().astype(np.float32)
    K, P = m.shape
    codes, scales = [], []
    for k in range(K):
        row_q, row_s = [], []
        for b0 in range(0, P, 256):
            d = [f32(m[k, j]) - f32(t[j]) for j in range(b0, min(P, b0 + 256))]
            if not all(math.isfinite(float(x)) for x in d):
                row_s.append(f32(np.nan)); row_q += [0] * len(d)
                continue
            s = max(abs(x) for x in d)
            with np.errstate(divide="ignore", over="ignore"):
                inv = f32(L) / f32(s)
            if not np.isfinite(inv):
                row_s.append(f32(0.0)); row_q += [0] * len(d)
                continue
            row_s.append(f32(s) / f32(L))
            for i, x in enumerate(d):
                j = b0 + i
                r = f32((_fmix32((keys[k] & 0xFFFFFFFF) ^ ((j * 0x9E3779B9) & 0xFFFFFFFF)) >> 8)) * f32(2.0 ** -24)
                u = f32(x * inv)
                fl = f32(math.floor(u))
                q = int(fl) + (1 if r < f32(u - fl) else 0)
                row_q.append(max(-L, min(L, q)))
        codes.append(row_q)
        scales.append(row_s)
    q = np.array(codes, dtype=np.int64)
    if bits == 8:
        payload = (q & 0xFF).astype(np.uint8)
    else:
        nib = q & 0xF
        if P % 2:
            nib = np.concatenate([nib, np.zeros((K, 1), dtype=np.int64)], axis=1)
        payload = (nib[:, 0::2] | (nib[:, 1::2] << 4)).astype(np.uint8)
    return torch.from_numpy(payload), torch.from_numpy(np.array(scales, dtype=np.float32))


def _deltas(K, P, seed):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    models = theta + torch.randn(K, P, generator=g) * torch.rand(K, 1, generator=g)
    return models, theta


@pytest.mark.parametrize("P", [1, 255, 256, 257, 1000, 4994])
@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_reference_matches_scalar_transcription(P, codec):
    models, theta = _deltas(2, P, seed=P)
    keys = [uplink_key("10.0.0.1:8777", 3), 0xFFFFFFFF]
    payload, scales = reference.encode_delta(models, theta, codec.bits, keys)
    want_p, want_s = _scalar_encode(models, theta, codec.bits, keys)
    assert payload.shape == (2, codec.payload_bytes(P)) and scales.shape == (2, codec.scale_count(P))
    assert torch.equal(payload, want_p)
    assert same_bits(scales, want_s)
    # CPU tensors through ops: the reference itself
    p2, s2 = ops.encode_delta(models, theta, codec, keys)
    assert torch.equal(p2, payload) and same_bits(s2, scales)


@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_edge_blocks(codec):
    P = 5 * 256 + 3                                  # odd P: the int4 pad nibble
    theta = torch.randn(P)
    d = torch.randn(2, P) * 0.1
    d[0, :256] = 0.0                                 # an all-zero block
    d[0, 256 + 17] = -5.0                            # the block's absmax element is negative
    d[0, 512 + 3] = float("inf")                     # a non-finite delta: NaN scale, all codes 0
    d[1, 768 + 9] = float("nan")
    d[1, 1024:1280] = 1e-38                          # L / s overflows: encodes as zeros
    models = theta + d
    models[0, 512 + 3] = float("inf")
    models[1, 768 + 9] = float("nan")
    keys = [11, 12]
    payload, scales = reference.encode_delta(models, theta, codec.bits, keys)
    want_p, want_s = _scalar_encode(models, theta, codec.bits, keys)
    assert torch.equal(payload, want_p) and same_bits(scales, want_s)
    q = reference.decode_codes(payload, codec.bits, P)
    assert scales[0, 0] == 0 and not q[0, :256].any()
    assert scales[0, 1] == np.float32(5.0) / np.float32(codec.levels) and q[0, 256 + 17] == -codec.levels
    assert math.isnan(scales[0, 2]) and not q[0, 512:768].any() and scales[0, 2].view(torch.int32) == 0x7FC00000
    assert math.isnan(scales[1, 3]) and not q[1, 768:1024].any()
    assert scales[1, 4] == 0 and not q[1, 1024:1280].any()
    if codec.bits == 4:
        assert int(payload[0, -1]) >> 4 == 0 and int(payload[1, -1]) >> 4 == 0   # pad nibble


@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_error_bound_and_unbiasedness(codec):
    P = 600
    models, theta = _deltas(1, P, seed=5)
    d = (models[0] - theta).numpy()
    n_keys = 4096
    keys = list(range(1000, 1000 + n_keys))
    payload, scales = reference.encode_delta(models.expand(n_keys, P), theta, codec.bits, keys)
    dec = reference.decode_delta(payload, scales, codec.bits, P).numpy()
    step = np.repeat(scales.numpy(), 256, axis=1)[:, :P]
    assert (np.abs(dec - d[None, :]) <= step).all()                       # |d^ - d| <= step, every key and element
    # unbiasedness: d^ = d + e with E[e] = 0 and Var[e] <= step^2 / 4, so the mean over n keys is within z step / (2 sqrt(n))
    # of d; z = 6 for the 600 elements (a per-element false-alarm rate far below 1e-6), plus float rounding of d / step
    bias = np.abs(dec.astype(np.float64).mean(0) - d)
    bound = 6.0 * step[0] / (2.0 * math.sqrt(n_keys)) + 1e-6 * np.abs(d)
    assert (bias <= bound).all(), float((bias / bound).max())
    # and it is not trivially so: the rounding really is random
    assert (dec.std(0) > 0).mean() > 0.9


def test_codec_object():
    assert UplinkCodec().kind == "fp32" and not UplinkCodec().quantized and UplinkCodec().payload_bytes(10) == 40
    c8, c4 = UplinkCodec("int8"), UplinkCodec("int4")
    assert (c8.bits, c8.levels, c4.bits, c4.levels, UplinkCodec.BLOCK) == (8, 127, 4, 7, 256)
    assert c8.payload_bytes(4994) == 4994 and c4.payload_bytes(4994) == 2497 and c4.payload_bytes(5) == 3
    assert c8.scale_count(4994) == 20 and c8.scale_count(256) == 1 and c8.scale_count(257) == 2
    for c in (c8, c4):                                                     # |q step| <= L max_scale stays finite
        assert np.isfinite(np.float32(c.levels) * np.float32(c.max_scale))
        with np.errstate(over="ignore"):
            assert not np.isfinite(np.float32(c.levels) * np.nextafter(np.float32(c.max_scale), np.float32(np.inf)))
    with pytest.raises(ValueError):
        UplinkCodec("int2")
    assert uplink_key("a", 1) != uplink_key("b", 1) and uplink_key("a", 1) != uplink_key("a", 2)


# ---- elementwise.cu on the SIMT CPU build ------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_quantize_delta_kernel_on_cpu_bit_exact(simt, K, codec):
    for P in (1000, 1001, 3 * 256):                      # 16-byte path with a partial block / scalar path (P % 4 != 0)
        models, theta = _deltas(K, P, seed=K * P)
        keys = [uplink_key(f"w{k}", 9) for k in range(K)]
        payload, scales = simt.quantize_delta(models, theta, keys_i32(keys), codec.bits)
        want_p, want_s = reference.encode_delta(models, theta, codec.bits, keys)
        assert payload.shape[1] % 16 == 0
        assert torch.equal(payload[:, :codec.payload_bytes(P)], want_p) and same_bits(scales, want_s)
    # rows that are not 16-byte aligned (a view one float into a buffer): the scalar path, same bits
    buf = torch.randn(K * 1000 + 1)
    models, theta = buf[1:].view(K, 1000), torch.randn(1000)
    payload, scales = simt.quantize_delta(models, theta, keys_i32([7] * K), codec.bits)
    want_p, want_s = reference.encode_delta(models, theta, codec.bits, [7] * K)
    assert torch.equal(payload[:, :codec.payload_bytes(1000)], want_p) and same_bits(scales, want_s)


def _encoded(K, P, codec, seed, poison=False):
    models, theta = _deltas(K, P, seed)
    if poison and K > 2:
        models[1] = theta + 1e4                          # a poisoned client
    payload, scales = reference.encode_delta(models, theta, codec.bits, [seed * 131 + k for k in range(K)])
    return theta, payload, scales


@pytest.mark.parametrize("K", [1, 3, 16, 33, 100])
@pytest.mark.parametrize("codec", CODECS, ids=lambda c: c.kind)
def test_fedavg_q_kernel_on_cpu(simt, K, codec):
    P = 1001 if K < 100 else 203
    theta, payload, scales = _encoded(K, P, codec, seed=K, poison=True)
    row = (payload.shape[1] + 15) // 16 * 16
    padded = torch.zeros(K, row, dtype=torch.uint8)
    padded[:, :payload.shape[1]] = payload
    w = torch.rand(K) + 0.1
    w /= w.sum()
    # weighted mean, server lr 0.7
    got = theta.clone()
    simt.fedavg_apply_quantized(got, padded, scales, w, codec.bits, 0.7)
    want = reference.fedavg_apply_quantized(theta.clone(), payload, scales, w, codec.bits, 0.7)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)
    # robust kinds: bit for bit
    for agg in ROBUST:
        got = theta.clone()
        simt.fedavg_apply_quantized(got, padded, scales, w, codec.bits, 1.0, 0, [], None, None, agg.code, agg.trim)
        want = reference.fedavg_apply_quantized(theta.clone(), payload, scales, None, codec.bits, 1.0, aggregator=agg)
        assert same_bits(got, want), agg


@pytest.mark.parametrize("agg", [None, Aggregator("trimmed_mean", 0.2)], ids=["mean", "trimmed_mean"])
def test_fedavg_q_kernel_with_adam_on_cpu(simt, agg):
    codec, K, P = UplinkCodec("int8"), 7, 1001
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(P), opt.init_state(P)
    theta = torch.randn(P)
    ref_theta = theta.clone()
    w = torch.full((K,), 1.0 / K)
    extra = [agg.code, agg.trim] if agg is not None else []
    for i in range(3):
        models = theta + 0.5 * torch.randn(K, P)
        payload, scales = reference.encode_delta(models, theta, codec.bits, list(range(i * K, i * K + K)))
        padded = torch.zeros(K, (P + 15) // 16 * 16, dtype=torch.uint8)
        padded[:, :P] = payload
        simt.fedavg_apply_quantized(theta, padded, scales, w, codec.bits, opt.lr, opt.code, opt.hyper, st.m, st.v, *extra)
        reference.fedavg_apply_quantized(ref_theta, payload, scales, w, codec.bits, opt=ref, aggregator=agg)
        torch.testing.assert_close(theta, ref_theta, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.m, ref.m, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.v, ref.v, rtol=1e-5, atol=1e-7)


def test_ops_on_cpu_is_the_reference():
    codec = UplinkCodec("int4")
    theta, payload, scales = _encoded(5, 700, codec, seed=3)
    w = torch.full((5,), 0.2)
    got = ops.fedavg_apply_quantized(theta.clone(), payload, scales, w, codec, 0.5)
    assert torch.equal(got, reference.fedavg_apply_quantized(theta.clone(), payload, scales, w, 4, 0.5))
    dec = reference.decode_delta(payload, scales, 4, 700)
    assert torch.equal(got, theta.clone().add_(0.5 * ((theta + reference.fedavg_flat(dec, w)) - theta)))
    with pytest.raises(ValueError):
        ops.fedavg_apply_quantized(theta.clone(), payload, scales, w, UplinkCodec("fp32"))
    with pytest.raises(ValueError):
        ops.fedavg_apply_quantized(theta.clone(), payload, scales, w, codec, 0.5, opt=ServerOpt("adam").init_state(700))


# ---- remote mode over TCP ---------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _make(tmp_path, args, rounds, remote=True):
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


def _remote_run(tmp_path, uplink, rounds=3, stub=None):
    from colearn_federated_learning_b200.control.arguments import Arguments
    args = Arguments(model="mlp", lr=0.1, batch_size=16, federate_after_n_batches=30, uplink=uplink, synthetic=64)
    torch.manual_seed(0)
    workers = [_worker(1), _worker(2)] + ([_worker(3, stub)] if stub is not None else [])
    try:
        c, pub, clock = _make(tmp_path / uplink, args, rounds)
        for _, port in workers:
            pub.publish("topic/state", f"(127.0.0.1, {port}, TRAINING)")
        c.drain()
        clock.advance(1.0)
        return c, c.windower.last_result, [w for w, _ in workers]
    finally:
        for w, _ in workers:
            w.stop()


def test_remote_rounds_with_quantized_uplink_train_and_save_traffic(tmp_path):
    fp32, res32, _ = _remote_run(tmp_path, "fp32")
    assert "error" not in (fp32.windower.history[-1] if fp32.windower.history else {})
    in32 = [r["bytes_in"] for r in fp32.metrics.records if "bytes_in" in r]
    assert res32["uplink"] == "fp32" and len(in32) == 3
    for kind, ratio in (("int8", 3.5), ("int4", 6.0)):
        c, res, workers = _remote_run(tmp_path, kind)
        assert res["uplink"] == kind and res["dropped"] == [] and all(w.fits_served == 3 for w in workers)
        losses = [np.mean(l) for l in c.metrics.per_round if l]
        assert len(losses) == 3 and losses[2] < losses[0], losses            # the loss falls over 3 rounds
        bytes_in = [r["bytes_in"] for r in c.metrics.records if "bytes_in" in r]
        assert all(a / b >= ratio for a, b in zip(in32, bytes_in)), (kind, in32, bytes_in)
        # the downlink stays fp32: the same bytes towards the devices as the fp32 run, up to the "uplink" request field
        out32 = [r["bytes_out"] for r in fp32.metrics.records if "bytes_out" in r]
        assert all(0 < b - a < 64 for a, b in zip(out32, [r["bytes_out"] for r in c.metrics.records if "bytes_out" in r]))


def _tampering_worker(mutate):
    from colearn_federated_learning_b200.control.workers import WorkerServer

    class Tampering(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            if req.get("op") == "fit" and resp.get("ok"):
                mutate(resp)
            return resp
    return Tampering


def _scales_with(value):
    def mutate(resp):
        s = np.frombuffer(resp["scales"], dtype="<f4").copy()
        s[1] = value
        resp["scales"] = s.tobytes()
    return mutate


@pytest.mark.parametrize("case", ["short_payload", "nan_scale", "oversize_scale", "wrong_codec", "missing_scales"])
def test_a_bad_quantized_reply_drops_the_device(tmp_path, case):
    mutate = {"short_payload": lambda r: r.update(payload=r["payload"][:-1]),
              "nan_scale": _scales_with(np.nan),
              "oversize_scale": _scales_with(np.float32(np.finfo(np.float32).max) / np.float32(100.0)),
              "wrong_codec": lambda r: r.update(uplink="int4"),
              "missing_scales": lambda r: r.pop("scales")}[case]
    c, res, workers = _remote_run(tmp_path, "int8", rounds=2, stub=_tampering_worker(mutate))
    bad = f"127.0.0.1:{workers[2].port}"
    assert res["dropped"] == [bad] and len(res["losses"]) == 2 and bad not in res["losses"]
    assert os.path.exists(c.path) and res["rounds"] == 2


def test_check_quantized_reply_limits():
    from colearn_federated_learning_b200.control.coordinator import check_quantized_reply
    codec, P = UplinkCodec("int4"), 600
    _, payload, scales = _encoded(1, P, codec, seed=2)
    good = {"uplink": "int4", "payload": payload.numpy().tobytes(), "scales": scales.numpy().astype("<f4").tobytes()}
    p, s = check_quantized_reply(good, codec, P)
    assert torch.equal(p, payload[0]) and torch.equal(s, scales[0])
    edge = dict(good, scales=np.full(3, codec.max_scale, dtype="<f4").tobytes())       # the largest legal scale
    check_quantized_reply(edge, codec, P)
    for bad in (dict(good, scales=np.full(3, np.nextafter(np.float32(codec.max_scale), np.float32(np.inf)), dtype="<f4").tobytes()),
                dict(good, scales=np.full(3, -np.inf, dtype="<f4").tobytes()), dict(good, payload=good["payload"] + b"\0"),
                dict(good, scales=good["scales"][:-4]), dict(good, payload=None), dict(good, uplink=None)):
        with pytest.raises(ValueError):
            check_quantized_reply(bad, codec, P)


# ---- local mode and the CLI -------------------------------------------------------------------------------------------------
def test_local_mode_with_int8_uplink(tmp_path):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.coordinator import train_virtual_workers
    from colearn_federated_learning_b200.data import BaseDataset, federate, synthetic_unsw
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    args = Arguments(synthetic=90, lr=0.05, uplink="int8")
    c, pub, clock = _make(tmp_path, args, rounds=2, remote=False)
    torch.manual_seed(0)
    init = FFNN()
    save_model(init, c.path)
    ips = ["10.0.0.1", "10.0.0.2", "10.0.0.3"]
    for ip in ips:
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert c.windower.last_result["uplink"] == "int8"
    cpu = torch.device("cpu")
    x, y = synthetic_unsw(90, seed=args.seed)
    fed = federate(BaseDataset(x, y), ips, cpu)
    cfg = c._fit_config("local")
    theta = flatten_params(init).clone()
    for r in range(2):
        flats, _, _ = train_virtual_workers(theta, FFNN(), fed, cfg, r)
        payload, scales = reference.encode_delta(flats, theta, 8, [uplink_key(ip, cfg.seed + r) for ip in ips])
        reference.fedavg_apply_quantized(theta, payload, scales, torch.full((3,), 1.0 / 3), 8)
    m = FFNN()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    assert torch.equal(flatten_params(m), theta)
    settings.training_devices.clear()


def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_cli_uplink_codec_flag():
    assert _cli().uplink == "fp32" and not _cli().uplink_codec().quantized
    assert _cli("--uplink-codec", "int8").uplink_codec().bits == 8
    assert _cli("--uplink-codec", "int4", "-r").uplink == "int4"
    assert _cli("--uplink-codec", "fp32", "--box").uplink == "fp32"
    for bad in (["--uplink-codec", "int2"], ["--uplink-codec", "int8", "--box"], ["--uplink-codec", "int4", "-e"]):
        with pytest.raises(SystemExit):
            _cli(*bad)
