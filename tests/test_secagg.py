"""Secure aggregation (fl/secagg.py, ops/csrc/secagg.cuh) without a GPU: the primitives against public test vectors
(ChaCha20: RFC 8439 §2.3.2 / §2.4.2; HKDF: RFC 5869 test case 1; the ffdhe2048 key agreement), the numpy reference against an
independent scalar transcription, mask cancellation with and without dropped devices, the decode's accuracy, both kernels on
the SIMT CPU build bit for bit, remote mode over TCP (training, a replayed oracle, dropped devices, an abandoned round,
tampered replies, the device's refusals, the traffic) and the CLI."""
import os
import socket
import struct

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl import secagg as sa
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.ops import reference

M32 = 0xFFFFFFFF


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


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    return [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n)]


# ---- primitives against public test vectors -----------------------------------------------------------------------------------
def test_chacha20_block_rfc8439_2_3_2():
    block = reference.chacha20_blocks(bytes(range(32)), 1, 1, bytes.fromhex("000000090000004a00000000"))[0]
    want = bytes.fromhex("10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
                         "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")
    assert block.astype("<u4").tobytes() == want


def test_chacha20_keystream_rfc8439_2_4_2():
    plain = (b"Ladies and Gentlemen of the class of '99: If I could offer you only one tip for the future, sunscreen would be it.")
    want = bytes.fromhex("6e2e359a2568f98041ba0728dd0d6981e97e7aec1d4360c20a27afccfd9fae0b"
                         "f91b65c5524733ab8f593dabcd62b3571639d624e65152ab8f530c359f0861d8"
                         "07ca0dbf500d6a6156a38e088a22b65e52bc514d16ccf806818ce91ab7793736"
                         "5af90bbf74a35be6b40b8eedf2785e42874d")
    stream = reference.chacha20_blocks(bytes(range(32)), 1, 2, bytes.fromhex("000000000000004a00000000")).astype("<u4").tobytes()
    assert bytes(a ^ b for a, b in zip(plain, stream)) == want


def test_hkdf_rfc5869_test_case_1():
    okm = sa.hkdf_sha256(bytes([0x0B] * 22), bytes(range(0xF0, 0xFA)), 42, salt=bytes(range(13)))
    assert okm.hex() == "3cb25f25faacd57a90434f64d0362f2a2d2d0a90cf1a5a4c5db02d56ecc4c5bf34007208d5b887185865"


def test_dh_both_ends_derive_the_same_seed_and_bad_keys_are_refused():
    a, b = sa.KeyPair.generate(), sa.KeyPair.generate()
    s_ab = sa.pair_seed(a.sk, b.pk, "tag", "u", "v")
    assert s_ab == sa.pair_seed(b.sk, a.pk, "tag", "u", "v") and len(s_ab) == 32
    assert s_ab != sa.pair_seed(a.sk, b.pk, "other", "u", "v")            # bound to the training's tag
    assert sa.round_seed(s_ab, 0) != sa.round_seed(s_ab, 1)
    assert pow(sa.P - 2, sa.Q, sa.P) != 1                                 # -2 is outside the prime-order subgroup
    for bad in (0, 1, sa.P - 1, sa.P, sa.P - 2):
        with pytest.raises(ValueError):
            sa.check_public_key(bad)
        with pytest.raises(ValueError):
            sa.pair_seed(a.sk, bad, "tag", "u", "v")
    with pytest.raises(ValueError):
        sa.pk_from_bytes(sa.pk_to_bytes(a.pk)[1:])


def test_frac_bits_keeps_every_honest_sum_inside_int32():
    for clip, n in ((1.0, 2), (1.0, 100), (0.01, 7), (1000.0, 3), (3.3, 1)):
        f = sa.frac_bits(clip, n)
        assert n * sa.code_bound(clip, f) <= 2 ** 31 - 1 and (f == 64 or n * sa.code_bound(clip, f + 1) > 2 ** 31 - 1)
    assert sa.frac_bits(1.0, 100) == 24
    for bad in (0.0, -1.0, float("inf"), float("nan"), 1e39):
        with pytest.raises(ValueError):
            sa.frac_bits(bad, 3)
    with pytest.raises(ValueError):
        sa.frac_bits(2.0 ** 30, 4)                                         # no fraction bit leaves room for 4 devices


# ---- the reference against a scalar transcription ---------------------------------------------------------------------------------
def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & M32


def _scalar_block(key, counter):
    k = list(struct.unpack("<8I", key))
    x = [0x61707865, 0x3320646E, 0x79622D32, 0x6B206574] + k + [counter, 0, 0, 0]
    s = list(x)

    def qr(a, b, c, d):
        s[a] = (s[a] + s[b]) & M32; s[d] = _rotl(s[d] ^ s[a], 16)   # noqa: E702
        s[c] = (s[c] + s[d]) & M32; s[b] = _rotl(s[b] ^ s[c], 12)   # noqa: E702
        s[a] = (s[a] + s[b]) & M32; s[d] = _rotl(s[d] ^ s[a], 8)    # noqa: E702
        s[c] = (s[c] + s[d]) & M32; s[b] = _rotl(s[b] ^ s[c], 7)    # noqa: E702
    for _ in range(10):
        for q in ((0, 4, 8, 12), (1, 5, 9, 13), (2, 6, 10, 14), (3, 7, 11, 15), (0, 5, 10, 15), (1, 6, 11, 12), (2, 7, 8, 13), (3, 4, 9, 14)):
            qr(*q)
    return [(s[i] + x[i]) & M32 for i in range(16)]


def _scalar_mask(model, theta, keys, signs, clip, f):
    c32 = np.float32(clip)
    out, clipped, nonfinite = [], 0, 0
    blocks = {}
    for e in range(len(model)):
        d = np.float32(model[e]) - np.float32(theta[e])
        if np.isnan(d):
            q = 0
            nonfinite += 1
        else:
            if np.isinf(d):
                nonfinite += 1
            elif abs(d) > c32:
                clipped += 1
            c = min(max(d, -c32), c32)
            q = int(np.rint(np.float32(c) * np.float32(2.0 ** f))) & M32
        for key, sign in zip(keys, signs):
            if (key, e // 16) not in blocks:
                blocks[(key, e // 16)] = _scalar_block(key, e // 16)
            w = blocks[(key, e // 16)][e % 16]
            q = (q + (w if sign > 0 else -w)) & M32
        out.append(q)
    return np.array(out, dtype=np.uint32), clipped, nonfinite


def _edge_pair(P, clip, f, seed):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    model = theta + clip * 2 * torch.rand(P, generator=g) - clip
    t = theta.numpy()
    edges = [float("nan"), float("inf"), float("-inf"), 0.0, -0.0, clip, -clip, clip * 1.5, -clip * 3, 0.5 * 2.0 ** -f, 1.5 * 2.0 ** -f,
             -2.5 * 2.0 ** -f, float(np.nextafter(np.float32(clip), np.float32(0)))]
    m = model.numpy()
    for i, v in enumerate(edges[:P]):
        j = (i * 7) % P
        t[j] = 0.0 if v in (0.0,) or abs(v) < 1 else t[j]
        m[j] = t[j] + np.float32(v) if np.isfinite(v) and t[j] != 0 else np.float32(v)
    return torch.from_numpy(m.copy()), torch.from_numpy(t.copy())


@pytest.mark.parametrize("P", [1, 15, 16, 17, 2401, 4994])
def test_reference_matches_scalar_transcription(P):
    clip, f = 0.25, 20
    model, theta = _edge_pair(P, clip, f, P)
    keys, signs = _keys(3, P), [1, -1, -1]
    y, clipped, nonfinite = reference.secagg_mask(model, theta, keys, signs, clip, f)
    want, wc, wn = _scalar_mask(model.numpy(), theta.numpy(), keys, signs, clip, f)
    assert y.dtype == torch.uint32 and np.array_equal(y.numpy(), want) and (clipped, nonfinite) == (wc, wn)
    q, _, _ = reference.secagg_encode((model - theta).numpy(), clip, f)
    z = q.view(np.int32).astype(np.int64)
    assert np.abs(z).max() <= sa.code_bound(clip, f)
    # decode of one device's codes: exact scaling of the nearest-even integer
    mean = reference.secagg_decode(q, f, 1)
    assert np.array_equal(mean, (z.astype(np.float32) * np.float32(2.0 ** -f)).astype(np.float32))


# ---- a simulated round ----------------------------------------------------------------------------------------------------------
def _round(K, P, clip=1.0, seed=0, scale=0.05):
    """K devices through setup and one round: (order, devices, deltas, masked rows, encodings, f)"""
    devices = [sa.SecAggDevice() for _ in range(K)]
    ids = [f"10.0.0.{i}:8777" for i in range(K)]
    pks = [d.setup("T") for d in devices]
    for d, me in zip(devices, ids):
        assert d.learn_peers("T", ids, pks) == me
    f = sa.frac_bits(clip, K)
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    deltas = scale * torch.randn(K, P, generator=g)
    rows, encs = [], []
    for i, d in enumerate(devices):
        keys, signs = d.begin_round("T", 0, ids, clip, f)
        y, _, _ = reference.secagg_mask(theta + deltas[i], theta, keys, signs, clip, f)
        rows.append(y.numpy())
        encs.append(reference.secagg_encode(((theta + deltas[i]) - theta).numpy(), clip, f)[0])
    return ids, devices, theta, deltas, np.stack(rows), np.stack(encs), f


def test_masks_cancel_without_dropped_devices():
    ids, devices, theta, deltas, rows, encs, f = _round(5, 2401)
    for i in range(5):
        assert (rows[i] != encs[i]).mean() > 0.99                          # one row alone shows nothing
    # the unmask of a round with D empty reveals only the self seeds; the pair masks cancel in the sum by themselves
    seeds = {u: sa.check_unmask_reply(d.unmask("T", 0, ids), []) for u, d in zip(ids, devices)}
    keys, signs = sa.correction_streams(ids, ids, [], seeds)
    assert len(keys) == 5 and signs == [-1] * 5
    z = reference.secagg_unmask_sum(torch.from_numpy(rows.view(np.int32)), keys, signs)
    assert np.array_equal(z, encs.sum(axis=0, dtype=np.uint32))
    self_masks = reference.secagg_streams(keys, [1] * 5, 2401)
    assert np.array_equal(rows.sum(axis=0, dtype=np.uint32), encs.sum(axis=0, dtype=np.uint32) + self_masks)


@pytest.mark.parametrize("ndrop", [1, 2, 3, 4])
def test_masks_cancel_with_dropped_devices(ndrop):
    K, P = 6, 999
    ids, devices, theta, deltas, rows, encs, f = _round(K, P, seed=ndrop)
    dropped = ids[1:1 + ndrop]
    survivors = [u for u in ids if u not in dropped]
    seeds = {u: sa.check_unmask_reply(devices[ids.index(u)].unmask("T", 0, survivors), dropped) for u in survivors}
    keys, signs = sa.correction_streams(ids, survivors, dropped, seeds)
    assert len(keys) == len(survivors) * (1 + ndrop)
    live = [ids.index(u) for u in survivors]
    z = reference.secagg_unmask_sum(torch.from_numpy(rows[live].view(np.int32)), keys, signs)
    assert np.array_equal(z, encs[live].sum(axis=0, dtype=np.uint32))
    # accuracy: nothing clips at this scale; the decoded mean is within 2^-f + 2 ulp of the fp32 mean of the survivors' deltas
    mean = reference.secagg_decode(z, f, len(survivors))
    want = ((theta + deltas[live]) - theta).double().mean(0).float().numpy()   # the deltas the devices formed
    assert (np.abs(mean - want) <= 2.0 ** -f + 2 * np.spacing(np.abs(want).astype(np.float32))).all()


# ---- the device's state machine ----------------------------------------------------------------------------------------------------
def test_device_refusals():
    ids, devices, theta, deltas, rows, encs, f = _round(4, 64)
    d = devices[0]
    with pytest.raises(ValueError):
        d.unmask("T", 0, ids[:1])                                          # |U2| < 2
    with pytest.raises(ValueError):
        d.unmask("T", 0, ids[1:])                                          # lists it as dropped
    with pytest.raises(ValueError):
        d.unmask("T", 0, ids + ["stranger"])                               # not a participant of the round
    out = d.unmask("T", 0, ids[:3])
    assert list(out["pair_seeds"]) == [ids[3]]
    with pytest.raises(ValueError):
        d.unmask("T", 0, ids[:3])                                          # a second unmask of the round
    with pytest.raises(ValueError):
        d.begin_round("T", 1, ids, 1.0, f)                                 # the revealed peer reappears
    with pytest.raises(ValueError):
        d.begin_round("T", 0, ids[:3], 1.0, f)                             # not after the last round
    with pytest.raises(ValueError):
        d.begin_round("T", 1, ids[:3] + ["stranger"], 1.0, f)              # unknown participant
    with pytest.raises(ValueError):
        d.begin_round("T", 1, ids[:3], 1.0, f + 2)                         # f breaks the bound for 3 participants
    keys, signs = d.begin_round("T", 1, ids[:3], 1.0, f)
    assert len(keys) == 3 and signs == [1, 1, 1]
    with pytest.raises(ValueError):
        d.unmask("T", 0, ids[:3])                                          # an earlier round can no longer be unmasked
    with pytest.raises(ValueError):
        devices[1].learn_peers("T", ids, [devices[1].setup("U")] * 4)     # its key listed more than once


def test_reply_checks():
    good = {"secagg": "masked", "masked": bytes(40), "clipped": 0, "nonfinite": 10}
    y, c, n = sa.check_masked_reply(good, 10)
    assert y.dtype == np.uint32 and y.size == 10 and (c, n) == (0, 10)
    for bad in ({"masked": bytes(39)}, {"masked": bytes(44)}, {"clipped": 11}, {"nonfinite": -1}, {"clipped": 1.0}, {"secagg": None},
                {"masked": None}):
        with pytest.raises(ValueError):
            sa.check_masked_reply({**good, **bad}, 10)
    seeds = {"self_seed": bytes(32), "pair_seeds": {"a": bytes(32), "b": bytes(32)}}
    assert sa.check_unmask_reply(seeds, ["b", "a"])[1] == {"a": bytes(32), "b": bytes(32)}
    for bad in ({"self_seed": bytes(31)}, {"pair_seeds": {"a": bytes(32)}}, {"pair_seeds": {"a": bytes(32), "c": bytes(32)}},
                {"pair_seeds": {"a": bytes(32), "b": bytes(33)}}, {"pair_seeds": [bytes(32)] * 2}):
        with pytest.raises(ValueError):
            sa.check_unmask_reply({**seeds, **bad}, ["a", "b"])


def test_ops_refuse_what_they_cannot_do():
    from colearn_federated_learning_b200.fl.aggregate import Aggregator
    theta = torch.zeros(20)
    with pytest.raises(ValueError):
        ops.fedavg_apply_secagg(theta, torch.zeros(2, 20, dtype=torch.int32), _keys(2, 0), [-1, -1], 20, 2, aggregator=Aggregator("median"))
    with pytest.raises(ValueError):
        ops.secagg_mask(theta, theta, _keys(1, 0), [1], float("inf"), 20)
    with pytest.raises(ValueError):
        ops.secagg_mask(theta, theta, _keys(2, 0), [1], 1.0, 20)         # one sign per key
    with pytest.raises(ValueError):
        reference.secagg_streams([bytes(31)], [1], 20)


# ---- the kernels on the SIMT CPU build --------------------------------------------------------------------------------------------
def _same(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("S", [0, 1, 3, 17])
def test_mask_kernel_on_cpu_bit_exact(simt, S):
    for P in (1, 17, 4994, 1000):
        model, theta = _edge_pair(P, 0.5, 21, S + P)
        keys, signs = _keys(S, S), [1 if i % 2 else -1 for i in range(S)]
        y, clipped, nonfinite = reference.secagg_mask(model, theta, keys, signs, 0.5, 21)
        got, counts = simt.secagg_mask(model, theta, ops.secagg_key_words(keys).reshape(-1, 8), torch.tensor(signs, dtype=torch.int32),
                                       0.5, 21)
        assert _same(got, y) and counts.tolist() == [clipped, nonfinite], (P, S)


@pytest.mark.parametrize("K", [1, 2, 3, 5, 8, 13, 20])
def test_apply_kernel_on_cpu_bit_exact(simt, K):
    P = 4994
    g = torch.Generator().manual_seed(K)
    theta = torch.randn(P, generator=g)
    masked = torch.randint(-2 ** 31, 2 ** 31, (K, P), generator=g, dtype=torch.int64).to(torch.int32)
    for ndrop in (0, 1, 3):
        S = K * (1 + ndrop)                                               # self streams plus pair streams of the dropped devices
        keys, signs = _keys(S, K * 10 + ndrop), [1 if i % 3 else -1 for i in range(S)]
        kw, sg = ops.secagg_key_words(keys), torch.tensor(signs, dtype=torch.int32)
        want = reference.fedavg_apply_secagg(theta.clone(), masked, keys, signs, 23, K + ndrop, 0.7)
        got = theta.clone()
        simt.fedavg_apply_secagg(got, masked, kw, sg, 23, K + ndrop, 0.7)
        assert _same(got, want), (K, ndrop)
        # FedAdam on the same masked sum
        opt = ServerOpt("adam", lr=0.05)
        st, ref = opt.init_state(P), opt.init_state(P)
        want = reference.fedavg_apply_secagg(theta.clone(), masked, keys, signs, 23, K + ndrop, opt=ref)
        got = theta.clone()
        simt.fedavg_apply_secagg(got, masked, kw, sg, 23, K + ndrop, float(opt.lr), opt.code, opt.hyper, st.m, st.v)
        assert _same(got, want) and _same(st.m, ref.m) and _same(st.v, ref.v), (K, ndrop)


def test_apply_kernel_split_path_on_cpu(simt):
    # few columns and many streams: the streams kernel adds chunks into the scratch row with atomics, then the finalize
    P, K, S = 2401, 4, 600
    g = torch.Generator().manual_seed(5)
    theta = torch.randn(P, generator=g)
    masked = torch.randint(-2 ** 31, 2 ** 31, (K, P), generator=g, dtype=torch.int64).to(torch.int32)
    keys, signs = _keys(S, 99), [1 if i % 2 else -1 for i in range(S)]
    want = reference.fedavg_apply_secagg(theta.clone(), masked, keys, signs, 22, K)
    got = theta.clone()
    simt.fedavg_apply_secagg(got, masked, ops.secagg_key_words(keys), torch.tensor(signs, dtype=torch.int32), 22, K, 1.0)
    assert _same(got, want)


# ---- remote mode over TCP ------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(seed, cls=None):
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw
    port = _free_port()
    w = (cls or WorkerServer)(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
    w.add_dataset(BaseDataset(*synthetic_unsw(256, seed=seed)))
    w.start(block=False)
    return w


def _args(model="ffnn", **kw):
    from colearn_federated_learning_b200.control.arguments import Arguments
    base = dict(model=model, lr=0.1, batch_size=16, federate_after_n_batches=30, synthetic=64, secure_agg=True, secagg_clip=0.5)
    return Arguments(**{**base, **kw})


def _train(tmp_path, args, workers, rounds):
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.models import build_model, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model
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

    os.makedirs(tmp_path, exist_ok=True)
    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, True, rounds, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "test.pth"),
                    device=torch.device("cpu"), metrics=Losses(), evaluate_after=False)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    torch.manual_seed(0)
    init = build_model(args.model)
    save_model(init, c.path)
    theta0 = flatten_params(init).detach().clone()
    for w in workers:
        pub.publish("topic/state", f"(127.0.0.1, {w.port}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    m = build_model(args.model)
    m.load_state_dict(torch.load(c.path, weights_only=True))
    settings.training_devices.clear()
    return c, c.windower.last_result, theta0, flatten_params(m).detach()


class _Recorder:
    """records every device's (trained, received) pair as ops.secagg_mask sees it, in call order"""

    def __init__(self, monkeypatch):
        self.calls = []
        real = ops.secagg_mask

        def wrapped(model, theta, keys, signs, clip, f):
            self.calls.append((model.detach().clone(), theta.detach().clone(), clip, f))
            return real(model, theta, keys, signs, clip, f)
        monkeypatch.setattr(ops, "secagg_mask", wrapped)


def _oracle(theta0, rounds):
    """replays the rounds from the devices' deltas: sum of the codes, decode, theta += 1 (a - theta)"""
    t = theta0.numpy().astype(np.float32)
    for calls in rounds:
        if not calls:
            continue
        f, clip = calls[0][3], calls[0][2]
        z = np.zeros(t.size, dtype=np.uint32)
        for model, received, _, _ in calls:
            z += reference.secagg_encode((model - received).numpy(), clip, f)[0]
        mean = reference.secagg_decode(z, f, len(calls))
        t = reference._server_opt_np(t, t + mean, None, 1.0)
    return torch.from_numpy(t)


def _stop(workers):
    for w in workers:
        w.stop()


def test_remote_training_matches_a_replayed_oracle(tmp_path, monkeypatch):
    rec = _Recorder(monkeypatch)
    workers = [_worker(s) for s in (1, 2, 3)]
    try:
        c, res, theta0, final = _train(tmp_path, _args("mlp", secagg_clip=1.0), workers, 3)
    finally:
        _stop(workers)
    recs = [r for r in c.metrics.records if "secagg_u2" in r]
    assert res["dropped"] == [] and len(recs) == 3 and all(w.fits_served == 3 for w in workers)
    assert all(r["secagg_u2"] == 3 and r["secagg_dropped"] == 0 and not r["secagg_abandoned"] for r in recs)
    losses = [np.mean(x) for x in c.metrics.per_round if x]
    assert losses[2] < losses[0], losses
    assert len(rec.calls) == 9 and rec.calls[0][3] == res["secagg_frac_bits"] == sa.frac_bits(1.0, 3)
    want = _oracle(theta0, [rec.calls[0:3], rec.calls[3:6], rec.calls[6:9]])
    assert torch.equal(final.view(torch.int32), want.view(torch.int32))


def test_a_device_that_drops_after_setup_leaves_and_the_round_aggregates(tmp_path, monkeypatch):
    from colearn_federated_learning_b200.control.workers import WorkerServer

    class Gone(WorkerServer):
        def _dispatch(self, req):
            if req.get("op") == "fit":
                return {"ok": False, "error": "gone"}
            return super()._dispatch(req)

    rec = _Recorder(monkeypatch)
    workers = [_worker(1), _worker(2), _worker(3, Gone), _worker(4)]
    try:
        c, res, theta0, final = _train(tmp_path, _args(), workers, 2)
    finally:
        _stop(workers)
    gone = f"127.0.0.1:{workers[2].port}"
    recs = [r for r in c.metrics.records if "secagg_u2" in r]
    assert res["dropped"] == [gone] and res["secagg_frac_bits"] == sa.frac_bits(0.5, 4)
    assert [(r["secagg_u2"], r["secagg_dropped"], r["secagg_abandoned"]) for r in recs] == [(3, 1, False), (3, 0, False)]
    # the survivors of round 0 revealed their pair seeds with the dropped device: round 1's participants exclude it
    assert all(gone in w._secagg._t[next(iter(w._secagg._t))].revealed for w in workers if w is not workers[2])
    want = _oracle(theta0, [rec.calls[0:3], rec.calls[3:6]])
    assert torch.equal(final.view(torch.int32), want.view(torch.int32))


def test_a_device_that_fails_the_unmask_abandons_the_round(tmp_path):
    from colearn_federated_learning_b200.control.workers import WorkerServer

    class Mute(WorkerServer):
        def _dispatch(self, req):
            if req.get("op") == "secagg_unmask":
                return {"ok": False, "error": "no"}
            return super()._dispatch(req)

    workers = [_worker(1), _worker(2, Mute), _worker(3)]
    try:
        c, res, theta0, final = _train(tmp_path, _args(), workers, 1)
    finally:
        _stop(workers)
    rec = [r for r in c.metrics.records if "secagg_u2" in r][0]
    assert rec["secagg_abandoned"] and rec["secagg_u2"] == 3 and res["dropped"] == [f"127.0.0.1:{workers[1].port}"]
    assert torch.equal(final, theta0)                                       # theta unchanged


@pytest.mark.parametrize("case", ["short_masked", "huge_count", "wrong_seed_count", "seed_for_pair_not_asked"])
def test_tampered_replies_are_dropped(tmp_path, case):
    from colearn_federated_learning_b200.control.workers import WorkerServer

    class Tamper(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            op = req.get("op")
            if op == "fit" and case == "short_masked":
                resp["masked"] = resp["masked"][:-4]
            elif op == "fit" and case == "huge_count":
                resp["clipped"] = 10 ** 6
            elif op == "secagg_unmask" and case == "wrong_seed_count":
                resp["pair_seeds"] = {}
            elif op == "secagg_unmask" and case == "seed_for_pair_not_asked":
                resp["pair_seeds"] = {**resp["pair_seeds"], "10.9.9.9:1": bytes(32)}
            return resp

    class Gone(WorkerServer):
        def _dispatch(self, req):
            return {"ok": False, "error": "gone"} if req.get("op") == "fit" else super()._dispatch(req)

    workers = [_worker(1), _worker(2), _worker(3, Tamper), _worker(4, Gone)]
    try:
        c, res, theta0, final = _train(tmp_path, _args(), workers, 1)
    finally:
        _stop(workers)
    rec = [r for r in c.metrics.records if "secagg_u2" in r][0]
    bad, gone = f"127.0.0.1:{workers[2].port}", f"127.0.0.1:{workers[3].port}"
    assert gone in res["dropped"] and bad in res["dropped"]
    if case in ("short_masked", "huge_count"):                             # its reply is refused: it counts as dropped
        assert (rec["secagg_u2"], rec["secagg_dropped"], rec["secagg_abandoned"]) == (2, 2, False) and not torch.equal(final, theta0)
    else:                                                                  # its seeds are refused: the round is abandoned
        assert rec["secagg_abandoned"] and torch.equal(final, theta0)


@pytest.fixture()
def one_device():
    """a worker, a client to it and two in-process peers, through the setup of training "T" """
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    from colearn_federated_learning_b200.fl.uplink import UplinkCodec
    from colearn_federated_learning_b200.models import FFNN, flatten_params

    w = _worker(1)
    client = RemoteWorkerClient(w.id, "127.0.0.1", w.port)
    peers = [sa.SecAggDevice(), sa.SecAggDevice()]
    ids = ["dev", "p1", "p2"]
    pks = [client.secagg_setup("T")] + [p.setup("T") for p in peers]
    client.secagg_peers("T", ids, pks)
    for p in peers:
        p.learn_peers("T", ids, pks)
    torch.manual_seed(0)
    theta = flatten_params(FFNN()).detach().clone()
    cfg = FitConfig(model="ffnn", loss="bce", batch_size=16, epochs=1, max_nr_batches=5, lr=0.1, shuffle=True, seed=1)
    f = sa.frac_bits(0.5, 3)

    def fit(t, u1, frac=f):
        return client.fit_update(theta, cfg, UplinkCodec(), secagg={"tag": "T", "t": t, "u1": u1, "clip": 0.5, "frac_bits": frac})
    yield client, ids, fit, w
    client.close()
    w.stop()


def test_the_device_refuses_over_the_wire(one_device):
    client, ids, fit, w = one_device
    with pytest.raises(RuntimeError):
        fit(0, ids, frac=sa.frac_bits(0.5, 3) + 1)                        # f breaks the bound
    update, _, _ = fit(0, ids)
    assert sa.check_masked_reply(update, 2401)[0].size == 2401
    with pytest.raises(RuntimeError):
        client.secagg_unmask("T", 0, ["p1", "p2"])                         # lists it as dropped
    with pytest.raises(RuntimeError):
        client.secagg_unmask("T", 0, ["dev"])                              # |U2| < 2
    seeds = client.secagg_unmask("T", 0, ["dev", "p1"])
    assert sa.check_unmask_reply(seeds, ["p2"])[0]
    with pytest.raises(RuntimeError):
        client.secagg_unmask("T", 0, ["dev", "p1"])                        # a second unmask for the same round
    with pytest.raises(RuntimeError):
        fit(1, ids)                                                        # the revealed peer reappears
    with pytest.raises(RuntimeError):
        client._call({"op": "fit", "config": {}, "params": b"", "uplink": "int8", "secagg": {"tag": "T"}})
    assert w.fits_served == 1
    assert fit(1, ["dev", "p1"])[0]["secagg"] == "masked"


def test_traffic_is_pinned(tmp_path):
    workers = [_worker(s) for s in (1, 2, 3)]
    try:
        c, res, _, _ = _train(tmp_path, _args(), workers, 2)
    finally:
        _stop(workers)
    P, K = 2401, 3
    recs = [r for r in c.metrics.records if "secagg_u2" in r]
    for r in recs:
        per_device = r["bytes_in"] / K
        # the masked row (4 P bytes, as fp32) and the unmask reply (one 32-byte self seed) plus msgpack framing
        assert 4 * P + 32 <= per_device <= 4 * P + 32 + 200, r
    # setup: one 256-byte key back per device; out: the setup request and the key list (3 keys) per device
    assert 256 * K <= res["secagg_setup_bytes_in"] <= (256 + 60) * K
    assert 256 * K * K <= res["secagg_setup_bytes_out"] <= (256 + 60) * K * K + 150 * K


def test_secure_aggregation_composes_with_a_topk_downlink(tmp_path):
    workers = [_worker(s) for s in (1, 2, 3)]
    try:
        c, res, _, _ = _train(tmp_path, _args(downlink="topk", downlink_topk=8), workers, 3)
    finally:
        _stop(workers)
    recs = [r for r in c.metrics.records if "secagg_u2" in r]
    assert res["dropped"] == [] and res["downlink"] == "topk" and all(w.fits_served == 3 for w in workers)
    assert all(not r["secagg_abandoned"] for r in recs)
    held = [w._replicas["ffnn"] for w in workers]
    assert held[0][0] == held[1][0] == held[2][0] and torch.equal(held[0][1], held[2][1])
    assert recs[2]["bytes_out"] < recs[0]["bytes_out"] / 5                  # later rounds send the replica's wire, not the model


def test_without_the_flag_requests_and_replies_are_unchanged(tmp_path):
    from colearn_federated_learning_b200.control.workers import WorkerServer
    seen = []

    class Recording(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            seen.append((req.get("op"), list(req), list(resp)))
            return resp

    workers = [_worker(1, Recording), _worker(2, Recording)]
    try:
        _train(tmp_path, _args(secure_agg=False), workers, 2)
    finally:
        _stop(workers)
    fits = [(req, resp) for op, req, resp in seen if op == "fit"]
    assert len(fits) == 4 and {op for op, _, _ in seen} == {"fit", "close"}
    assert all(r == ["op", "config", "params", "dataset_key"] for r, _ in fits)
    assert all(r == ["ok", "params", "loss", "n", "path"] for _, r in fits)


# ---- the CLI --------------------------------------------------------------------------------------------------------------------------
def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_cli_secure_agg_flags():
    a = _cli()
    assert a.secure_agg is False and a.secagg_clip == 1.0
    b = _cli("-r", "--secure-agg", "--secagg-clip", "0.25", "--server-opt", "adam", "--downlink-codec", "int8")
    assert b.secure_agg and b.secagg_clip == 0.25 and b.downlink_codec().quantized
    for bad in (["--secure-agg"], ["-r", "--secure-agg", "--box"], ["-r", "--secure-agg", "-e"],
                ["-r", "--secure-agg", "--uplink-codec", "int8"], ["-r", "--secure-agg", "--aggregator", "median"],
                ["-r", "--secure-agg", "--weighted"], ["-r", "--secure-agg", "--secagg-clip", "0"],
                ["-r", "--secure-agg", "--secagg-clip", "inf"], ["-r", "--secure-agg", "--secagg-clip", "nan"],
                ["-r", "--secure-agg", "--model", "resnet18"]):
        with pytest.raises(SystemExit):
            _cli(*bad)
