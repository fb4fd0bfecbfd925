"""Top-k sparsified uplink with error feedback without a GPU: the numpy definition against an independent scalar
transcription (edge blocks included), the error-feedback invariants, the kernel sources of elementwise.cu on the SIMT CPU
build, remote mode over TCP (traffic, validation of untrusted replies, the worker's residual), local mode and the CLI.

The encode is bit-exact everywhere (the selection is integer compares on fixed keys and the values are two fixed fp32
roundings; NaN is compared as NaN because the GPU writes its canonical NaN).  The fused sparse decode + FedAvg compares with
the tolerance of the quantized apply tests (the kernel's fmaf chain against the reference's torch sum), and with the
tests/test_server_opt.py tolerance for a FedAdam composition."""
import os
import socket

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops, settings
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec
from colearn_federated_learning_b200.ops import reference

KS = [1, 8, 32]


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
    a, b = a.cpu(), b.cpu()
    nan = a.isnan()
    return bool(torch.equal(nan, b.isnan()) and torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32)))


# ---- an independent scalar transcription of uplink_topk.cuh -----------------------------------------------------------------
def _key(x):
    a = int(np.array(x, dtype=np.float32).view(np.uint32)) & 0x7FFFFFFF
    return 0x7F800001 if a > 0x7F800000 else a


def _scalar_topk(models, theta, residual, k):
    """block by block in Python lists and numpy float32 scalars"""
    f32 = np.float32
    m, t, e = models.numpy(), theta.numpy(), residual.numpy()
    K, P = m.shape
    out_i, out_v, res = [], [], np.zeros_like(e)
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(K):
            ids, vals = [], []
            for b0 in range(0, P, 256):
                js = list(range(b0, min(P, b0 + 256)))
                v = {j: (f32(m[r, j]) - f32(t[j])) + f32(e[r, j]) for j in js}
                kept = sorted(sorted(js, key=lambda j: (-_key(v[j]), j))[:min(k, len(js))])
                ids += [j - b0 for j in kept]
                vals += [v[j] for j in kept]
                for j in js:
                    res[r, j] = f32(0.0) if j in kept else v[j]
            out_i.append(ids)
            out_v.append(vals)
    return (torch.tensor(np.array(out_i, dtype=np.uint8)), torch.from_numpy(np.array(out_v, dtype=np.float32)),
            torch.from_numpy(res))


def _inputs(K, P, seed, residual=True):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    models = theta + torch.randn(K, P, generator=g) * torch.rand(K, 1, generator=g)
    res = 0.1 * torch.randn(K, P, generator=g) if residual else torch.zeros(K, P)
    return models, theta, res


@pytest.mark.parametrize("P", [1, 255, 256, 257, 1001, 4994])
@pytest.mark.parametrize("k", KS)
def test_reference_matches_scalar_transcription(P, k):
    models, theta, res = _inputs(2, P, seed=P + k)
    want_i, want_v, want_r = _scalar_topk(models, theta, res, k)
    r = res.clone()
    idx, val = reference.encode_topk_delta(models, theta, r, k)
    codec = UplinkCodec("topk", k)
    assert idx.shape == val.shape == (2, codec.entries(P)) and idx.dtype == torch.uint8
    assert torch.equal(idx, want_i) and same_bits(val, want_v) and same_bits(r, want_r)
    # CPU tensors through ops: the reference itself
    r2 = res.clone()
    i2, v2 = ops.encode_topk_delta(models, theta, r2, codec)
    assert torch.equal(i2, idx) and same_bits(v2, val) and same_bits(r2, r)


def _edge_inputs(P=5 * 256 + 3):
    """row 0: an all-zero block, a block of equal magnitudes (ties go to the lower index), a block of +-0 and tiny values, a
    block with several NaNs of different payloads, a block with +-Inf; row 1: random with a residual; last block 3 long"""
    theta = torch.randn(P)
    theta[:768] = 0.0                                            # v = d exactly in the first three blocks and the last
    theta[1280:] = 0.0
    d = 0.1 * torch.randn(2, P)
    d[0, :256] = 0.0
    d[0, 256:512] = 0.5 * torch.tensor([1.0, -1.0]).repeat(128)
    d[0, 512:768] = torch.tensor([0.0, -0.0]).repeat(128)
    d[0, 512 + 200] = 1e-40                                      # a subnormal: the only non-zero key of its block
    models = theta + d
    res = torch.zeros(2, P)
    res[0, 512:768] = torch.tensor([0.0, -0.0]).repeat(128)      # -0 + -0 = -0: keys 0 either way
    res[1] = 0.05 * torch.randn(P)
    nan_bits = np.array([0x7FC00001, 0xFFC00002, 0x7F800003, 0x7FC00000], dtype=np.uint32).view(np.float32)
    for i, j in enumerate((768 + 9, 768 + 3, 768 + 100, 768 + 40)):
        models[0, j] = float(nan_bits[i])
    models[0, 1024 + 5], models[0, 1024 + 6] = float("inf"), float("-inf")
    models[0, 1280] = theta[1280] + 1.0
    return models, theta, res


@pytest.mark.parametrize("k", [1, 2, 8, 32])
def test_edge_blocks(k):
    models, theta, res = _edge_inputs()
    r = res.clone()
    idx, val = reference.encode_topk_delta(models, theta, r, k)
    want_i, want_v, want_r = _scalar_topk(models, theta, res, k)
    assert torch.equal(idx, want_i) and same_bits(val, want_v) and same_bits(r, want_r)
    row = idx[0].long().view(-1)
    blocks = [row[b * k:(b + 1) * k].tolist() for b in range(5)] + [row[5 * k:].tolist()]
    assert blocks[0] == list(range(k))                           # all zero: the lowest offsets
    assert blocks[1] == list(range(k))                           # equal magnitudes: ties go to the lower index
    assert 200 in blocks[2] and blocks[2] == sorted([200] + list(range(k))[:k - 1])
    nans = [3, 9, 40, 100]                                       # NaNs are kept first, the lower index winning among them
    assert set(nans[:k]) <= set(blocks[3]) and (k < 4 or len(set(blocks[3]) & set(nans)) == 4)
    for b, offs in ((3, nans), (4, [5, 6])):
        got = {o: float(x) for o, x in zip(blocks[b], val[0, b * k:(b + 1) * k])}
        assert set(offs[:k]) <= set(got) and all(not np.isfinite(got[o]) for o in offs[:k])
    assert blocks[5][:1] == [0] and len(blocks[5]) == min(k, 3) and float(val[0, 5 * k]) == 1.0


@pytest.mark.parametrize("k", KS)
def test_sent_plus_residual_is_v_bit_for_bit(k):
    P = 1001
    models, theta, res = _inputs(3, P, seed=k)
    v = (models - theta) + res
    r = res.clone()
    idx, val = reference.encode_topk_delta(models, theta, r, k)
    sent = reference.decode_topk_delta(idx, val, k, P)
    mask = torch.zeros(3, P, dtype=torch.bool)
    pos = idx.long() + (torch.arange(idx.shape[1]) // k * 256)
    mask.scatter_(1, pos, True)
    assert int(mask.sum()) == 3 * UplinkCodec("topk", k).entries(P)        # disjoint supports, every entry distinct
    assert (r[mask] == 0).all() and (sent[~mask] == 0).all()
    assert same_bits(torch.where(mask, sent, r), v)
    # the kept entries are the k_b largest |v| of each block
    for b0 in range(0, P, 256):
        blk = v[:, b0:b0 + 256].abs()
        kept = mask[:, b0:b0 + 256]
        kb = min(k, blk.shape[1])
        assert (kept.sum(1) == kb).all()
        if kb < blk.shape[1]:
            assert (blk.masked_fill(~kept, float("inf")).amin(1) >= blk.masked_fill(kept, -1.0).amax(1)).all()


def test_error_feedback_delivers_every_delta():
    """over 20 rounds the decoded updates plus the final residual add up to the sum of the deltas: nothing is lost"""
    K, P, k = 2, 777, 4
    g = torch.Generator().manual_seed(0)
    theta = torch.randn(P, generator=g)
    res = torch.zeros(K, P)
    total_d = torch.zeros(K, P, dtype=torch.float64)
    total_sent = torch.zeros(K, P, dtype=torch.float64)
    for _ in range(20):
        models = theta + 0.01 * torch.randn(K, P, generator=g)
        total_d += (models - theta).double()
        idx, val = reference.encode_topk_delta(models, theta, res, k)
        total_sent += reference.decode_topk_delta(idx, val, k, P).double()
    torch.testing.assert_close(total_sent + res.double(), total_d, rtol=0, atol=1e-5)
    assert float((total_sent - total_d).abs().max()) > 1e-3          # the residual really carries something over


def test_codec_object():
    c = UplinkCodec("topk")
    assert c.k == 8 and c.sparse and not c.quantized and c.scale_count(1000) == 0
    assert not UplinkCodec("int8").sparse and UplinkCodec("int8").quantized
    assert UplinkCodec("int8", k=99).bits == 8                       # k is ignored by the other kinds
    # FFNN: 2,401 parameters, 10 blocks, the last one 97 long
    assert c.entries(2401) == 80 and c.payload_bytes(2401) == 400
    assert UplinkCodec("topk", 32).entries(2401) == 32 * 9 + 32 and UplinkCodec("topk", 1).entries(1) == 1
    assert UplinkCodec("topk", 8).entries(257) == 9 and UplinkCodec("topk", 8).entries(4994) == 8 * 19 + 8
    for p in (1, 255, 256, 257, 1001, 4994):
        assert c.entries(p) == reference.topk_entries(p, 8)
    for bad in (0, 33, -1, 8.0, True, None):
        with pytest.raises(ValueError):
            UplinkCodec("topk", bad)


def test_ops_apply_on_cpu_is_the_reference():
    codec, K, P = UplinkCodec("topk", 8), 5, 700
    models, theta, res = _inputs(K, P, seed=3)
    idx, val = reference.encode_topk_delta(models, theta, res, codec.k)
    w = torch.full((K,), 0.2)
    got = ops.fedavg_apply_topk(theta.clone(), idx, val, w, codec, 0.5)
    assert torch.equal(got, reference.fedavg_apply_topk(theta.clone(), idx, val, w, 8, 0.5))
    dec = reference.decode_topk_delta(idx, val, 8, P)
    assert torch.equal(got, theta.clone().add_(0.5 * ((theta + reference.fedavg_flat(dec, w)) - theta)))
    with pytest.raises(ValueError):
        ops.fedavg_apply_topk(theta.clone(), idx, val, w, UplinkCodec("int8"))
    with pytest.raises(ValueError):
        ops.fedavg_apply_topk(theta.clone(), idx, val, w, codec, 0.5, opt=ServerOpt("adam").init_state(P))
    for agg in (Aggregator("median"), Aggregator("trimmed_mean", 0.1)):
        with pytest.raises(ValueError):
            ops.fedavg_apply_topk(theta.clone(), idx, val, w, codec, aggregator=agg)
    ops.fedavg_apply_topk(theta.clone(), idx, val, w, codec, aggregator=Aggregator("mean"))
    with pytest.raises(ValueError):
        ops.encode_topk_delta(models, theta, res, UplinkCodec("int4"))


# ---- elementwise.cu on the SIMT CPU build ------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", KS)
def test_topk_delta_kernel_on_cpu_bit_exact(simt, k):
    K = 3
    for P in (1000, 1024, 1001, 5):               # 16-byte path (with a partial block) / scalar path (P % 4 != 0), k > m_last
        models, theta, res = _inputs(K, P, seed=K * P + k)
        if P >= 1000:
            models[1, 260] = float("nan")
            models[1, 300] = float("-inf")
            models[2, :256] = theta[:256]          # an all-zero block (residual 0 there)
            res[2, :256] = 0.0
        r_ref, r_sim = res.clone(), res.clone()
        want_i, want_v = reference.encode_topk_delta(models, theta, r_ref, k)
        idx, val = simt.topk_delta(models, theta, r_sim, k)
        assert torch.equal(idx, want_i) and same_bits(val, want_v) and same_bits(r_sim, r_ref), P
    # rows that are not 16-byte aligned (a view one float into a buffer): the scalar path, same bits
    buf = torch.randn(K * 1000 + 1)
    models, theta, res = buf[1:].view(K, 1000), torch.randn(1000), torch.zeros(K, 1000)
    r_ref = res.clone()
    want_i, want_v = reference.encode_topk_delta(models, theta, r_ref, k)
    idx, val = simt.topk_delta(models, theta, res, k)
    assert torch.equal(idx, want_i) and same_bits(val, want_v) and same_bits(res, r_ref)


@pytest.mark.parametrize("K", [1, 3, 16, 33, 100])
@pytest.mark.parametrize("k", [1, 8, 32])
def test_fedavg_topk_kernel_on_cpu(simt, K, k):
    P = 1001 if K < 100 else 203
    models, theta, res = _inputs(K, P, seed=K + k)
    if K > 2:
        models[1] = theta + 1e4                          # a large client
    idx, val = reference.encode_topk_delta(models, theta, res, k)
    w = torch.rand(K) + 0.1
    w /= w.sum()
    got = theta.clone()
    simt.fedavg_apply_topk(got, idx, val, w, k, 0.7)
    want = reference.fedavg_apply_topk(theta.clone(), idx, val, w, k, 0.7)
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def test_fedavg_topk_kernel_with_adam_on_cpu(simt):
    K, P, k = 7, 1001, 8
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(P), opt.init_state(P)
    theta = torch.randn(P)
    ref_theta = theta.clone()
    res = torch.zeros(K, P)
    w = torch.full((K,), 1.0 / K)
    for _ in range(3):
        models = theta + 0.5 * torch.randn(K, P)
        idx, val = reference.encode_topk_delta(models, theta, res, k)
        simt.fedavg_apply_topk(theta, idx, val, w, k, opt.lr, opt.code, opt.hyper, st.m, st.v)
        reference.fedavg_apply_topk(ref_theta, idx, val, w, k, opt=ref)
        torch.testing.assert_close(theta, ref_theta, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.m, ref.m, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.v, ref.v, rtol=1e-5, atol=1e-7)


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


def _remote_run(tmp_path, uplink, rounds=3, stub=None, model="ffnn"):
    from colearn_federated_learning_b200.control.arguments import Arguments
    args = Arguments(model=model, lr=0.1, batch_size=16, federate_after_n_batches=30, uplink=uplink, uplink_topk=8, synthetic=64)
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


def test_remote_rounds_with_topk_uplink_train_and_save_traffic(tmp_path):
    # traffic on the FFNN: 2,401 parameters, 10 blocks (the last one 97 long), 80 entries = 400 B against 9,604 B of fp32
    fp32, res32, _ = _remote_run(tmp_path / "a", "fp32")
    in32 = [r["bytes_in"] for r in fp32.metrics.records if "bytes_in" in r]
    assert res32["uplink"] == "fp32" and len(in32) == 3
    c, res, workers = _remote_run(tmp_path / "b", "topk")
    assert res["uplink"] == "topk" and res["dropped"] == [] and all(w.fits_served == 3 for w in workers)
    bytes_in = [r["bytes_in"] for r in c.metrics.records if "bytes_in" in r]
    assert all(a / b >= 15 for a, b in zip(in32, bytes_in)), (in32, bytes_in)
    # every worker carries a residual of the model's size after its fits
    assert all(w._residuals["ffnn"].shape == (1, 2401) and bool(w._residuals["ffnn"].any()) for w in workers)
    # training: the loss falls over 3 rounds (the MLP; the FFNN's loss does not fall in 3 rounds even with fp32 replies)
    c, res, _ = _remote_run(tmp_path / "c", "topk", model="mlp")
    losses = [np.mean(l) for l in c.metrics.per_round if l]
    assert res["dropped"] == [] and len(losses) == 3 and losses[2] < losses[0], losses


def _tampering_worker(mutate):
    from colearn_federated_learning_b200.control.workers import WorkerServer

    class Tampering(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            if req.get("op") == "fit" and resp.get("ok"):
                mutate(resp)
            return resp
    return Tampering


def _indices_with(fn):
    def mutate(resp):
        i = np.frombuffer(resp["indices"], dtype=np.uint8).copy()
        fn(i)
        resp["indices"] = i.tobytes()
    return mutate


def _set(i, pos, value):
    i[pos] = value


def _nan_value(resp):
    v = np.frombuffer(resp["values"], dtype="<f4").copy()
    v[3] = np.nan
    resp["values"] = v.tobytes()


@pytest.mark.parametrize("case", ["short_indices", "descending_index", "index_past_last_block", "nan_value", "wrong_topk"])
def test_a_bad_topk_reply_drops_the_device(tmp_path, case):
    mutate = {"short_indices": lambda r: r.update(indices=r["indices"][:-1]),
              "descending_index": _indices_with(lambda i: i.__setitem__(slice(8, 10), i[8:10][::-1].copy())),
              "index_past_last_block": _indices_with(lambda i: _set(i, -1, 97)),          # the FFNN's last block is 97 long
              "nan_value": _nan_value,
              "wrong_topk": lambda r: r.update(topk=9)}[case]
    c, res, workers = _remote_run(tmp_path, "topk", rounds=2, stub=_tampering_worker(mutate))
    bad = f"127.0.0.1:{workers[2].port}"
    assert res["dropped"] == [bad] and len(res["losses"]) == 2 and bad not in res["losses"]
    assert os.path.exists(c.path) and res["rounds"] == 2


def test_check_topk_reply_limits():
    from colearn_federated_learning_b200.control.coordinator import check_topk_reply
    codec, P = UplinkCodec("topk", 8), 600                  # 3 blocks, the last one 88 long: 24 entries
    models, theta, res = _inputs(1, P, seed=2)
    idx, val = reference.encode_topk_delta(models, theta, res, 8)
    good = {"uplink": "topk", "topk": 8, "indices": idx.numpy().tobytes(), "values": val.numpy().astype("<f4").tobytes()}
    i, v = check_topk_reply(good, codec, P)
    assert torch.equal(i, idx[0]) and torch.equal(v, val[0])
    edge = np.frombuffer(good["indices"], dtype=np.uint8).copy()
    edge[-1] = 87                                            # the last offset of the last block
    edge[7] = 255                                            # the last offset of a full block
    edge[:7] = np.arange(7)
    check_topk_reply(dict(good, indices=edge.tobytes()), codec, P)
    # an offset may repeat across blocks, but not inside one
    same = edge.copy()
    same[6] = same[5]
    for bad in (dict(good, topk=8.0), dict(good, topk=True), dict(good, uplink="int8"), dict(good, indices=None),
                dict(good, values=good["values"] + b"\0\0\0\0"), dict(good, indices=same.tobytes()),
                dict(good, indices=np.where(np.arange(24) == 23, 88, edge).astype(np.uint8).tobytes()),
                dict(good, values=np.full(24, np.inf, dtype="<f4").tobytes())):
        with pytest.raises(ValueError):
            check_topk_reply(bad, codec, P)


def test_worker_residual_lifetime():
    """ef_reset zeroes the residual, a fit without topk leaves it alone, a k outside 1..32 is refused before the fit"""
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    from colearn_federated_learning_b200.models import FFNN, flatten_params

    w, port = _worker(1)
    client = RemoteWorkerClient(w.id, "127.0.0.1", port)
    try:
        codec = UplinkCodec("topk", 4)
        theta = flatten_params(FFNN()).detach().clone()
        cfg = FitConfig(model="ffnn", loss="bce", batch_size=16, epochs=1, max_nr_batches=5, lr=0.1, shuffle=True, seed=1)

        def fit(reset):
            update, _, _ = client.fit_update(theta, cfg, codec, ef_reset=reset)
            from colearn_federated_learning_b200.control.coordinator import check_topk_reply
            idx, val = check_topk_reply(update, codec, theta.numel())
            sent = reference.decode_topk_delta(idx.view(1, -1), val.view(1, -1), 4, theta.numel())
            return sent, w._models["ffnn"][1].detach().clone().view(1, -1) - theta, w._residuals["ffnn"].clone()

        sent, d, r = fit(True)
        assert same_bits(torch.where(sent != 0, sent, r), d)               # residual 0 before: sent + new residual == d
        sent2, d2, r2 = fit(False)
        assert same_bits(torch.where(sent2 != 0, sent2, r2), d2 + r)      # the residual is carried over
        client.fit(theta, cfg)                                             # an fp32 fit leaves the residual alone
        assert torch.equal(w._residuals["ffnn"], r2)
        sent3, d3, r3 = fit(True)                                          # reset: as if there were no residual
        assert same_bits(torch.where(sent3 != 0, sent3, r3), d3)
        with pytest.raises(RuntimeError):
            client._call({"op": "fit", "config": cfg.to_dict(), "params": theta.numpy().tobytes(), "uplink": "topk", "topk": 33})
        assert w.fits_served == 4 and torch.equal(w._residuals["ffnn"], r3)
    finally:
        client.close()
        w.stop()


# ---- local mode and the CLI -------------------------------------------------------------------------------------------------
def test_local_mode_with_topk_uplink(tmp_path):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.coordinator import train_virtual_workers
    from colearn_federated_learning_b200.data import BaseDataset, federate, synthetic_unsw
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    from colearn_federated_learning_b200.utils.checkpoint import save_model

    args = Arguments(synthetic=90, lr=0.05, uplink="topk", uplink_topk=4)
    c, pub, clock = _make(tmp_path, args, rounds=3, remote=False)
    torch.manual_seed(0)
    init = FFNN()
    save_model(init, c.path)
    ips = ["10.0.0.1", "10.0.0.2", "10.0.0.3"]
    for ip in ips:
        pub.publish("topic/state", f"({ip}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert c.windower.last_result["uplink"] == "topk"
    cpu = torch.device("cpu")
    x, y = synthetic_unsw(90, seed=args.seed)
    fed = federate(BaseDataset(x, y), ips, cpu)
    cfg = c._fit_config("local")
    theta = flatten_params(init).clone()
    res = torch.zeros(3, theta.numel())
    for r in range(3):
        flats, _, _ = train_virtual_workers(theta, FFNN(), fed, cfg, r)
        idx, val = reference.encode_topk_delta(flats, theta, res, 4)
        reference.fedavg_apply_topk(theta, idx, val, torch.full((3,), 1.0 / 3), 4)
    m = FFNN()
    m.load_state_dict(torch.load(c.path, weights_only=True))
    assert torch.equal(flatten_params(m), theta)
    settings.training_devices.clear()


def _cli(*argv):
    import federated_coordinator as fc
    return fc.arguments_from_cli(fc.parse_cli(["-t", "topic/state", *argv]))


def test_cli_uplink_topk_flags():
    assert _cli().uplink_topk == 8 and not _cli().uplink_codec().sparse
    c = _cli("--uplink-codec", "topk").uplink_codec()
    assert c.sparse and c.k == 8
    assert _cli("--uplink-codec", "topk", "--uplink-topk", "32", "-r").uplink_codec().k == 32
    assert _cli("--uplink-codec", "topk", "--aggregator", "mean").uplink_codec().k == 8
    assert _cli("--uplink-codec", "int8", "--uplink-topk", "99").uplink_codec().bits == 8   # ignored by the other kinds
    assert _cli("--aggregator", "median").uplink == "fp32"
    for bad in (["--uplink-codec", "topk", "--box"], ["--uplink-codec", "topk", "-e"], ["--uplink-codec", "topk", "--uplink-topk", "0"],
                ["--uplink-codec", "topk", "--uplink-topk", "33"], ["--uplink-codec", "topk", "--aggregator", "median"],
                ["--uplink-codec", "topk", "--aggregator", "trimmed_mean"]):
        with pytest.raises(SystemExit):
            _cli(*bad)
