"""Federated anomaly detection (fl/anomaly.py) without a GPU: the autoencoder's persistent-kernel instances and
recon_summary_kernel through the SIMT build (the kernel sources on the CPU), the choice of the alarm bin, the checks on a
device's reply, local and remote runs that end in a threshold and 0 / 1 alarms, and every refusal."""
import importlib.util
import json
import math
import os
import shutil

import numpy as np
import pytest
import torch

import test_mlp_kernel_edges as E
from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl import anomaly
from colearn_federated_learning_b200.ops import reference as R

AE_DIMS = (10, 32, 4, 32, 10)
E.NETS.setdefault("autoencoder", (3, AE_DIMS, "none"))
ROUND_KEYS = ("round", "selected", "n_k", "loss_k", "fed_eval", "agg_weights")


@pytest.fixture(scope="module")
def simt():
    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- the autoencoder's instances of the persistent kernel ---------------------------------------------------------------
def ae_fit_case(ex, tag, n, B, epochs, variants):
    """target = input: the client's y is its x; the fit of every variant against the float64 replay"""
    theta0 = E._theta0("autoencoder")
    x = torch.rand(n, 10, generator=torch.Generator().manual_seed(1000 + n))
    perm = E._perm(n, epochs)
    ref = E._reference("autoencoder", "mse", x, x, perm, B, epochs, -1, theta0)
    out = {}
    for v in variants:
        outs, losses = ex.fit("autoencoder", "mse", [dict(x=x, y=x, theta_in=theta0, perm=perm)], B, epochs, -1, v)
        E._check_fit(tag, ref, theta0, outs[0], losses[0])
        out[v] = (outs[0], losses[0])
    return out


@pytest.mark.parametrize("n,B", [(0, 1), (1, 1), (65, 1), (70, 32), (32, 32)])
def test_autoencoder_fit_matches_float64_cpu(simt, n, B):
    ae_fit_case(E.Simt(simt), "cpu ae", n, B, 1 if B == 1 else 2, (5, 1, 3, 6))


def test_autoencoder_forward_and_parameter_count_cpu(simt):
    from colearn_federated_learning_b200.models import build_model
    assert ops.NET_KINDS[(AE_DIMS, "none")] == 3 and build_model("autoencoder").spec.n_params == 974
    E._forward(E.Simt(simt), "autoencoder", (1, 263, 265))


# ---- recon_summary_kernel ---------------------------------------------------------------------------------------------------
def special_rows():
    """x̂ - x differences whose error is 0, subnormal as a float, exactly 2^-24 / 2^8 and the floats next to them"""
    f32 = np.float32
    targets = [0.0, 2.0 ** -140, 2.0 ** -126, 2.0 ** -24, float(np.nextafter(f32(2.0 ** -24), f32(0))),
               float(np.nextafter(f32(2.0 ** -24), f32(1))), 256.0, float(np.nextafter(f32(256), f32(0))), float(np.nextafter(f32(256), f32(1e9))),
               1.0, 3.0, 1e30]
    xs, xh = [], []
    for t in targets:
        x = torch.zeros(10)
        h = torch.zeros(10)
        h[0] = float(np.float32(math.sqrt(t)))          # e = (float)sqrt(t)^2, within an ulp of t: the neighbours are exercised
        xs.append(x)
        xh.append(h)
    # a row whose error rounds to exactly 2^-24 and 2^8 as a float
    for t in (2.0 ** -24, 256.0):
        x, h = torch.zeros(10), torch.zeros(10)
        h[3] = math.sqrt(t)
        xs.append(x)
        xh.append(h)
    return torch.stack(xh), torch.stack(xs)


def make_recon_case(N, seed, dirty=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(N, 10, generator=g)
    scale = torch.exp(torch.randn(N, 1, generator=g) * 6.0)          # errors over every octave and beyond
    xh = x + torch.randn(N, 10, generator=g) * scale.sqrt() * 0.1
    y = (torch.rand(N, generator=g) < 0.3).float()
    if dirty and N > 20:
        sh, sx = special_rows()
        k = min(sh.shape[0], N - 10)
        xh[:k], x[:k] = sh[:k], sx[:k]
        xh[k, 2] = float("nan")
        x[k + 1, 5] = float("inf")
        xh[k + 2, 0] = float("-inf")
        y[k + 3] = 2.0
        y[k + 4] = 0.5
        y[k + 5] = float("nan")
        y[k + 6] = -1.0
    return xh.contiguous(), x.contiguous(), y


def segments_for(N):
    if N < 3:
        return [N]
    return [N // 3, 0, N - N // 3 - N // 5, N // 5]


def same_result(a, b):
    (c1, s1, e1, f1), (c2, s2, e2, f2) = a, b
    assert torch.equal(c1, c2)
    assert torch.equal(s1.view(torch.int64), s2.view(torch.int64))
    if e1 is None or e2 is None:
        assert e1 is None and e2 is None
        return
    assert torch.equal(torch.isnan(e1), torch.isnan(e2)) and torch.equal(e1[~torch.isnan(e1)], e2[~torch.isnan(e2)])
    assert torch.equal(f1, f2)


def offsets_of(segs):
    return torch.tensor([0] + np.cumsum(segs).tolist(), dtype=torch.int64)


@pytest.mark.parametrize("N", [0, 1, 2047, 2048, 2049, 5000])
@pytest.mark.parametrize("B", [32, 256, 4096])
def test_simt_recon_summary_matches_the_reference_bit_for_bit(simt, N, B):
    xh, x, y = make_recon_case(N, 7 * N + B)
    segs = segments_for(N)
    offs = offsets_of(segs)
    j = B // 2 + 3
    c, s, e, f = simt.recon_summary(xh, x, y, offs, B, j, 0)
    same_result((c, s, e, f), R.recon_summary(xh, x, y, B, offs.tolist(), j))
    c2, s2, _, _ = simt.recon_summary(xh, x, None, offs, B, -1, 3)          # no labels: every valid row counts as label 0
    same_result((c2, s2, None, None), R.recon_summary(xh, x, None, B, offs.tolist())[:2] + (None, None))
    if N > 100:
        assert int(c[:, 0].sum()) == N and int(c[:, 2 + B:].sum()) > 0 and int(c2[:, 2 + B:].sum()) == 0


def test_recon_bins_at_the_edges():
    e = torch.tensor([0.0, 2.0 ** -150, 2.0 ** -24, float(np.nextafter(np.float32(2.0 ** -24), np.float32(0))), 1.0, 1.5, 255.99,
                      256.0, 1e300, 2.0 ** -24 * 1.5], dtype=torch.float64)
    assert R.recon_bin(e, 32).tolist() == [0, 0, 0, 0, 24, 24, 31, 31, 31, 0]
    assert R.recon_bin(e, 64).tolist() == [0, 0, 0, 0, 48, 49, 63, 63, 63, 1]
    for bins in (32, 256, 4096):
        edges = torch.tensor([anomaly.bin_edge(j, bins) for j in range(1, bins)], dtype=torch.float64)
        assert R.recon_bin(edges, bins).tolist() == list(range(1, bins))                  # every lower edge opens its bin
        below = torch.from_numpy(np.nextafter(edges.float().numpy(), np.float32(0))).double()
        assert R.recon_bin(below, bins).tolist() == list(range(0, bins - 1))
    assert anomaly.bin_edge(0, 256) == 0.0 and anomaly.bin_edge(256, 256) == math.inf


def test_simt_recon_summary_grids_and_segments(simt):
    xh, x, y = make_recon_case(9000, 3)
    segs = [4100, 0, 1, 4899]
    offs = offsets_of(segs)
    base = simt.recon_summary(xh, x, y, offs, 256, 100, 0)
    for grid in (1, 2, 7):
        same_result(simt.recon_summary(xh, x, y, offs, 256, 100, grid), base)
    lo = 0
    for i, n in enumerate(segs):            # a segment's result does not depend on the others
        c, s, _, _ = simt.recon_summary(xh[lo:lo + n].contiguous(), x[lo:lo + n].contiguous(), y[lo:lo + n].contiguous(),
                                        torch.tensor([0, n]), 256, -1, 0)
        assert torch.equal(c[0], base[0][i]) and torch.equal(s.view(torch.int64)[0], base[1].view(torch.int64)[i])
        lo += n


def test_recon_summary_refuses_bad_arguments(simt):
    xh, x, y = make_recon_case(100, 1, dirty=False)
    for bins in (16, 48, 8192):
        with pytest.raises(ValueError):
            ops.recon_summary(xh, x, y, bins)
        with pytest.raises(RuntimeError):
            simt.recon_summary(xh, x, y, torch.tensor([0, 100]), bins, -1, 0)
    with pytest.raises(ValueError):
        ops.recon_summary(xh, x, y, 256, [50, 49])
    with pytest.raises(RuntimeError):
        simt.recon_summary(xh, x, y, torch.tensor([0, 60, 50, 100]), 256, -1, 0)
    with pytest.raises(ValueError):
        ops.recon_summary(xh, x, y, 256, alarm_bin=257)
    with pytest.raises(RuntimeError):
        simt.recon_summary(xh, x, y, torch.tensor([0, 100]), 256, 257, 0)
    with pytest.raises(ValueError):
        ops.recon_summary(xh[:, :5], x, y, 256)
    with pytest.raises(ValueError):
        R.recon_summary_limits(10, 256, 1 << 32)


# ---- the threshold and the replies --------------------------------------------------------------------------------------------
def test_alarm_bin_on_hand_made_histograms():
    h = np.zeros(64, dtype=np.int64)
    h[10] = 1000                                               # every row in one bin
    assert anomaly.alarm_bin(h, 0.01) == 11                    # 1000 > floor(10): the bin itself must stay silent
    assert anomaly.alarm_bin(h, 0.999) == 11
    h = np.zeros(64, dtype=np.int64)
    h[:50] = 2                                                 # N0 = 100, fpr N0 = 5 exactly -> 4 rows may alarm (bins 48, 49)
    assert anomaly.alarm_bin(h, 0.05) == 48 and int(h[48:].sum()) <= 5
    assert anomaly.alarm_bin(h, 0.06) == 47                    # floor(6) = 6 rows: bins 47..49
    assert anomaly.alarm_bin(h, 0.001) == 50                   # budget 0: above the last occupied bin
    h[63] = 3                                                  # the top bin alone exceeds the budget: no alarm at all
    assert anomaly.alarm_bin(h, 0.01) == 64 and anomaly.bin_edge(64, 64) == math.inf
    assert anomaly.alarm_bin(np.zeros(64, dtype=np.int64), 0.01) is None
    s = anomaly.ReconSummary(64, 10, 0, 1.0, np.stack([np.zeros(64, dtype=np.int64), np.eye(64, dtype=np.int64)[5] * 10]))
    rec = anomaly.record({"a": s}, 0.01, 64)
    assert rec["alarm_bin"] is None and rec["threshold"] is None and rec["total"]["fpr"] is None and rec["total"]["detection_rate"] is None


def test_metrics_at_the_alarm_bin():
    h0 = np.zeros(32, dtype=np.int64)
    h1 = np.zeros(32, dtype=np.int64)
    h0[:10] = 10                                               # 100 benign rows in bins 0..9
    h1[8:20] = 5                                               # 60 attack rows in bins 8..19
    s = anomaly.ReconSummary(32, 163, 3, 40.0, np.stack([h0, h1]))
    rec = anomaly.record({"a": s}, 0.1, 32)
    m = rec["total"]
    assert rec["alarm_bin"] == 9 and rec["threshold"] == anomaly.bin_edge(9, 32) == 2.0 ** -15
    assert (m["fp"], m["tn"], m["tp"], m["fn"]) == (10, 90, 55, 5) and m["fpr"] == 0.1 <= rec["fpr"]
    assert m["mean_error"] == 40.0 / 160 and m["detection_rate"] == 55 / 60 and m["precision"] == 55 / 65
    from colearn_federated_learning_b200.fl.fedeval import _auc_ap
    assert (m["auc"], m["ap"]) == _auc_ap(h0, h1)


def good_wire():
    xh, x, y = make_recon_case(500, 2)
    c, s, _, _ = R.recon_summary(xh, x, y, 64)
    return anomaly.to_wire(anomaly._summaries(c, s, 64)[0])


def test_tampered_replies_are_refused():
    ok = good_wire()
    assert anomaly.from_wire(dict(ok), 64).n == 500
    bad = []
    bad.append(dict(ok, counts=ok["counts"][:-4]))                                  # word count
    bad.append(dict(ok, counts=ok["counts"] + b"\0\0\0\0"))
    bad.append(dict(ok, n=ok["n"] + 1))                                               # hist != n - n_invalid
    bad.append(dict(ok, n_invalid=ok["n_invalid"] + 1))
    bad.append(dict(ok, n_invalid=-1))
    bad.append(dict(ok, err_sum=float("nan")))
    bad.append(dict(ok, err_sum=-1.0))
    bad.append(dict(ok, err_sum=float("inf")))
    bad.append(dict(ok, n="500"))
    bad.append(dict(ok, n=True))
    words = np.frombuffer(ok["counts"], dtype="<u4").copy()
    words[3] += 1
    bad.append(dict(ok, counts=words.tobytes()))
    for b in bad:
        with pytest.raises(ValueError):
            anomaly.from_wire(b, 64)
    with pytest.raises(ValueError):
        anomaly.from_wire(ok, 128)                                                  # the coordinator's bins, not the device's


# ---- the modes --------------------------------------------------------------------------------------------------------------
def local_run(tmp_path, device=torch.device("cpu"), **kw):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.utils.metrics import RoundLogger
    tmp_path.mkdir(parents=True, exist_ok=True)
    broker, clock = InProcessBroker(), FakeClock()
    metrics = RoundLogger(str(tmp_path / "rounds.jsonl"), str(tmp_path / "round.txt"))
    args = dict(synthetic=4000, lr=0.05, model="autoencoder", fed_eval_every=1, eval_fraction=0.25)
    args.update(kw)
    torch.manual_seed(0)                          # the fresh model's initialisation (the coordinator does not seed it)
    c = Coordinator(1, False, 3, False, False, args=Arguments(**args), broker=broker, timer_factory=clock,
                    path=str(tmp_path / "test.pth"), device=device, metrics=metrics)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    pub.publish("topic/state", "(192.168.1.7, TRAINING)")
    pub.publish("topic/state", "(192.168.1.8, TRAINING)")
    c.drain()
    clock.advance(1.0)
    recs = [json.loads(line) for line in open(tmp_path / "rounds.jsonl")]
    return c, recs, json.load(open(str(tmp_path / "test.pth") + ".json"))


AUC_BOUND = 0.9     # CPU runs of the 3-round, 4000-row synthetic case reach 0.97-0.99


def check_local(recs, meta):
    assert len(recs) == 3 and all("fed_eval" in r for r in recs)
    fe = recs[-1]["fed_eval"]
    assert fe["bins"] == 256 and fe["fpr"] == 0.01 and fe["alarm_bin"] is not None and 0 < fe["threshold"] < math.inf
    assert fe["threshold"] == anomaly.bin_edge(fe["alarm_bin"], 256)
    tot = fe["total"]
    assert tot["n"] == 1000 and tot["fpr"] <= 0.01 and tot["auc"] > AUC_BOUND and tot["detection_rate"] > 0.5
    assert sum(d["n"] for d in fe["devices"].values()) == 1000
    # every shard trains on its benign rows only: n_k = the benign count of its 1500 training rows
    assert all(0 < k < 1500 for k in recs[-1]["n_k"])
    assert meta["anomaly"] == {k: fe[k] for k in ("alarm_bin", "bins", "threshold", "fpr")}


def test_local_run_sets_a_threshold_and_repeats_exactly(tmp_path):
    _, recs, meta = local_run(tmp_path / "a")
    check_local(recs, meta)
    _, recs2, _ = local_run(tmp_path / "b")
    assert [{k: r.get(k) for k in ROUND_KEYS} for r in recs] == [{k: r.get(k) for k in ROUND_KEYS} for r in recs2]


def test_local_run_with_an_int8_uplink(tmp_path):
    _, recs, meta = local_run(tmp_path, uplink="int8")
    check_local(recs, meta)


def test_synthetic_anomaly_is_seeded():
    from colearn_federated_learning_b200.data import synthetic_anomaly, synthetic_for_model
    a, b = synthetic_anomaly(500, 3), synthetic_anomaly(500, 3)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and not torch.equal(a[0], synthetic_anomaly(500, 4)[0])
    x, y = synthetic_for_model("autoencoder", 4000, seed=1)
    assert x.shape == (4000, 10) and bool(((x >= 0) & (x <= 1)).all()) and 0.07 < float(y.mean()) < 0.13


def test_remote_run_ends_in_an_inference_of_alarms(tmp_path):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_anomaly
    from colearn_federated_learning_b200.fl.fedeval import split_eval
    from test_coordinator import TOPIC, _free_port, make
    from colearn_federated_learning_b200.control.workers import WorkerServer
    servers, ports = [], []
    try:
        for seed in (1, 2):
            port = _free_port()
            w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
            x, y = synthetic_anomaly(1500, seed=seed)
            w.add_dataset(BaseDataset(x, y))
            xt, yt, xe, ye = split_eval(*w.datasets["training"], 0.3, seed)
            w.datasets["training"], w.datasets["evaluation"] = (xt, yt), (xe, ye)
            w.load_data([r for r in synthetic_anomaly(8, seed=9)[0]], tag="inference")
            w.start(block=False)
            servers.append(w)
            ports.append(port)
        c, pub, clock = make(tmp_path, remote=True, rounds=2, evaluate_after=False,
                             args=Arguments(model="autoencoder", lr=0.05, fed_eval_every=1))
        for p in ports:
            pub.publish(TOPIC, f"(127.0.0.1, {p}, TRAINING)")
        c.drain()
        clock.advance(2.0)
        res = c.windower.last_result
        fe = res["fed_eval"]
        assert fe["alarm_bin"] is not None and fe["total"]["n"] == 900 and fe["eval_excluded"] == [] and fe["total"]["fpr"] <= 0.01
        assert json.load(open(c.path + ".json"))["anomaly"]["alarm_bin"] == fe["alarm_bin"]
        pub.publish(TOPIC, f"(127.0.0.1, {ports[0]}, INFERENCE)")
        c.drain()
        assert c.last_predictions is not None and len(c.last_predictions) == 8 and set(c.last_predictions) <= {0, 1}
    finally:
        for w in servers:
            w.stop()


def test_inference_without_a_threshold_is_refused(tmp_path, caplog):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.models import build_model
    from colearn_federated_learning_b200.utils.checkpoint import save_model
    from test_coordinator import TOPIC, _free_port, make
    port = _free_port()
    w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
    w.load_data([torch.rand(10) for _ in range(3)], tag="inference")
    w.start(block=False)
    try:
        c, pub, _ = make(tmp_path, remote=True, args=Arguments(model="autoencoder", fed_eval_every=1))
        save_model(build_model("autoencoder"), c.path, meta={"model": "autoencoder"})
        import logging
        with caplog.at_level(logging.INFO):
            pub.publish(TOPIC, f"(127.0.0.1, {port}, INFERENCE)")
            c.drain()
        assert c.last_predictions is None and "no alarm threshold" in caplog.text
    finally:
        w.stop()


def test_worker_predict_needs_an_alarm_bin():
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient, WorkerServer
    from colearn_federated_learning_b200.models import build_model, flatten_params
    from test_coordinator import _free_port
    port = _free_port()
    w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
    w.load_data([torch.rand(10) for _ in range(4)], tag="inference")
    w.start(block=False)
    try:
        cl = RemoteWorkerClient("x", "127.0.0.1", port)
        flat = flatten_params(build_model("autoencoder"))
        with pytest.raises(RuntimeError):
            cl.predict(flat, "autoencoder")
        assert cl.predict(flat, "autoencoder", alarm={"alarm_bin": 0, "bins": 256}) == [1, 1, 1, 1]      # bin 0: everything alarms
        assert cl.predict(flat, "autoencoder", alarm={"alarm_bin": 256, "bins": 256}) == [0, 0, 0, 0]
        cl.close()
    finally:
        w.stop()


def parse(argv):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import federated_coordinator
    return federated_coordinator.parse_cli(argv)


@pytest.mark.parametrize("argv", [
    ["--model", "autoencoder"],                                                      # no threshold without federated evaluation
    ["--model", "autoencoder", "--fed-eval-every", "0"],
    ["--model", "autoencoder", "--fed-eval-every", "1", "--eval-fraction", "0.2", "--eval-threshold", "0.7"],
    ["--model", "autoencoder", "--fed-eval-every", "1", "--eval-fraction", "0.2", "--eval-bins", "16"],
    ["--model", "autoencoder", "--fed-eval-every", "1", "--eval-fraction", "0.2", "--alarm-fpr", "0"],
    ["--model", "autoencoder", "--fed-eval-every", "1", "--eval-fraction", "0.2", "--alarm-fpr", "1"],
    ["--model", "autoencoder", "--fed-eval-every", "1", "--eval-fraction", "0.2", "--box"],
    ["--model", "autoencoder", "-e"],
])
def test_cli_refusals(argv):
    with pytest.raises(SystemExit):
        parse(["-t", "topic/state"] + argv)


def test_cli_accepts_the_autoencoder_with_federated_evaluation():
    ns = parse(["-t", "topic/state", "--model", "autoencoder", "--fed-eval-every", "1", "--eval-fraction", "0.2", "--alarm-fpr", "0.05"])
    assert ns.alarm_fpr == 0.05
    ns = parse(["-t", "topic/state", "-r", "--model", "autoencoder", "--fed-eval-every", "2"])
    assert ns.model == "autoencoder"


def test_coordinator_refuses_without_federated_evaluation(tmp_path):
    from colearn_federated_learning_b200.control.arguments import Arguments
    with pytest.raises(ValueError, match="fed-eval-every"):
        anomaly.check_settings(Arguments(model="autoencoder"))
    with pytest.raises(ValueError, match="box"):
        anomaly.check_settings(Arguments(model="autoencoder", fed_eval_every=1), box=True)
    with pytest.raises(ValueError):
        anomaly.check_settings(Arguments(model="autoencoder", fed_eval_every=1), encryption=True)
