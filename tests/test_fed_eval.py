"""Federated evaluation without a GPU: the detection-metrics summary (``ops/csrc/eval_summary.cuh``) — its PyTorch
transcription against independent numpy / scipy oracles, the kernel source on the SIMT CPU build against the transcription
(counts exact, loss to rtol 1e-6) over the edge cases of its grid, chunk and segment logic — the metrics and reply checks of
``fl/fedeval.py``, and federated evaluation in local, remote and box mode.

Loss tolerance.  Both sides sum float64 row losses in 2048-row chunks and the chunks in order; only the order inside a chunk
differs (the kernel's lane / warp tree, torch's own), so they agree to ~1e-15 relative: rtol 1e-6 leaves room for the
last-bit differences of the float64 log / exp of the two libraries."""
import json
import math
import os
import socket
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl import fedeval
from colearn_federated_learning_b200.ops import reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def make_case(C, N, seed, dirty=True):
    """scores [N, C] (probabilities for C = 1, logits otherwise) and labels [N], with NaN / infinite rows, out-of-range and
    non-integral labels when ``dirty``"""
    g = torch.Generator().manual_seed(seed)
    if C == 1:
        s = torch.rand(N, 1, generator=g)
        y = (torch.rand(N, generator=g) > 0.6).float()
    else:
        s = 3 * torch.randn(N, C, generator=g)
        y = torch.randint(0, C, (N,), generator=g).float()
    if dirty and N > 20:
        s[3] = float("nan")
        s[5, 0] = float("inf")
        y[7], y[9], y[11], y[13] = 0.5, float(max(C, 2)), -1.0, float("nan")
        if C == 1:
            s[15, 0], s[17, 0] = 1.5, -0.25                 # outside [0, 1]: not a score
            s[19, 0], s[20, 0] = 0.0, 1.0                   # the ends of the range (BCE log floor)
    return s, y


def segments_for(N):
    a = N // 3
    return [a, 0, N - a]


def np_counts(s, y, C, B, thr):
    """counts of one segment by plain numpy loops over the definition"""
    s, y = s.numpy().astype(np.float64), y.numpy().astype(np.float64)
    k = 2 if C == 1 else C
    conf = np.zeros((k, k), np.int64)
    hist = np.zeros((C, 2, B), np.int64)
    bad = 0
    for i in range(len(y)):
        lab = y[i]
        ok = np.isfinite(s[i]).all() and np.isfinite(lab) and lab >= 0 and lab < k and lab == math.floor(lab)
        if C == 1:
            ok = ok and 0.0 <= s[i, 0] <= 1.0
        if not ok:
            bad += 1
            continue
        t = int(lab)
        if C == 1:
            p = float(np.float32(s[i, 0]))
            conf[t, int(p > thr)] += 1
            hist[0, t, min(B - 1, int(p * B))] += 1
        else:
            z = s[i]
            m = z.max()
            e = np.exp(z - m)
            conf[t, int(np.argmax(z))] += 1
            for c in range(C):
                hist[c, int(t == c), min(B - 1, int(e[c] / e.sum() * B))] += 1
    return bad, conf, hist


@pytest.mark.parametrize("C", [1, 2, 10])
def test_reference_counts_match_a_numpy_oracle(C):
    s, y = make_case(C, 3000, 1)
    counts, loss = reference.eval_summary(s, y, 64, 0.3)
    bad, conf, hist = np_counts(s, y, C, 64, 0.3)
    k = 2 if C == 1 else C
    assert counts[0, 0] == 3000 and counts[0, 1] == bad
    assert np.array_equal(counts[0, 2:2 + k * k].numpy().reshape(k, k), conf)
    assert np.array_equal(counts[0, 2 + k * k:].numpy().reshape(C, 2, 64), hist)
    # loss: float64 per row
    sd, yd = s.double().numpy(), y.double().numpy()
    tot = 0.0
    for i in range(3000):
        lab = yd[i]
        ok = np.isfinite(sd[i]).all() and np.isfinite(lab) and 0 <= lab < k and lab == math.floor(lab) and (C > 1 or 0 <= sd[i, 0] <= 1)
        if not ok:
            continue
        if C == 1:
            p = sd[i, 0]
            tot += -max(math.log(p) if p > 0 else -math.inf, -100) if lab == 1 else -max(math.log1p(-p) if p < 1 else -math.inf, -100)
        else:
            z = sd[i]
            tot += math.log(np.exp(z - z.max()).sum()) - (z[int(lab)] - z.max())
    assert float(loss[0]) == pytest.approx(tot, rel=1e-12)


def test_auc_and_ap_match_mann_whitney_and_a_hand_computed_ap():
    from scipy.stats import mannwhitneyu, rankdata
    B = 32
    s, y = make_case(1, 4000, 2, dirty=False)
    s = s ** 3                                                      # skewed scores, many ties after quantisation
    counts, loss = reference.eval_summary(s, y, B, 0.5)
    summ = fedeval.Summary(1, B, int(counts[0, 0]), int(counts[0, 1]), float(loss[0]), counts[0, 2:].numpy())
    m = fedeval.metrics(summ)
    q = np.minimum(B - 1, (s[:, 0].numpy() * B).astype(np.int64))
    pos, neg = q[y.numpy() == 1], q[y.numpy() == 0]
    u = mannwhitneyu(pos, neg).statistic
    assert m["auc"] == pytest.approx(u / (len(pos) * len(neg)), abs=1e-12)
    r = rankdata(np.concatenate([pos, neg]))
    assert m["auc"] == pytest.approx((r[:len(pos)].sum() - len(pos) * (len(pos) + 1) / 2) / (len(pos) * len(neg)), abs=1e-12)
    # AP: thresholds at every distinct quantized score, highest first: sum (R_t - R_{t-1}) P_t
    ap, prev_r = 0.0, 0.0
    for t in sorted(set(q.tolist()), reverse=True):
        tp, fp = int((pos >= t).sum()), int((neg >= t).sum())
        rec = tp / len(pos)
        ap += (rec - prev_r) * tp / (tp + fp)
        prev_r = rec
    assert m["ap"] == pytest.approx(ap, abs=1e-12)
    tn, fp, fn, tp = (int(v) for v in summ.confusion.reshape(-1))
    assert (m["tp"], m["fp"], m["tn"], m["fn"]) == (tp, fp, tn, fn)
    assert m["detection_rate"] == pytest.approx(tp / (tp + fn)) and m["fpr"] == pytest.approx(fp / (fp + tn))
    assert m["f1"] == pytest.approx(2 * tp / (2 * tp + fp + fn)) and m["accuracy"] == pytest.approx((tp + tn) / 4000)


@pytest.mark.parametrize("C", [1, 2, 10])
@pytest.mark.parametrize("N", [0, 1, 2047, 2048, 2049, 20000])
@pytest.mark.parametrize("B", [2, 256, 4096])
def test_simt_build_matches_the_reference(simt, C, N, B):
    if C * 2 * B > 32768:
        pytest.skip("outside the summary's limits (tested as a refusal)")
    s, y = make_case(C, N, 10 * C + N % 7)
    offs = torch.tensor([0] + np.cumsum(segments_for(N)).tolist(), dtype=torch.int64)
    c1, l1 = simt.eval_summary(s, y, offs, B, 0.5, 0)
    c2, l2 = reference.eval_summary(s, y, B, 0.5, offs.tolist())
    assert torch.equal(c1, c2)
    assert torch.allclose(l1, l2, rtol=1e-6, atol=0)


@pytest.mark.parametrize("C", [1, 10])
def test_simt_build_misaligned_scores_and_one_bin(simt, C):
    N = 5000
    s, y = make_case(C, N, 3)
    buf = torch.empty(N * C + 1)
    buf[1:] = s.reshape(-1)
    mis = buf[1:].view(N, C)                                        # 4 bytes past a 16-byte boundary
    assert mis.data_ptr() % 16 == 4
    offs = torch.tensor([0, 1234, N])
    c1, l1 = simt.eval_summary(mis, y, offs, 256, 0.5, 0)
    c2, l2 = reference.eval_summary(s, y, 256, 0.5, offs.tolist())
    assert torch.equal(c1, c2) and torch.allclose(l1, l2, rtol=1e-6, atol=0)
    # every row in one bin: a trained detector's confident scores (the hot-bin case of the warp aggregation)
    one = torch.full((N, C), 0.999 if C == 1 else -20.0)
    if C > 1:
        one[:, 0] = 20.0
    c3, l3 = simt.eval_summary(one, y, offs, 256, 0.5, 0)
    c4, l4 = reference.eval_summary(one, y, 256, 0.5, offs.tolist())
    assert torch.equal(c3, c4) and torch.allclose(l3, l4, rtol=1e-6, atol=0)
    k = 2 if C == 1 else C
    h = c3[:, 2 + k * k:].reshape(2, C, 2, 256)
    assert int(h[:, 0, :, 255].sum()) == int(c3[:, 0].sum() - c3[:, 1].sum())


@pytest.mark.parametrize("C", [1, 10])
def test_simt_grid_and_segment_independence(simt, C):
    N = 9000
    s, y = make_case(C, N, 4)
    offs = torch.tensor([0, 2049, 2049, 7000, N])
    c0, l0 = simt.eval_summary(s, y, offs, 128, 0.5, 0)
    for grid in (1, 2, 5):
        c, l = simt.eval_summary(s, y, offs, 128, 0.5, grid)
        assert torch.equal(c, c0) and torch.equal(l.view(torch.int64), l0.view(torch.int64))
    for i in range(4):
        lo, hi = int(offs[i]), int(offs[i + 1])
        c, l = simt.eval_summary(s[lo:hi].contiguous(), y[lo:hi].contiguous(), torch.tensor([0, hi - lo]), 128, 0.5, 0)
        assert torch.equal(c[0], c0[i]) and torch.equal(l.view(torch.int64)[0], l0.view(torch.int64)[i])


def _summaries(counts, loss, C, B):
    return [fedeval.Summary(C, B, int(c[0]), int(c[1]), float(l), c[2:].numpy()) for c, l in zip(counts, loss)]


@pytest.mark.parametrize("C", [1, 2, 10])
def test_segments_add_up_to_the_concatenation(C):
    N = 7000
    s, y = make_case(C, N, 5)
    parts = _summaries(*ops.eval_summary(s, y, 64, 0.5, [1000, 0, 2500, 3500]), C, 64)
    whole = _summaries(*ops.eval_summary(s, y, 64, 0.5), C, 64)[0]
    tot = fedeval.add(parts)
    assert (tot.n, tot.n_invalid) == (whole.n, whole.n_invalid) and np.array_equal(tot.counts, whole.counts)
    assert tot.loss_sum == pytest.approx(whole.loss_sum, rel=1e-12)
    for p in parts:
        fedeval.check(p)
    m = fedeval.metrics(whole)
    assert m["n"] == N and m["n_invalid"] > 0 and 0 <= m["accuracy"] <= 1 and m["auc"] is not None


def test_accuracy_at_one_half_equals_evaluate():
    from colearn_federated_learning_b200.fl.evaluate import evaluate, forward_flat
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    torch.manual_seed(0)
    model = FFNN()
    x = torch.rand(3000, 10)
    y = (torch.rand(3000) > 0.5).float()
    flat = flatten_params(model)
    ref = evaluate(model, x, y.view(-1, 1), flat=flat, verbose=False)
    s = fedeval.summarize(model, flat, x, y)[0]
    m = fedeval.metrics(s)
    assert m["accuracy"] == ref["accuracy"] and s.n_invalid == 0
    out = forward_flat(model, flat, x).reshape(-1)
    half = torch.full_like(out, 0.5)                                # p = 0.5 exactly: round-half-even and p > 0.5 agree
    assert fedeval.metrics(fedeval.Summary(1, 256, 3000, 0, 0.0, ops.eval_summary(half, y)[0][0, 2:].numpy()))["accuracy"] == \
        int((torch.round(half) == y).sum()) / 3000


def test_undefined_metrics_are_none():
    s = fedeval.Summary(1, 4, 3, 0, 0.3, np.array([3, 0, 0, 0] + [3, 0, 0, 0] + [0, 0, 0, 0], np.int64))
    fedeval.check(s)
    m = fedeval.metrics(s)
    assert m["recall"] is None and m["auc"] is None and m["ap"] is None and m["f1"] is None and m["fpr"] == 0.0
    empty = fedeval.Summary(1, 4, 2, 2, 0.0, np.zeros(12, np.int64))
    m = fedeval.metrics(fedeval.check(empty))
    assert m["loss"] is None and m["accuracy"] == 0.0
    assert all(v is None or not (isinstance(v, float) and math.isnan(v)) for v in m.values())


def _good_reply():
    s, y = make_case(1, 500, 6)
    return fedeval.to_wire(_summaries(*ops.eval_summary(s, y, 16, 0.5), 1, 16)[0])


def test_reply_checks_refuse_malformed_summaries():
    good = _good_reply()
    s = fedeval.from_wire(good, 1, 16)
    assert s.n == 500 and s.n_invalid > 0 and len(good["counts"]) == 4 * (4 + 32)
    assert fedeval.to_wire(fedeval.Summary(1, 256, 0, 0, 0.0, np.zeros(516, np.int64)))["counts"].__len__() == 2064   # FFNN, B = 256
    words = np.frombuffer(good["counts"], "<u4").copy()

    def bad(**kw):
        r = dict(good, **kw)
        with pytest.raises(ValueError):
            fedeval.from_wire(r, 1, 16)

    bad(counts=good["counts"][:-4])                                   # short
    bad(counts=good["counts"] + b"\0\0\0\0")                          # long
    bad(counts=None)
    bad(n=good["n_invalid"] - 1)                                     # n_invalid > n
    bad(n=-1)
    bad(n=True)
    bad(n=good["n"] + 1)                                             # confusion no longer sums to n - n_invalid
    w = words.copy(); w[0] += 1                                      # confusion and histograms disagree
    bad(counts=w.astype("<u4").tobytes(), n=good["n"] + 1)
    w = words.copy(); w[4] -= 1; w[4 + 16] += 1                      # a negative moved into the positive histogram
    bad(counts=w.astype("<u4").tobytes())
    bad(loss_sum=float("nan"))
    bad(loss_sum=-1.0)
    bad(loss_sum="1.0")
    with pytest.raises(ValueError):
        fedeval.from_wire(good, 2, 16)                               # a 2-class layout has other lengths


def test_refusals_and_limits():
    from colearn_federated_learning_b200.models import TestingRemote, flatten_params
    m = TestingRemote()
    with pytest.raises(ValueError, match="sigmoid"):
        fedeval.summarize(m, flatten_params(m), torch.rand(10, 2), torch.zeros(10))
    s = torch.rand(10, 1)
    for kw in (dict(bins=3), dict(bins=1), dict(bins=8192), dict(threshold=1.5), dict(threshold=float("nan"))):
        with pytest.raises(ValueError):
            ops.eval_summary(s, torch.zeros(10), **kw)
    with pytest.raises(ValueError, match="32768"):
        ops.eval_summary(torch.rand(10, 10), torch.zeros(10), bins=4096)
    with pytest.raises(ValueError):
        ops.eval_summary(torch.rand(10, 33), torch.zeros(10))
    with pytest.raises(ValueError):
        ops.eval_summary(s, torch.zeros(10), segments=[4, 5])
    import federated_coordinator as fc
    for argv in (["-r", "--secure-agg", "--fed-eval-every", "1"], ["--fed-eval-every", "1"],
                 ["--fed-eval-every", "1", "--eval-fraction", "0.2", "--model", "testing_remote"],
                 ["--fed-eval-every", "1", "--eval-fraction", "0.2", "--eval-bins", "100"],
                 ["--eval-fraction", "0.2"], ["-r", "--fed-eval-every", "1", "--eval-fraction", "0.2"],
                 ["-e", "--fed-eval-every", "1", "--eval-fraction", "0.2"]):
        with pytest.raises(SystemExit):
            fc.parse_cli(["-t", "t", *argv])
    ns = fc.parse_cli(["-t", "t", "--fed-eval-every", "2", "--eval-fraction", "0.2", "--eval-bins", "64", "--eval-threshold", "0.7"])
    a = fc.arguments_from_cli(ns)
    assert (a.fed_eval_every, a.eval_bins, a.eval_threshold, a.eval_fraction) == (2, 64, 0.7, 0.2)


def test_split_eval_is_a_seeded_random_subset_and_keeps_training_order():
    x = torch.arange(100).float().view(-1, 1)
    y = torch.arange(100).float()
    xt, yt, xe, ye = fedeval.split_eval(x, y, 0.2, 7)
    perm = torch.randperm(100, generator=torch.Generator().manual_seed(7))
    assert torch.equal(ye, perm[:20].float()) and torch.equal(xe.view(-1), ye)
    assert torch.equal(yt, torch.sort(perm[20:]).values.float()) and torch.equal(xt.view(-1), yt)


# ---- the modes ----------------------------------------------------------------------------------------------------------------
def _local(tmp_path, **kw):
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.utils.metrics import RoundLogger
    broker, clock = InProcessBroker(), FakeClock()
    metrics = RoundLogger(str(tmp_path / "rounds.jsonl"), str(tmp_path / "round.txt"))
    c = Coordinator(1, False, 3, False, False, args=Arguments(synthetic=200, lr=0.05, **kw), broker=broker, timer_factory=clock,
                    path=str(tmp_path / "test.pth"), device=torch.device("cpu"), metrics=metrics)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    pub.publish("topic/state", "(192.168.1.7, TRAINING)")
    pub.publish("topic/state", "(192.168.1.8, TRAINING)")
    c.drain()
    clock.advance(1.0)
    return c, [json.loads(l) for l in open(tmp_path / "rounds.jsonl")]


def test_local_mode_writes_fed_eval_records(tmp_path):
    c, recs = _local(tmp_path, fed_eval_every=2, eval_fraction=0.2)
    assert [("fed_eval" in r) for r in recs] == [False, True, True]        # every 2nd round and the last one
    fe = recs[-1]["fed_eval"]
    assert set(fe["devices"]) == {"192.168.1.7", "192.168.1.8"} and fe["eval_excluded"] == [] and fe["eval_missing"] == []
    assert fe["total"]["n"] == 40 and sum(d["n"] for d in fe["devices"].values()) == 40      # 0.2 of two 100-row shards
    assert all(k in fe["total"] for k in ("detection_rate", "fpr", "precision", "f1", "auc", "ap", "balanced_accuracy"))
    assert recs[-1]["n_k"] == [80, 80]
    assert c.windower.last_result["fed_eval"] == fe
    assert open(tmp_path / "round.txt").read().count("Federated evaluation round") == 2


def test_defaults_leave_records_and_shards_unchanged(tmp_path):
    c, recs = _local(tmp_path)
    assert all("fed_eval" not in r for r in recs) and recs[-1]["n_k"] == [100, 100]
    assert "fed_eval" not in c.windower.last_result


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_remote_mode_lists_a_device_without_evaluation_data(tmp_path):
    """coordinator -r with two remote_worker.py processes: one holds 25% of its rows out, the other has no evaluation data"""
    bport, w1, w2 = _free_port(), _free_port(), _free_port()
    metrics = str(tmp_path / "rounds.jsonl")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    coord = subprocess.Popen([sys.executable, os.path.join(ROOT, "federated_coordinator.py"), "-t", "topic/state", "-r",
                              "-w", "2", "-f", "2", "-p", str(bport), "--embedded-broker", "--checkpoint", str(tmp_path / "test.pth"),
                              "--max-batches", "20", "--exit-after", "1", "--no-cuda", "--metrics", metrics, "--fed-eval-every", "1"],
                             env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    workers = []
    try:
        time.sleep(4.0)
        for port, extra in ((w1, ["--eval-fraction", "0.25"]), (w2, [])):
            workers.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "remote_worker.py"), "--host", "127.0.0.1",
                                             "-p", str(port), "-b", "127.0.0.1", "--broker-port", str(bport), "-t", "topic/state",
                                             "-w", "1", "--synthetic", "64", "--no-cuda", *extra], env=env,
                                            stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL))
        out, _ = coord.communicate(timeout=120)
        assert coord.returncode == 0, out[-2000:]
        recs = [json.loads(l) for l in open(metrics)]
        assert len(recs) == 2 and all("fed_eval" in r for r in recs)
        fe = recs[-1]["fed_eval"]
        assert list(fe["devices"]) == [f"127.0.0.1:{w1}"] and fe["eval_missing"] == [f"127.0.0.1:{w2}"] and fe["eval_excluded"] == []
        assert fe["total"]["n"] == 16 and fe["devices"][f"127.0.0.1:{w1}"]["n"] == 16
    finally:
        for w in workers:
            w.kill()
        if coord.poll() is None:
            coord.kill()


def test_box_mode_two_ranks_gloo(tmp_path):
    metrics = str(tmp_path / "rounds.jsonl")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                          "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "federated_coordinator.py"),
                          "-t", "topic/state", "--box", "--model", "mlp", "--synthetic", "200", "-f", "3", "-w", "10",
                          "--checkpoint", str(tmp_path / "test.pth"), "--batch-size", "8", "--metrics", metrics,
                          "--fed-eval-every", "2", "--eval-fraction", "0.2", "--exit-after", "1"],
                         env=env, capture_output=True, text=True, timeout=240, cwd=str(tmp_path))
    assert out.returncode == 0, out.stderr[-2000:]
    recs = [json.loads(l) for l in open(metrics)]
    assert [("fed_eval" in r) for r in recs] == [False, True, True]
    fe = recs[-1]["fed_eval"]
    assert list(fe["devices"]) == ["10.0.0.1:8777", "10.0.0.2:8778"] and fe["total"]["n"] == 40
    assert recs[-1]["n_k"] == [80, 80] and fe["total"]["macro_f1"] is not None and len(fe["total"]["per_class"]) == 2
    assert out.stderr.count("Federated evaluation round") == 2


# ---- the global model is what is scored, and the coordinator decides the shape ---------------------------------------------
class _Head(torch.nn.Module):
    """a model that is not an MLPNet: forward_flat runs the module itself"""

    def __init__(self):
        super().__init__()
        self.body = torch.nn.Linear(10, 8)
        self.head = torch.nn.Linear(8, 3)

    def forward(self, x):
        return self.head(torch.relu(self.body(x)))


@pytest.mark.parametrize("name", ["head", "resnet18"])
def test_a_non_mlp_summary_scores_the_parameters_passed_in(name):
    from colearn_federated_learning_b200.models import build_model, flatten_params
    torch.manual_seed(0)
    model = _Head() if name == "head" else build_model("resnet18")
    x = torch.rand(64, 10) if name == "head" else torch.rand(8, 3, 32, 32)
    y = torch.randint(0, 3 if name == "head" else 10, (x.shape[0],)).float()
    theta = flatten_params(model).clone()
    other = theta + 0.5 * torch.randn_like(theta)
    a = fedeval.summarize(model, theta, x, y)[0]
    b = fedeval.summarize(model, other, x, y)[0]             # the module now holds `other`
    a2 = fedeval.summarize(model, theta, x, y)[0]            # ... and theta is loaded back before the forward
    assert a.loss_sum != b.loss_sum and a2.loss_sum == a.loss_sum and np.array_equal(a2.counts, a.counts)
    model.eval()
    with torch.no_grad():
        out = model(x)
    c, l = reference.eval_summary(out, y, 256, 0.5)
    assert np.array_equal(a2.counts, c[0, 2:].numpy()) and a2.loss_sum == pytest.approx(float(l[0]), rel=1e-12)
    assert fedeval.check_model(model) == (3 if name == "head" else 10)


class _FakeDevice:
    def __init__(self, reply):
        self.reply = reply

    def evaluate(self, flat, model_name, bins, threshold, timeout=None):
        return self.reply


def test_remote_replies_of_another_class_count_are_excluded_not_fatal(tmp_path):
    import asyncio
    from concurrent.futures import ThreadPoolExecutor

    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock

    def reply(C, seed):
        s, y = make_case(C, 300, seed, dirty=False)
        return {"ok": True, **fedeval.to_wire(_summaries(*ops.eval_summary(s, y, 16, 0.5), C, 16)[0])}

    c = Coordinator(1, True, 1, False, False, args=Arguments(fed_eval_every=1, eval_bins=16), broker=InProcessBroker(),
                    timer_factory=FakeClock(), path=str(tmp_path / "test.pth"), device=torch.device("cpu"))
    alive = {"a": _FakeDevice(reply(2, 1)), "b": _FakeDevice(reply(10, 2)), "c": _FakeDevice(reply(1, 3)),
             "d": _FakeDevice({"ok": False, "eval_missing": True}), "e": _FakeDevice({"ok": False, "error": "refused"})}
    pool = ThreadPoolExecutor(max_workers=4)
    loop = asyncio.new_event_loop()
    try:
        rec = loop.run_until_complete(c._remote_fed_eval(alive, torch.zeros(1), 2, loop, pool))
    finally:
        loop.close()
        pool.shutdown()
    assert list(rec["devices"]) == ["a"] and rec["eval_excluded"] == ["b", "c", "e"] and rec["eval_missing"] == ["d"]
    assert rec["total"]["n"] == 300 and len(rec["total"]["per_class"]) == 2


def test_worker_refuses_a_bad_evaluate_request_cleanly():
    from colearn_federated_learning_b200.control.workers import WorkerServer, _to_bytes
    from colearn_federated_learning_b200.models import FFNN, flatten_params
    w = WorkerServer("127.0.0.1:0", "127.0.0.1", 0, device=torch.device("cpu"))
    try:
        w.datasets["evaluation"] = (torch.rand(20, 7), torch.zeros(20))
        params = _to_bytes(flatten_params(FFNN()))
        for req in ({"op": "evaluate", "params": params, "model": "no_such_model"},
                    {"op": "evaluate", "params": params},
                    {"op": "evaluate", "params": params, "model": "ffnn"},              # 7 features, the FFNN wants 10
                    {"op": "evaluate", "params": params, "model": "ffnn", "bins": 3}):
            resp = w._dispatch(req)
            assert resp["ok"] is False and resp["error"], req
        w.datasets["evaluation"] = (torch.rand(20, 10), torch.zeros(20))
        resp = w._dispatch({"op": "evaluate", "params": params, "model": "ffnn", "bins": 16})
        assert resp["ok"] and fedeval.from_wire(resp, 1, 16).n == 20
    finally:
        w._server.server_close()                                       # (never started: nothing to shut down)
