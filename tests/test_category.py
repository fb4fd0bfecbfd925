"""Attack categorisation (``--model ffnn_category``, fl/category.py), CPU side.

* The attack-category FFNN (10-50-30-10-5, softmax cross-entropy; ``mlp_v2.cuh``'s fused softmax head) through the SIMT build
  of the kernel source against the float64 replay of ``reference.mlp_local_sgd``, with the bounds and helpers of
  ``test_mlp_kernel_edges.py``: batch 1 around every chunk boundary, batches 2-100, an empty shard, ``max_nr_batches``
  inside an epoch, several clients in one launch, saturated logits and non-finite features; variant 6 = variant 5.
* ``mlp_forward`` of the new kind, the host executor against the reference, the refusal of a label outside [0, 5).
* The data layer: the category vocabulary, the load refusals, and the binary tensors unchanged.
* End to end in local mode (synthetic data) and in remote mode (remote_worker.py processes over TCP for the plain training,
  in-process workers for the int8 uplink and FedBuff), and the CLI refusals.

The head's softmax budget (``_replay_cat(absolute=True)``): per logit, ``ex2.approx`` (2 ulp) with the rounding of
``(z_c − m)·log2 e`` (``|z_c − m|`` ulp), the C − 1 additions of the sum and its ``rcp.approx`` (1 ulp), the product and the
subtraction: ``(8 + 2 C + 2 max_c |z_c − m|) u`` relative to ``(p + 1) / B``, carried back like the binary heads' budget."""
import json
import math
import os
import subprocess
import sys
import time
from unittest import mock

import numpy as np
import pytest
import torch

import test_mlp_kernel_edges as E
from colearn_federated_learning_b200.ops import reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAT = "ffnn_category"
DIMS = (10, 50, 30, 10, 5)
U, LR = E.U, E.LR
MACRO_F1_MIN = 0.8                               # synthetic_category: the majority class (Normal) is 40 % of the rows


def _data(n, seed=0):
    g = torch.Generator().manual_seed(2000 + 17 * n + seed)
    return torch.rand(n, 10, generator=g), torch.randint(0, 5, (n, 1), generator=g).float()


def _replay_cat(theta0, x, y, perm, B, epochs, max_b, dtype=torch.float64, absolute=False):
    """test_mlp_kernel_edges._replay for the C-class softmax head (see the module docstring for its budget)"""
    C = DIMS[-1]
    flat = theta0.to(dtype).clone()
    n = x.shape[0]
    x, y = x.to(dtype), y.to(dtype)
    losses, it = [], 0
    acc = torch.zeros_like(flat) if absolute else None
    L = len(DIMS) - 1
    k = sum(DIMS[i] + DIMS[i + 1] + 4 for i in range(L))
    gam = k * U / (1 - k * U)
    for e in range(epochs):
        order = perm[e % perm.shape[0]].long()
        for lo in range(0, n, B):
            idx = order[lo:lo + B]
            xb, yb = x[idx], y[idx]
            out, acts = R.mlp_forward(flat, DIMS, xb, "none")
            value, dz = R.loss_and_dz(out, yb, "xent", "none")
            g = R.mlp_backward(flat, DIMS, acts, dz)
            if absolute:
                views = R.mlp_views(flat, DIMS)
                h, aabs = xb.abs(), []
                for w, b in views:
                    aabs.append(h)
                    h = h @ w.abs().t() + b.abs()
                scale = 1.0 / xb.shape[0]
                mag = (torch.softmax(out, 1) + 1.0) * scale
                spread = (out - out.max(1, keepdim=True).values).abs().max(1, keepdim=True).values
                mufu = (8 + 2 * C + 2 * spread) * U * torch.ones_like(out)
                D = gam * mag + mufu * mag + 2 * scale * gam * h
                for li in range(L - 1, -1, -1):
                    w, _ = views[li]
                    gw, gb = R.mlp_views(acc, DIMS)[li]
                    gw += LR * (D.t() @ aabs[li])
                    gb += LR * D.sum(0)
                    if li > 0:
                        D = (D @ w.abs()) * (acts[li] != 0).to(dtype)
            flat.sub_(LR * g)
            losses.append(value)
            it += 1
            if max_b > 0 and it >= max_b:
                return flat, losses, acc
    return flat, losses, acc


def _reference(x, y, perm, B, epochs, max_b, theta0):
    steps = E._steps(x.shape[0], B, epochs, max_b)
    if steps == 0:
        return steps, None, None
    r64 = _replay_cat(theta0, x, y, perm, B, epochs, max_b, absolute=steps <= 3)
    r32 = _replay_cat(theta0, x, y, perm, B, epochs, max_b, dtype=torch.float32) if steps > 3 else None
    return steps, r64, r32


def fit_case(ex, tag, n, B, epochs, max_b, variants, perm_rows=None, bits_pairs=False, x=None, y=None, theta0=None):
    theta0 = E._theta0(CAT) if theta0 is None else theta0
    if x is None:
        x, y = _data(n)
    perm = E._perm(n, perm_rows or epochs)
    ref = _reference(x, y, perm, B, epochs, max_b, theta0)
    results = {}
    for v in variants:
        outs, losses = ex.fit(CAT, "xent", [dict(x=x, y=y, perm=perm, theta_in=theta0)], B, epochs, max_b, v)
        results[v] = (outs[0], losses[0])
        E._check_fit(tag, ref, theta0, outs[0], losses[0])
    if 5 in results and 6 in results:
        assert torch.equal(results[5][0], results[6][0]) and torch.equal(results[5][1], results[6][1]), "variant 6 != 5"
    if bits_pairs:
        v = variants[0]
        outs, losses = ex.fit(CAT, "xent", [dict(x=x, y=y, perm=perm, theta_in=theta0)], B, epochs, max_b, v)
        assert torch.equal(outs[0], results[v][0]) and torch.equal(losses[0], results[v][1]), "two launches differ"
    return results


def saturated(ex, scale, variants):
    """Logits spread to ±scale around the label's: one step, finite, within the bound"""
    theta0 = E._theta0(CAT)
    x, y = _data(4)
    for i in range(4):
        th = theta0.clone()
        hw, hb = R.mlp_views(th, DIMS)[-1]
        hw.mul_(scale)
        hb.mul_(scale)
        xi, yi = x[i:i + 1], y[i:i + 1]
        for v in variants:
            outs, losses = ex.fit(CAT, "xent", [dict(x=xi, y=yi, perm=E._perm(1, 1), theta_in=th)], 1, 1, -1, v)
            assert bool(torch.isfinite(outs[0]).all()), (scale, v)
            E._check_fit(f"cat saturated x{scale}", _reference(xi, yi, E._perm(1, 1), 1, 1, -1, th), th, outs[0], losses[0])


def many_clients(ex, B, count, variants):
    """``count`` clients of mixed sizes in one launch: each one's output and losses are its own launch's, bit for bit"""
    theta0 = E._theta0(CAT)
    clients = []
    for i in range(count):
        n = (0, 1, 64, 65, 130)[i % 5]
        x, y = _data(n, seed=i)
        clients.append(dict(x=x, y=y, perm=E._perm(n, 2, seed=i), theta_in=theta0))
    for v in variants:
        outs, losses = ex.fit(CAT, "xent", clients, B, 2, -1, v)
        for i in range(count):
            o, lo = ex.fit(CAT, "xent", [clients[i]], B, 2, -1, v)
            assert torch.equal(outs[i], o[0]) and torch.equal(losses[i], lo[0]), (v, i)


simt = E.simt


@pytest.fixture(scope="module", autouse=True)
def cat_net():
    """The executors and helpers of test_mlp_kernel_edges look nets up in its NETS table: the category net is in it for the
    tests of this module only"""
    with mock.patch.dict(E.NETS, {CAT: (4, DIMS, "none")}):
        yield


# ---- the kernel through the SIMT build -------------------------------------------------------------------------------
@pytest.mark.parametrize("n", E.CPU_BATCH1_N)
def test_batch1_chunk_edges_cpu(simt, n):
    fit_case(simt, "cat cpu b1", n, 1, 1, -1, (5, 6, 1, 3) if n in (1, 65) else (5,))


@pytest.mark.parametrize("B,n", [(2, 9), (7, 75), (63, 130), (64, 129), (65, 131), (100, 203), (9, 9), (5, 0)])
def test_batches_cpu(simt, B, n):
    fit_case(simt, "cat cpu batch", n, B, 2, -1, (5, 6, 1, 3) if B in (7, 65) else (5,))


@pytest.mark.parametrize("B,n,epochs,max_b", [(1, 20, 3, 13), (7, 30, 3, 6), (1, 20, 2, 20)])
def test_max_batches_cpu(simt, B, n, epochs, max_b):
    fit_case(simt, "cat cpu max_b", n, B, epochs, max_b, (5, 1))


@pytest.mark.parametrize("B", [1, 3])
def test_clients_in_one_launch_cpu(simt, B):
    many_clients(simt, B, 6, (5, 1))


@pytest.mark.parametrize("scale", [20, 60, 100])
def test_saturated_logits_cpu(simt, scale):
    saturated(simt, scale, (5, 1))


@pytest.mark.parametrize("what", ["x_nan", "x_inf", "x_-inf"])
def test_non_finite_features_cpu(simt, what):
    E._non_finite(simt, CAT, "xent", what, (5, 6, 1, 3))


def test_forward_cpu(simt):
    E._forward(simt, CAT, (1, 263, 265))


# ---- ops, host executor ----------------------------------------------------------------------------------------------
def test_net_kind_and_model():
    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.models import DEFAULT_LOSS, build_model, num_params
    from colearn_federated_learning_b200.ops import fused_mlp
    m = build_model(CAT)
    assert m.spec.dims == DIMS and m.spec.target == "category" and DEFAULT_LOSS[CAT] == "xent"
    assert ops.net_kind_for(DIMS, "none") == 4 and fused_mlp.BEST_VARIANT[4] == 5 and num_params(m) == 2445


def test_host_executor_against_reference():
    from colearn_federated_learning_b200.ops import host
    if not host.available():
        pytest.skip("the host executor is not built")
    theta0 = E._theta0(CAT)
    x, y = _data(50)
    perm = E._perm(50, 2)
    for B in (1, 7):
        flat = theta0.clone()
        host.mlp_local_sgd_multi(DIMS, "none", [flat], [x], [y], [perm], B, LR, 2, -1, "xent", threads=1)
        ref = theta0.double().clone()
        R.mlp_local_sgd(ref, DIMS, x.double(), y.double(), perm, B, LR, 2, -1, "xent", "none")
        r32 = _replay_cat(theta0, x, y, perm, B, 2, -1, dtype=torch.float32)[0]
        bound = E.C_LONG * (r32.double() - ref).abs().max().item() + 2.0 ** -20 * (ref - theta0.double()).abs().max().item()
        assert (flat.double() - ref).abs().max().item() <= bound, B


@pytest.mark.parametrize("bad", [5.0, -1.0, 2.5, float("nan")])
def test_out_of_range_label_refused(bad):
    from colearn_federated_learning_b200 import ops
    theta0 = E._theta0(CAT)
    x, y = _data(8)
    y[3, 0] = bad
    flat = theta0.clone()
    with pytest.raises(ValueError, match="row 3 is not a class index"):
        ops.mlp_local_sgd(flat, DIMS, x, y, None, 1, LR, 1, -1, "xent", "none")
    assert torch.equal(flat, theta0)
    # no other net kind gains the check: the FFNN takes an SSE target of 7 (outside [0, 5), valid for its loss) as before
    flat = E._theta0("ffnn").clone()
    ops.mlp_local_sgd(flat, (10, 50, 30, 10, 1), torch.rand(4, 10), torch.tensor([[0.0], [bad], [7.0], [1.0]]), None, 1, LR, 1,
                      -1, "sse", "sigmoid")
    assert not torch.equal(flat, E._theta0("ffnn"))


# ---- data ----------------------------------------------------------------------------------------------------------
def _csv(tmp_path, n=200, seed=3, edit=None):
    from colearn_federated_learning_b200.data import write_synthetic_csv
    import pandas as pd
    p = str(tmp_path / f"d{seed}.csv")
    write_synthetic_csv(p, n, seed=seed)
    if edit is not None:
        df = pd.read_csv(p)
        edit(df)
        df.to_csv(p, index=False)
    return p


def test_vocabulary_and_codes(tmp_path):
    from colearn_federated_learning_b200.data import CATEGORIES, NetworkTrafficDataset
    import pandas as pd
    assert CATEGORIES == ("Normal", "DDoS", "DoS", "Reconnaissance", "Theft")
    p = _csv(tmp_path)
    ds = NetworkTrafficDataset(p)
    df = pd.read_csv(p)
    assert ds.categories.tolist() == [CATEGORIES.index(c) for c in df["category"]]
    assert ((ds.categories != 0) == (df["attack"].to_numpy() != 0)).all()


def test_load_refusals(tmp_path):
    from colearn_federated_learning_b200.data import NetworkTrafficDataset

    def unknown(df):
        df.loc[7, "category"] = "Worm"

    def disagree(df):
        i = int(np.flatnonzero(df["attack"].to_numpy() == 0)[0])
        df.loc[i, "category"] = "DoS"
        df.attrs["row"] = i

    with pytest.raises(ValueError, match=r"d3\.csv:9: category 'Worm' is not one of Normal, DDoS"):
        NetworkTrafficDataset(_csv(tmp_path, edit=unknown))
    import pandas as pd
    p = _csv(tmp_path, seed=4, edit=disagree)
    i = int(np.flatnonzero((pd.read_csv(p)["attack"].to_numpy() == 0) & (pd.read_csv(p)["category"] == "DoS").to_numpy())[0])
    with pytest.raises(ValueError, match=rf"d4\.csv:{i + 2}: attack 0 disagrees with category 'DoS'"):
        NetworkTrafficDataset(p)


def test_no_category_column(tmp_path):
    """A CSV without the column loads as before; only the category model is refused on it"""
    from colearn_federated_learning_b200.data import NetworkTrafficDataset, category_tensors
    p = _csv(tmp_path, edit=lambda df: df.drop(columns=["category"], inplace=True))
    ds = NetworkTrafficDataset(p)
    assert ds.categories is None and ds.tensors()[0].shape == (200, 10)
    with pytest.raises(ValueError, match="no attack categories"):
        category_tensors(ds)


def test_binary_tensors_unchanged(tmp_path):
    """x, y and tensors() are what the parent computed: MinMax of the ten features and the attack column, bit for bit"""
    from colearn_federated_learning_b200.data import FEATURE_COLUMNS, NetworkTrafficDataset, minmax_scale
    import pandas as pd
    p = _csv(tmp_path)
    df = pd.read_csv(p)
    ds = NetworkTrafficDataset(p)
    x, y = ds.tensors()
    assert torch.equal(x, torch.from_numpy(np.ascontiguousarray(minmax_scale(df[FEATURE_COLUMNS].values))).float())
    assert torch.equal(y, torch.from_numpy(df["attack"].to_numpy(dtype=np.float32)).view(-1, 1))
    d, lab = ds[5]
    assert np.array_equal(lab, np.array([df["attack"].iloc[5]]))


def test_synthetic_category_and_unchanged_generators():
    from colearn_federated_learning_b200.data import synthetic_category, synthetic_for_model, synthetic_unsw
    x, y = synthetic_category(4000, seed=1)
    assert x.shape == (4000, 10) and bool(((x >= 0) & (x <= 1)).all())
    counts = torch.bincount(y.view(-1).long(), minlength=5).tolist()
    assert len(counts) == 5 and all(c > 0 for c in counts) and max(counts) == counts[0]
    assert torch.equal(synthetic_for_model(CAT, 100, 2)[1], synthetic_category(100, 2)[1])
    assert torch.equal(synthetic_for_model("ffnn", 100, 2)[0], synthetic_unsw(100, 2)[0])


# ---- end to end ----------------------------------------------------------------------------------------------------
def hand_collapse(conf):
    conf = np.asarray(conf)
    return {"tn": int(conf[0, 0]), "fp": int(conf[0, 1:].sum()), "fn": int(conf[1:, 0].sum()), "tp": int(conf[1:, 1:].sum())}


def test_attack_view_is_the_collapsed_matrix():
    from colearn_federated_learning_b200.fl import category, fedeval
    rng = np.random.default_rng(0)
    bins = 16
    conf = rng.integers(0, 50, (5, 5))
    hist = np.stack([np.stack([rng.multinomial(int(conf.sum() - r), np.ones(bins) / bins), rng.multinomial(int(r), np.ones(bins) / bins)])
                     for r in conf.sum(1)])
    s = fedeval.Summary(classes=5, bins=bins, n=int(conf.sum()), n_invalid=0, loss_sum=1.0,
                        counts=np.concatenate([conf.reshape(-1), hist.reshape(-1)]).astype(np.int64))
    v = category.attack_view(s)
    want = hand_collapse(conf)
    assert {k: v[k] for k in want} == want
    assert v["detection_rate"] == want["tp"] / (want["tp"] + want["fn"]) and v["fpr"] == want["fp"] / (want["fp"] + want["tn"])
    # ROC-AUC of "attack" ranked by 1 - p(Normal) is the Normal-vs-rest ROC-AUC of p(Normal)
    assert math.isclose(v["auc"], fedeval._auc_ap(hist[0, 0], hist[0, 1])[0])


def local_run(tmp_path, device=torch.device("cpu"), **kw):
    """A 4-worker local training on synthetic_category with a federated evaluation after every round (test_anomaly.local_run)"""
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.utils.metrics import RoundLogger
    tmp_path.mkdir(parents=True, exist_ok=True)
    broker, clock = InProcessBroker(), FakeClock()
    metrics = RoundLogger(str(tmp_path / "rounds.jsonl"), str(tmp_path / "round.txt"))
    args = dict(synthetic=4000, lr=0.05, model=CAT, loss="xent", fed_eval_every=1, eval_fraction=0.25)
    args.update(kw)
    torch.manual_seed(0)
    c = Coordinator(1, False, 4, False, False, args=Arguments(**args), broker=broker, timer_factory=clock,
                    path=str(tmp_path / "test.pth"), device=device, metrics=metrics)
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    for i in range(4):
        pub.publish("topic/state", f"(192.168.1.{7 + i}, TRAINING)")
    c.drain()
    clock.advance(1.0)
    recs = [json.loads(line) for line in open(tmp_path / "rounds.jsonl")]
    return c, recs, json.load(open(str(tmp_path / "test.pth") + ".json"))


def check_local(recs, meta):
    """Macro F1 over MACRO_F1_MIN (the majority class alone gives macro F1 ~0.11), and the attack block is the hand collapse of
    the record's confusion counts"""
    assert recs and all("fed_eval" in r for r in recs)
    fe = recs[-1]["fed_eval"]
    assert fe["classes"] == ["Normal", "DDoS", "DoS", "Reconnaissance", "Theft"] and meta["classes"] == fe["classes"]
    tot = fe["total"]
    assert tot["macro_f1"] >= MACRO_F1_MIN, tot["macro_f1"]
    assert len(tot["per_class"]) == 5 and tot["n"] == 1000
    att = fe["attack"]
    assert att["tp"] + att["fp"] + att["tn"] + att["fn"] == tot["n"] - tot["n_invalid"]
    # the Normal row of the collapsed matrix: recall of class 0 = tn / (tn + fp)
    assert math.isclose(tot["per_class"][0]["recall"], att["tn"] / (att["tn"] + att["fp"]))
    assert math.isclose(att["detection_rate"], att["tp"] / (att["tp"] + att["fn"]))
    return fe


def test_local_mode_end_to_end(tmp_path):
    _, recs, meta = local_run(tmp_path)
    check_local(recs, meta)


def test_record_attack_block_equals_hand_collapse():
    from colearn_federated_learning_b200.fl import category, fedeval
    from colearn_federated_learning_b200.models import build_model, flatten_params
    from colearn_federated_learning_b200.data import synthetic_category
    model = build_model(CAT)
    x, y = synthetic_category(600, 4)
    sums = fedeval.summarize(model, flatten_params(model), x, y, 64, 0.5, [300, 300])
    rec = category.record({"a": sums[0], "b": sums[1]})
    tot = fedeval.add(sums)
    assert {k: rec["attack"][k] for k in ("tn", "fp", "fn", "tp")} == hand_collapse(tot.confusion)
    assert rec["classes"][0] == "Normal" and rec["total"] == fedeval.metrics(tot)


def parse(argv):
    sys.path.insert(0, ROOT)
    import federated_coordinator
    return federated_coordinator.parse_cli(argv)


@pytest.mark.parametrize("flags", [["--box"], ["-e"]])
def test_box_and_encryption_refused(flags, capsys):
    with pytest.raises(SystemExit):
        parse(["-t", "topic/state", "--model", CAT, *flags])
    assert f"--model {CAT} does not run" in capsys.readouterr().err


def _servers(csvs, tmp_path):
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import NetworkTrafficDataset
    from test_coordinator import _free_port
    servers, ports = [], []
    for seed, csv in enumerate(csvs):
        port = _free_port()
        w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
        w.add_dataset(NetworkTrafficDataset(csv))
        w.hold_out_evaluation(0.3, seed)
        w.load_data([r for r in w.datasets["evaluation"][0][:6]], tag="inference")
        w.start(block=False)
        servers.append(w)
        ports.append(port)
    return servers, ports


def test_remote_worker_processes(tmp_path):
    """coordinator -r with three remote_worker.py processes over TCP, each holding 30 % of its rows out: a Bot-IoT CSV, synthetic
    rows made for the category model (--synthetic --data-model ffnn_category), and a CSV without the category column.  The
    first two train and are scored as a 5-class model; the third refuses the fit with its reason and leaves the training."""
    from test_fed_eval import _free_port
    bport, w1, w2, w3 = _free_port(), _free_port(), _free_port(), _free_port()
    metrics = str(tmp_path / "rounds.jsonl")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    csv = _csv(tmp_path, n=400, seed=1)
    plain = _csv(tmp_path, n=400, seed=2, edit=lambda df: df.drop(columns=["category"], inplace=True))
    coord = subprocess.Popen([sys.executable, os.path.join(ROOT, "federated_coordinator.py"), "-t", "topic/state", "-r",
                              "-w", "20", "-f", "2", "-p", str(bport), "--embedded-broker", "--checkpoint", str(tmp_path / "cat.pth"),
                              "--max-batches", "50", "--exit-after", "1", "--no-cuda", "--metrics", metrics, "--fed-eval-every", "1",
                              "--model", CAT, "--loss", "xent", "--lr", "0.05"],
                             env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    workers = []
    try:
        time.sleep(4.0)
        for port, data in ((w1, ["-dt", csv]), (w2, ["--synthetic", "400", "--data-model", CAT]), (w3, ["-dt", plain])):
            workers.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "remote_worker.py"), "--host", "127.0.0.1",
                                             "-p", str(port), "-b", "127.0.0.1", "--broker-port", str(bport), "-t", "topic/state",
                                             "-w", "1", "--eval-fraction", "0.3", "--no-cuda", *data], env=env,
                                            stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL))
        out, _ = coord.communicate(timeout=300)
        assert coord.returncode == 0, out[-3000:]
        recs = [json.loads(line) for line in open(metrics)]
        assert len(recs) == 2 and all("fed_eval" in r for r in recs)
        fe = recs[-1]["fed_eval"]
        ok, refused = [f"127.0.0.1:{w1}", f"127.0.0.1:{w2}"], f"127.0.0.1:{w3}"
        # the refused device leaves the training after its first fit (it is not asked to evaluate): it is in no round
        assert all(sorted(r["selected"]) == sorted(ok) for r in recs), [r["selected"] for r in recs]
        assert f"Worker {refused} failed its fit" in out and "trains on attack categories" in out
        assert sorted(fe["devices"]) == sorted(ok)
        assert fe["classes"][0] == "Normal" and len(fe["total"]["per_class"]) == 5 and fe["total"]["n"] == 240
        assert json.load(open(str(tmp_path / "cat.pth") + ".json"))["classes"] == fe["classes"]
    finally:
        for w in workers:
            w.kill()
        if coord.poll() is None:
            coord.kill()


def test_synthetic_category_rows_keep_their_codes():
    """remote_worker.py --synthetic N --data-model ffnn_category hosts the class indices as categories and the binary attack
    label as targets, so the device accepts the category model's fit"""
    sys.path.insert(0, ROOT)
    import remote_worker
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import synthetic_category
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    from colearn_federated_learning_b200.models import build_model, flatten_params
    from test_coordinator import _free_port
    args = remote_worker.build_parser().parse_args(["--host", "127.0.0.1", "-b", "x", "-t", "t", "--synthetic", "100",
                                                    "--data-model", CAT, "--seed", "3"])
    ds = remote_worker.pick_dataset(args)
    x, codes = synthetic_category(100, 3)
    assert ds.categories.tolist() == codes.view(-1).long().tolist() and torch.equal(ds.targets, (codes != 0).float())
    port = _free_port()
    w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
    w.add_dataset(ds)
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient
    w.start(block=False)
    try:
        cl = RemoteWorkerClient("x", "127.0.0.1", port)
        got, loss, n = cl.fit(flatten_params(build_model(CAT)), FitConfig(model=CAT, loss="xent", max_nr_batches=10))
        assert n == 100 and got.numel() == 2445 and math.isfinite(float(loss))
        cl.close()
    finally:
        w.stop()


@pytest.mark.parametrize("extra", [{"uplink": "int8"}, {"async_buffer": 2}])
def test_remote_mode_end_to_end(tmp_path, extra):
    """Two devices with categories and one without over TCP: the two train and are scored as a 5-class model, the third is
    refused (ok: False) and listed; INFERENCE returns class indices"""
    from colearn_federated_learning_b200.control.arguments import Arguments
    from test_coordinator import TOPIC, make
    csvs = [_csv(tmp_path, n=600, seed=s) for s in (1, 2)] + [_csv(tmp_path, n=300, seed=9, edit=lambda df: df.drop(columns=["category"], inplace=True))]
    servers, ports = _servers(csvs, tmp_path)
    try:
        c, pub, clock = make(tmp_path, remote=True, rounds=2, evaluate_after=False,
                             args=Arguments(model=CAT, loss="xent", lr=0.05, fed_eval_every=1, **extra))
        for p in ports:
            pub.publish(TOPIC, f"(127.0.0.1, {p}, TRAINING)")
        c.drain()
        clock.advance(2.0)
        res = c.windower.last_result
        fe = res["fed_eval"]
        assert fe["classes"][0] == "Normal" and len(fe["total"]["per_class"]) == 5
        assert f"127.0.0.1:{ports[2]}" in res["dropped"] + fe["eval_missing"] + fe["eval_excluded"]
        assert fe["total"]["n"] == 360
        assert json.load(open(c.path + ".json"))["classes"] == fe["classes"]
        pub.publish(TOPIC, f"(127.0.0.1, {ports[0]}, INFERENCE)")
        c.drain()
        assert c.last_predictions is not None and len(c.last_predictions) == 6 and set(c.last_predictions) <= set(range(5))
    finally:
        for w in servers:
            w.stop()


def test_device_without_categories_refuses_the_fit():
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient, WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    from colearn_federated_learning_b200.models import build_model, flatten_params
    from test_coordinator import _free_port
    port = _free_port()
    w = WorkerServer(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"))
    w.add_dataset(BaseDataset(torch.rand(20, 10), torch.zeros(20, 1)))
    w.start(block=False)
    try:
        cl = RemoteWorkerClient("x", "127.0.0.1", port)
        with pytest.raises(RuntimeError, match="trains on attack categories"):
            cl.fit(flatten_params(build_model(CAT)), FitConfig(model=CAT, loss="xent"))
        cl.close()
    finally:
        w.stop()
