"""Asynchronous buffered aggregation in remote mode (``--async-buffer``, ``fl/asyncagg.py``): the staleness weights, the drop of
stale replies and the buffer order; the flag refusals; the worker's version echo; and an end-to-end run over loopback TCP
with one slow device whose recorded steps replay through ``ops.reference`` to the saved model bit for bit."""
import socket
import threading
import time

import pytest
import torch

import federated_coordinator as fc
from colearn_federated_learning_b200 import settings
from colearn_federated_learning_b200.control import workers as workers_mod
from colearn_federated_learning_b200.control.arguments import Arguments
from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
from colearn_federated_learning_b200.control.coordinator import Coordinator
from colearn_federated_learning_b200.control.window import FakeClock
from colearn_federated_learning_b200.control.workers import RemoteWorkerClient, WorkerServer
from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw
from colearn_federated_learning_b200.fl import FitConfig
from colearn_federated_learning_b200.fl.asyncagg import AsyncSettings, Reply, plan_step, replay, staleness_weight
from colearn_federated_learning_b200.models import FFNN, flatten_params

TOPIC = "topic/state"


# ---- semantics --------------------------------------------------------------------------------------------------------------
def test_staleness_weight_is_fedbuffs_inverse_square_root():
    assert staleness_weight(0, 0.5) == 1.0 and staleness_weight(3, 0.5) == 0.5 and staleness_weight(7, 1.0) == 0.125


def test_plan_drops_stale_replies_sorts_by_base_and_device_and_does_not_renormalise():
    st = AsyncSettings(buffer=4, max_staleness=2)
    buf = [Reply("b", 5, None, 10, 0.0), Reply("a", 5, None, 30, 0.0), Reply("c", 2, None, 10, 0.0), Reply("d", 4, None, 10, 0.0)]
    plan = plan_step(buf, 6, st, weighted=False)
    assert [r.device for r in plan.kept] == ["d", "a", "b"] and plan.stale_dropped == ["c"]
    assert plan.record == [["d", 4, 2, plan.weights[0]], ["a", 5, 1, plan.weights[1]], ["b", 5, 1, plan.weights[2]]]
    s2, s1 = 3 ** -0.5, 2 ** -0.5
    assert plan.weights == pytest.approx([s2 / 3, s1 / 3, s1 / 3], rel=1e-6)
    assert sum(plan.weights) < 1.0                                   # stale buffers make shorter steps
    w = plan_step(buf, 6, st, weighted=True).weights
    assert w == pytest.approx([0.2 * s2, 0.6 * s1, 0.2 * s1], rel=1e-6)
    # the arrival order does not matter, and every tau = 0 is the synchronous weighting
    assert plan_step(buf[::-1], 6, st, weighted=False).record == plan.record
    fresh = plan_step([Reply("x", 3, None, 1, 0.0), Reply("y", 3, None, 3, 0.0)], 3, st, weighted=True)
    assert fresh.weights == [0.25, 0.75] and fresh.stale_dropped == []


def test_settings_are_checked():
    for bad in (dict(buffer=0), dict(buffer=2, concurrency=-1), dict(buffer=2, max_staleness=-1), dict(buffer=2, exponent=-0.5)):
        with pytest.raises(ValueError):
            AsyncSettings(**bad)
    assert AsyncSettings(buffer=2, max_staleness=4).ring_slots == 6


# ---- flag refusals ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra,reason", [
    ([], "applies to remote mode"),                                                     # local mode
    (["-r", "--box"], "applies to remote mode"),
    (["-r", "-e"], "applies to remote mode"),
    (["-r", "--secure-agg"], "synchronous cohort"),
    (["-r", "--uplink-codec", "int8", "--downlink-codec", "int8"], "every device has seen every broadcast"),
    (["-r", "--model", "resnet18"], "BatchNorm"),
    (["-r", "--max-staleness", "-1"], "max-staleness"),
])
def test_async_flag_refusals(capsys, extra, reason):
    with pytest.raises(SystemExit):
        fc.parse_cli(["-t", TOPIC, "--async-buffer", "2", *extra])
    assert reason in capsys.readouterr().err


def test_async_settings_without_a_buffer_are_refused(capsys):
    with pytest.raises(SystemExit):
        fc.parse_cli(["-t", TOPIC, "-r", "--max-staleness", "2"])
    assert "need --async-buffer" in capsys.readouterr().err


def test_local_mode_coordinator_refuses_async(tmp_path):
    c, pub, clock = make(tmp_path, remote=False, rounds=1, args=Arguments(async_buffer=2, synthetic=64))
    with pytest.raises(ValueError, match="remote mode only"):
        c.starting_training_local({"192.168.1.7": object()})


# ---- protocol ---------------------------------------------------------------------------------------------------------------
def test_unversioned_fit_request_and_reply_are_unchanged(monkeypatch):
    w, port = worker(seed=1)
    sent = []
    real = workers_mod._send_msg
    monkeypatch.setattr(workers_mod, "_send_msg", lambda sock, obj: sent.append(obj) or real(sock, obj))
    try:
        client = RemoteWorkerClient("w", "127.0.0.1", port)
        cfg = FitConfig(model="ffnn", loss="bce", batch_size=8, epochs=1, lr=0.05)
        theta = flatten_params(FFNN())
        client.fit(theta, cfg, timeout=30)
        client.fit(theta, cfg, timeout=30, version=7)
        req0, req1 = [m for m in sent if m.get("op") == "fit"]
        assert list(req0) == ["op", "config", "params", "dataset_key"] and req1["version"] == 7
        assert {k: v for k, v in req1.items() if k != "version"} == req0
        assert "version" not in w._dispatch(dict(req0)) and w._dispatch(dict(req1))["version"] == 7
        client.close()
    finally:
        w.stop()


# ---- end to end over loopback TCP -------------------------------------------------------------------------------------------
def make(tmp_path, remote=False, rounds=1, args=None, device=torch.device("cpu"), **kw):
    broker, clock = InProcessBroker(), FakeClock()
    c = Coordinator(1, remote, rounds, False, False, args=args or Arguments(synthetic=64), broker=broker, timer_factory=clock,
                    path=str(tmp_path / "test.pth"), device=device, **kw)
    c.connect()
    c.subscribe(TOPIC)
    pub = BusClient("pub", broker=broker)
    pub.connect()
    return c, pub, clock


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class RecordingWorker(WorkerServer):
    """the worker remote_worker.py runs, with a fixed delay per fit and a log of (version, model sent, model returned)"""

    def __init__(self, *a, delay=0.0, **kw):
        super().__init__(*a, **kw)
        self.delay, self.log = delay, []

    def _dispatch(self, req):
        resp = super()._dispatch(req)
        if req.get("op") == "fit":
            time.sleep(self.delay)
            self.log.append((req.get("version"), workers_mod._from_bytes(req["params"]).clone(), workers_mod._from_bytes(resp["params"]).clone()))
        return resp


def worker(seed, delay=0.0):
    port = free_port()
    w = RecordingWorker(f"127.0.0.1:{port}", "127.0.0.1", port, device=torch.device("cpu"), delay=delay)
    w.add_dataset(BaseDataset(*synthetic_unsw(48, seed=seed)))
    w.start(block=False)
    return w, port


SERIALISE_DELAY = 0.15      # a busy executor: every fit request of the coordinator is serialised this much later than dispatched


def run_async(tmp_path, device, monkeypatch):
    real = workers_mod._to_bytes

    def late_to_bytes(t):
        if threading.current_thread().name.startswith("fit-rpc"):
            time.sleep(SERIALISE_DELAY)
        return real(t)

    monkeypatch.setattr(workers_mod, "_to_bytes", late_to_bytes)
    fast, slow = 0.1, 0.45
    ws = [worker(1, fast), worker(2, fast), worker(3, slow)]
    try:
        args = Arguments(lr=0.05, synthetic=64, federate_after_n_batches=5, async_buffer=2, max_staleness=10)
        c, pub, clock = make(tmp_path, remote=True, rounds=6, args=args, device=device, fit_timeout=30)
        for _, p in ws:
            pub.publish(TOPIC, f"(127.0.0.1, {p}, TRAINING)")
        c.drain()
        t0 = time.time()
        clock.advance(1.0)
        elapsed = time.time() - t0
        res = c.windower.last_result
        assert res is not None and "error" not in res, res
        return c, res, elapsed, ws, slow + SERIALISE_DELAY
    finally:
        for w, _ in ws:
            w.stop()


@pytest.mark.parametrize("device", [pytest.param("cpu"), pytest.param("cuda", marks=pytest.mark.gpu)])
def test_async_rounds_over_tcp_workers_replay_bit_for_bit(tmp_path, device, monkeypatch):
    if device == "cuda" and not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    c, res, elapsed, ws, slow = run_async(tmp_path, torch.device(device), monkeypatch)
    steps = [r for r in c.metrics.records if "async" in r]
    assert res["async_steps"] == 6 and len(steps) == 6 and res["dropped"] == []
    assert elapsed < 0.6 * 6 * slow                                   # synchronous rounds would wait 6 x the slow device
    slow_id = f"127.0.0.1:{ws[2][1]}"
    taus = {}
    for v, r in enumerate(steps):
        a = r["async"]
        assert a["version"] == v and len(a["replies"]) == 2 and a["stale_dropped"] == []
        for dev, base, tau, _ in a["replies"]:
            assert tau == v - base and 0 <= tau <= 10
            taus.setdefault(dev, []).append(tau)
    assert taus.get(slow_id) and min(taus[slow_id]) > 0
    # replay: each step's recorded replies, in record order, from the models the devices returned
    logs = {f"127.0.0.1:{p}": list(w.log) for w, p in ws}
    theta0 = next(sent for w, _ in ws for ver, sent, _ in w.log if ver == 0)
    plan = []
    for r in steps:
        models, bases, weights = [], [], []
        for dev, base, _, wk in r["async"]["replies"]:
            i = next(i for i, (ver, _, _) in enumerate(logs[dev]) if ver == base)
            models.append(logs[dev].pop(i)[2])
            bases.append(base)
            weights.append(wk)
        plan.append((models, bases, weights))
    versions = replay(theta0, plan, AsyncSettings(buffer=2, max_staleness=10))
    state = torch.load(c.path, map_location="cpu", weights_only=True)
    model = FFNN()
    model.load_state_dict(state)
    assert torch.equal(flatten_params(model).view(torch.int32), versions[-1].view(torch.int32))
    # what every device received is the version the coordinator recorded as its base, even when the request left late
    fits = [(ver, sent) for w, _ in ws for ver, sent, _ in w.log]
    assert fits and all(torch.equal(sent.view(torch.int32), versions[ver].view(torch.int32)) for ver, sent in fits)
    # every fit a device served was applied, dropped as stale or counted as discarded after the last step
    applied = sum(len(r["async"]["replies"]) + len(r["async"]["stale_dropped"]) for r in steps)
    assert len(fits) == applied + res["async_discarded"]
    assert len(settings.training_devices) == 0
