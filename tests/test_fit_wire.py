"""The fit wire of every uplink / downlink / secure-aggregation / asynchronous combination the CLI accepts, pinned frame by frame.

Two devices with fixed ids train a two-round (or two-step) remote training over loopback TCP.  Every frame a device serves is
reduced to its op, the key order of its request and its reply, and the length of every bytes value in them.  No float value
and no executor path is kept, so ``tests/golden/fit_wire.json`` is the same on every machine; ``python tests/test_fit_wire.py``
rewrites it.  Which device takes which fit under asynchronous aggregation depends on timing, so those runs keep each device's
distinct frames in first-seen order; the synchronous runs keep every frame.
"""
import json
import os
import socket
import sys

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fit_wire.json")

RUNS = {
    "fp32": {},
    "int8": {"uplink": "int8"},
    "int4": {"uplink": "int4"},
    "topk": {"uplink": "topk"},
    "int8+int8": {"uplink": "int8", "downlink": "int8"},
    "topk+topk": {"uplink": "topk", "downlink": "topk"},
    "int4+topk": {"uplink": "int4", "downlink": "topk"},
    "secagg": {"secure_agg": True},
    "secagg+topk": {"secure_agg": True, "downlink": "topk"},
    "async-fp32": {"async_buffer": 2},
    "async-int8": {"async_buffer": 2, "uplink": "int8"},
    "async-topk": {"async_buffer": 2, "uplink": "topk"},
}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def record(tmp_path, kw):
    """every ``(request, reply)`` each of the two devices served in a two-round remote training with the settings ``kw``"""
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.control.workers import WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw

    class Recorder(WorkerServer):
        def _dispatch(self, req):
            resp = super()._dispatch(req)
            self.frames.append((req, resp))
            return resp

    workers = []
    for i in range(2):
        w = Recorder(f"dev-{i}", "127.0.0.1", _free_port(), device=torch.device("cpu"))
        w.frames = []
        w.add_dataset(BaseDataset(*synthetic_unsw(256, seed=i + 1)))
        w.start(block=False)
        workers.append(w)
    try:
        torch.manual_seed(0)
        args = Arguments(model="ffnn", lr=0.1, batch_size=16, federate_after_n_batches=30, synthetic=64, uplink_topk=8,
                         downlink_topk=8, secagg_clip=0.5, **kw)
        broker, clock = InProcessBroker(), FakeClock()
        c = Coordinator(1, True, 2, False, False, args=args, broker=broker, timer_factory=clock, path=str(tmp_path / "test.pth"),
                        device=torch.device("cpu"), evaluate_after=False, fit_timeout=60)
        c.connect()
        c.subscribe("topic/state")
        pub = BusClient("pub", broker=broker)
        pub.connect()
        for w in workers:
            pub.publish("topic/state", f"(127.0.0.1, {w.port}, TRAINING)")
        c.drain()
        clock.advance(1.0)
        res = c.windower.last_result
        assert res is not None and res["dropped"] == [], res
    finally:
        for w in workers:
            w.stop()
    return [w.frames for w in workers]


def _lengths(v):
    """the lengths of the bytes in ``v``, in its shape (None: ``v`` holds no bytes)"""
    if isinstance(v, bytes):
        return len(v)
    if isinstance(v, dict):
        out = {k: _lengths(x) for k, x in v.items()}
        return {k: x for k, x in out.items() if x is not None} or None
    if isinstance(v, list):
        out = [_lengths(x) for x in v]
        return out if any(x is not None for x in out) else None
    return None


def summary(kw, frames):
    """per device, what the fixture pins of its frames"""
    out = []
    for served in frames:
        got = []
        for req, resp in served:
            f = {"op": req.get("op"), "request": list(req), "reply": list(resp),
                 "request_bytes": _lengths(req) or {}, "reply_bytes": _lengths(resp) or {}}
            if "async_buffer" not in kw or f not in got:
                got.append(f)
        out.append(got)
    return out


@pytest.mark.parametrize("name", list(RUNS))
def test_fit_wire_is_pinned(tmp_path, name):
    with open(GOLDEN) as fh:
        want = json.load(fh)[name]
    assert summary(RUNS[name], record(tmp_path, RUNS[name])) == want


if __name__ == "__main__":
    import pathlib
    import tempfile
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    golden = {}
    for name, kw in RUNS.items():
        with tempfile.TemporaryDirectory() as d:
            golden[name] = summary(kw, record(pathlib.Path(d), kw))
    with open(GOLDEN, "w") as fh:
        json.dump(golden, fh, indent=1)
        fh.write("\n")
