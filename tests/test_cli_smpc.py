"""CLI flag parity + an end-to-end run of the real CLIs over the TCP bus; SMPC numerics."""
import os
import socket
import subprocess
import sys
import time

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_coordinator_cli_flags_match_reference():
    import federated_coordinator as fc
    ns = fc.build_parser().parse_args(["-t", "topic/state"])
    assert (ns.port, ns.host, ns.window, ns.federated_round, ns.remote, ns.encryption, ns.iot) == \
        (1883, "localhost", 1, 1, False, False, False)
    ns = fc.build_parser().parse_args(["-p", "1999", "--host", "h", "-t", "x", "-r", "-w", "3", "-e", "-f", "6", "-i"])
    assert (ns.port, ns.host, ns.topic, ns.remote, ns.window, ns.encryption, ns.federated_round, ns.iot) == \
        (1999, "h", "x", True, 3, True, 6, True)
    with pytest.raises(SystemExit):
        fc.build_parser().parse_args([])                # --topic is required


def test_worker_cli_flags_match_reference():
    import remote_worker as rw
    ns = rw.build_parser().parse_args(["--host", "127.0.0.1", "-b", "localhost", "-t", "topic/state"])
    assert (ns.port, ns.wait, ns.event, ns.training, ns.inference, ns.verbose) == (8777, 5, "TRAINING", None, None, False)
    ns = rw.build_parser().parse_args(["--host", "1.2.3.4", "-p", "8778", "-b", "b", "-t", "t", "-w", "1", "-e", "INFERENCE",
                                       "-dt", "a.csv", "-di", "b.csv", "-v"])
    assert (ns.port, ns.event, ns.training, ns.inference, ns.verbose) == (8778, "INFERENCE", "a.csv", "b.csv", True)
    for missing in (["-b", "b", "-t", "t"], ["--host", "h", "-t", "t"], ["--host", "h", "-b", "b"]):
        with pytest.raises(SystemExit):
            rw.build_parser().parse_args(missing)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_real_clis_remote_training_end_to_end(tmp_path):
    """README flow: coordinator -r, two remote_worker.py processes on 127.0.0.1, 2 rounds → test.pth."""
    bport, w1, w2 = _free_port(), _free_port(), _free_port()
    ckpt = str(tmp_path / "test.pth")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    coord = subprocess.Popen([sys.executable, os.path.join(ROOT, "federated_coordinator.py"), "-t", "topic/state", "-r",
                              "-w", "2", "-f", "2", "-p", str(bport), "--embedded-broker", "--checkpoint", ckpt,
                              "--max-batches", "20", "--exit-after", "1", "--no-cuda",
                              "--round-log", str(tmp_path / "round.txt")],
                             env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    workers = []
    try:
        time.sleep(4.0)
        for port in (w1, w2):
            workers.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "remote_worker.py"), "--host", "127.0.0.1",
                                             "-p", str(port), "-b", "127.0.0.1", "--broker-port", str(bport), "-t", "topic/state",
                                             "-w", "1", "--synthetic", "64", "--no-cuda"], env=env,
                                            stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL))
        out, _ = coord.communicate(timeout=120)
        assert coord.returncode == 0, out[-2000:]
        assert os.path.exists(ckpt)
        state = torch.load(ckpt, weights_only=True)
        assert state["fc4.weight"].shape == (1, 10)
        log = open(tmp_path / "round.txt").read()
        assert "Testing round on: 20" in log and "Time round 1 :" in log and "Total training time:" in log
        assert log.count("Loss for worker id: 127.0.0.1:") == 4
    finally:
        for w in workers:
            w.kill()
        if coord.poll() is None:
            coord.kill()


def test_killed_worker_is_withdrawn_through_its_mqtt_last_will(tmp_path):
    """Failure detection on the control plane: ``remote_worker.py`` registers a NOT_READY last-will with the broker;
    SIGKILL-ing it after it announced TRAINING makes the (in-test) MQTT broker publish the will, and a Coordinator
    listening through the same broker drops the device before the window closes."""
    from colearn_federated_learning_b200 import settings
    from colearn_federated_learning_b200.control.bus import TcpBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock

    wport = _free_port()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    with TcpBroker(port=0) as tb:
        clock = FakeClock()
        c = Coordinator(30, True, 1, False, False, transport="tcp", timer_factory=clock, path=str(tmp_path / "t.pth"),
                        device=torch.device("cpu"))
        c.connect(tb.host, tb.port)
        c.subscribe("topic/state")
        c.loop_start()
        w = subprocess.Popen([sys.executable, os.path.join(ROOT, "remote_worker.py"), "--host", "127.0.0.1", "-p", str(wport),
                              "-b", "127.0.0.1", "--broker-port", str(tb.port), "-t", "topic/state", "-w", "1",
                              "--synthetic", "16", "--no-cuda"], env=env, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        try:
            ident = f"127.0.0.1:{wport}"
            deadline = time.time() + 60
            while ident not in settings.training_devices and time.time() < deadline:
                time.sleep(0.05)
            assert ident in settings.training_devices and c.windower.state == "COLLECTING"
            w.kill()                                             # no DISCONNECT: the broker fires the will
            deadline = time.time() + 20
            while ident in settings.training_devices and time.time() < deadline:
                time.sleep(0.05)
            assert ident not in settings.training_devices and ident not in c.known_workers
            clock.advance(30.0)                                  # window closes with nobody left: no training
            assert c.trainings_done == 0
        finally:
            if w.poll() is None:
                w.kill()
            c.shutdown()
            c.disconnect()


# ---- SMPC -------------------------------------------------------------------------------------------------------
def test_fixed_point_and_sharing_roundtrip():
    from colearn_federated_learning_b200.smpc import CryptoProvider, fix_precision, float_precision, share
    x = torch.tensor([[0.1234, -5.5], [3.0, 0.0004]])
    fx = fix_precision(x)
    assert fx.dtype == torch.int64 and fx.tolist() == [[123, -5500], [3000, 0]]          # round(x * 10^3)
    s = share(fx, CryptoProvider(1))
    assert not torch.equal(s.shares[0], fx) and torch.equal(s.get(), fx)
    assert torch.equal(s.refresh().get(), fx)
    assert torch.allclose(float_precision(s.get()), torch.round(x * 1000) / 1000)


def test_beaver_matmul_and_mul_are_correct():
    from colearn_federated_learning_b200.smpc import CryptoProvider, fix_precision, float_precision, share
    p = CryptoProvider(2)
    a, b = torch.randn(4, 6), torch.randn(6, 3)
    c = float_precision(share(fix_precision(a), p).matmul(share(fix_precision(b), p)).truncate().get())
    assert (c - a @ b).abs().max() < 0.02
    u, v = torch.randn(5), torch.randn(5)
    w = float_precision(share(fix_precision(u), p).mul(share(fix_precision(v), p)).truncate().get())
    assert (w - u * v).abs().max() < 0.01
    bits = share(fix_precision(u), p).positive_bit().get()
    assert bits.tolist() == (fix_precision(u) > 0).long().tolist()
    assert p.triples_dealt == 2 and p.comparisons == 1


def test_encrypted_training_tracks_plaintext_training():
    from colearn_federated_learning_b200.models import FFNN
    from colearn_federated_learning_b200.smpc import CryptoProvider, SharedMLP, fix_precision, float_precision, share
    torch.manual_seed(0)
    m = FFNN()
    p = CryptoProvider(3)
    sm = SharedMLP.from_module(m, p)
    x, y = torch.rand(1, 10), torch.ones(1, 1)
    losses = [float(float_precision(sm.step(share(fix_precision(x), p), share(fix_precision(y), p), 0.1).get()))
              for _ in range(25)]
    assert losses[-1] < losses[0] * 0.7
    before = torch.cat([q.detach().reshape(-1) for q in m.parameters()]).clone()
    sm.reveal_into(m)
    after = torch.cat([q.detach().reshape(-1) for q in m.parameters()])
    assert not torch.equal(before, after) and (m(x) > 0.5).all()


def _closed_windows(stderr: str):
    """[(sorted members, sorted selected), ...] of the 'window closed:' log lines (devices register in arrival order)."""
    import ast
    import re
    out = []
    for ln in stderr.splitlines():
        m = re.search(r"window closed: members=(\[.*?\]) selected=(\[.*?\])", ln)
        if m:
            out.append((sorted(ast.literal_eval(m.group(1))), sorted(ast.literal_eval(m.group(2)))))
    return out


def test_box_mode_cli_two_ranks_gloo(tmp_path):
    """``federated_coordinator.py --box`` under torchrun: rank 0 runs parser/window/selection on the in-process bus,
    both ranks train, rank 0 writes the reference-format checkpoint (CPU/gloo stand-in for the fused GPU path)."""
    ckpt = str(tmp_path / "test.pth")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    # each rank announces TRAINING once it has started, and the first announcement opens the window: on a loaded machine the
    # second rank can start more than a second after the first, so the window is long enough for both to be in it
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                          "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "federated_coordinator.py"),
                          "-t", "topic/state", "--box", "--model", "mlp", "--synthetic", "128", "-f", "2", "--weighted",
                          "-w", "10", "--checkpoint", ckpt, "--batch-size", "4", "--exit-after", "1"], env=env, capture_output=True, text=True,
                         timeout=240, cwd=str(tmp_path))
    assert out.returncode == 0, out.stderr[-2000:]
    assert _closed_windows(out.stderr) == [(["10.0.0.1:8777", "10.0.0.2:8778"],) * 2]     # (members, selected), arrival order ignored
    assert out.stderr.count("Loss for worker id: 10.0.0.") == 4
    state = torch.load(ckpt, weights_only=True)
    assert state["fc1.weight"].shape == (64, 10) and state["fc3.weight"].shape == (2, 64)


def test_box_mode_is_a_coordinator_service(tmp_path):
    """``--box`` serves window after window like the reference coordinator (fc.py:294-300): devices ask again after a
    training, NOT_READY withdraws one from the open window, a withdrawn device that announces later rides the next window,
    INFERENCE runs the global model on the asking rank's tagged rows, ``--evaluate`` scores every trained model, and the
    job ends after ``--exit-after`` trainings."""
    ckpt = str(tmp_path / "test.pth")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                          "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "federated_coordinator.py"),
                          "-t", "topic/state", "--box", "--model", "ffnn", "--synthetic", "64", "-w", "1", "--checkpoint", ckpt,
                          "--batch-size", "4", "--exit-after", "3", "--evaluate",
                          "--box-script", "1:NOT_READY:1,1:INFERENCE:1,1:TRAINING:2"], env=env, capture_output=True, text=True,
                         timeout=300, cwd=str(tmp_path))
    assert out.returncode == 0, out.stderr[-3000:]
    both, only0 = ["10.0.0.1:8777", "10.0.0.2:8778"], ["10.0.0.1:8777"]
    assert _closed_windows(out.stderr) == [(both, both), (only0, only0), (both, both)], out.stderr[-3000:]
    assert "10.0.0.2:8778 is not ready anymore" in out.stderr
    inf = [ln for ln in out.stderr.splitlines() if "inference on 10.0.0.2:8778: [" in ln]
    assert len(inf) == 1 and inf[0].count(",") == 4                              # 5 tagged rows -> 5 predictions
    assert out.stderr.count("Loss evaluation global model after training") == 3
    assert torch.load(ckpt, weights_only=True)["fc4.weight"].shape == (1, 10)


def test_box_mode_encrypted_demo_on_three_ranks(tmp_path):
    """``--box -e``: rank 0 = coordinator + crypto provider (dealer), ranks 1 and 2 = the share holders.  One window admits the
    devices, the model and the first N samples are secret-shared out, SGD runs on shares (the per-multiplication opens travel
    between the two share holders), the coordinator reconstructs and saves the model (reference fc.py:394-472)."""
    ckpt = str(tmp_path / "test.pth")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "3", "--master-addr",
                          "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "federated_coordinator.py"),
                          "-t", "topic/state", "--box", "-e", "--model", "ffnn", "--synthetic", "64", "-w", "1", "--checkpoint", ckpt,
                          "--batch-size", "4", "--enc-items", "32", "--log-interval", "4"], env=env, capture_output=True, text=True,
                         timeout=300, cwd=str(tmp_path))
    assert out.returncode == 0, out.stderr[-3000:]
    assert out.stderr.count("share holder 0:") == 1 and out.stderr.count("share holder 1:") == 1 and "336 opens" in out.stderr   # 8 batches x 42 opens
    assert "168 Beaver triples, 24 comparisons" in out.stderr
    state = torch.load(ckpt, weights_only=True)
    assert state["fc1.weight"].shape == (50, 10) and all(torch.isfinite(v).all() for v in state.values())
    # same training in one process (both shares side by side): same fixed-point result up to the +-1 ulp of the probabilistic
    # truncation (which depends on the share randomness)
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw
    from colearn_federated_learning_b200.fl.encrypted import train_encrypted
    from colearn_federated_learning_b200.models import build_model, flatten_params
    a = Arguments()
    a.batch_size, a.n_train_items_enc, a.log_interval, a.seed = 4, 32, 4, 1
    torch.manual_seed(a.seed)
    ref = build_model("ffnn")
    init = flatten_params(ref).clone()
    x, y = synthetic_unsw(64, seed=a.seed)
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        train_encrypted(ref, BaseDataset(x, y), ["10.0.0.2", "10.0.0.3"], a)
    got = build_model("ffnn")
    got.load_state_dict(state)
    d_box, d_ref = flatten_params(got) - init, flatten_params(ref) - init
    assert float(d_ref.abs().max()) > 1e-3 and float((d_box - d_ref).abs().max()) < 5e-3, (float(d_ref.abs().max()), float((d_box - d_ref).abs().max()))


def test_box_mode_metrics_jsonl_and_periodic_checkpoints(tmp_path):
    """``--metrics`` / ``--save-every`` in box mode: one JSONL record per round with the fields SURVEY §5 lists
    (selection, n_k, loss_k, device time as max over ranks, bytes of both collective legs, GB/s, link-roofline
    fraction) and a checkpoint that exists before the last round finishes."""
    import json
    ckpt, metrics = str(tmp_path / "test.pth"), str(tmp_path / "rounds.jsonl")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                          "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "federated_coordinator.py"),
                          "-t", "topic/state", "--box", "--model", "mlp", "--synthetic", "96", "-f", "3", "-w", "1",
                          "--checkpoint", ckpt, "--batch-size", "8", "--metrics", metrics, "--save-every", "1", "--dtype", "bf16",
                          "--exit-after", "1"],
                         env=env, capture_output=True, text=True, timeout=240, cwd=str(tmp_path))
    assert out.returncode == 0, out.stderr[-2000:]
    recs = [json.loads(l) for l in open(metrics)]
    assert [r["round"] for r in recs] == [0, 1, 2]
    for r in recs:
        assert r["selected"] == ["10.0.0.1:8777", "10.0.0.2:8778"] and r["n_k"] == [48, 48] and len(r["loss_k"]) == 2
        assert r["t_round_max_over_ranks_ms"] > 0 and r["bytes_bcast"] == r["bytes_reduce"] == 2 * 4 * 4994
        assert 0 < r["roofline_frac"] < 1 and r["GBps"] > 0 and r["link_time_lower_bound_ms"] > 0
    assert out.stderr.count("checkpoint after round") == 2 and out.stderr.count("Time round") == 3
    assert torch.load(ckpt, weights_only=True)["fc1.weight"].shape == (64, 10)


def test_save_every_in_remote_mode(tmp_path):
    """``--save-every`` on the classic coordinator: the checkpoint (marked partial in its sidecar) exists while
    later rounds are still running."""
    from colearn_federated_learning_b200.control.arguments import Arguments
    from colearn_federated_learning_b200.control.bus import BusClient, InProcessBroker
    from colearn_federated_learning_b200.control.coordinator import Coordinator
    from colearn_federated_learning_b200.control.window import FakeClock
    from colearn_federated_learning_b200.utils.checkpoint import load_meta

    broker, clock = InProcessBroker(), FakeClock()
    a = Arguments()
    a.synthetic, a.save_every, a.model, a.batch_size = 48, 1, "mlp", 8
    seen = []

    class Spy(Coordinator):
        def _maybe_checkpoint(self, model, theta, r, meta):
            super()._maybe_checkpoint(model, theta, r, meta)
            if os.path.exists(self.path):
                seen.append((r, load_meta(self.path).get("partial", False), load_meta(self.path).get("rounds")))

    c = Spy(1, False, 3, False, False, args=a, broker=broker, timer_factory=clock, path=str(tmp_path / "t.pth"),
            device=torch.device("cpu"))
    c.connect()
    c.subscribe("topic/state")
    pub = BusClient("pub", broker=broker)
    pub.connect()
    pub.publish("topic/state", "(192.168.1.7, TRAINING)")
    pub.publish("topic/state", "(192.168.1.8, TRAINING)")
    c.drain()
    clock.advance(1.0)
    assert seen[:2] == [(0, True, 1), (1, True, 2)]            # rounds 1 and 2 left partial checkpoints behind
    meta = load_meta(c.path)
    assert meta["rounds"] == 3 and not meta.get("partial", False)


def test_bench_paper_experiment_runs_end_to_end():
    """``bench.py --config paper``: the reference's published experiment (12 rounds x 1000 it, 2 remote worker
    processes over TCP, FFNN + BCE) through the real coordinator and ``remote_worker.py`` — one JSON line, rounds/s
    far above the published 0.1133 (2 x RPi 3B+)."""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--config", "paper", "--steps", "1", "--warmup", "3"],
                       capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-2000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1]
    out = json.loads(line)
    assert out["config"]["name"] == "paper" and out["config"]["rounds_per_training"] == 12 and out["config"]["workers"] == 2
    assert out["unit"] == "rounds/s" and out["value"] > 1.0 and out["vs_baseline"] > 8
    assert len(out["config"]["final_losses"]) == 2


def test_plugin_registers_model_and_dataset_for_both_clis(tmp_path):
    """The reference's "use your own model/dataset" (README.md:119-169) without editing sources: a plugin registers a
    new architecture and a dataset adapter; the coordinator CLI trains it in VirtualWorker mode, a worker hosts it."""
    import math
    import subprocess
    import sys

    import torch

    from colearn_federated_learning_b200.data import DATASET_REGISTRY, load_dataset, register_dataset
    from colearn_federated_learning_b200.models import MODEL_REGISTRY, build_model, load_plugins, register_model

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    plugin = os.path.join(root, "examples", "my_plugin.py")
    csv_path = tmp_path / "moons.csv"
    g = torch.Generator().manual_seed(0)
    with open(csv_path, "w") as f:
        for i in range(200):
            lab = i % 2
            a = float(torch.rand(1, generator=g)) * math.pi
            x0 = math.cos(a) + (1.0 if lab else 0.0) + 0.05 * float(torch.randn(1, generator=g))
            x1 = (math.sin(a) if not lab else 0.5 - math.sin(a)) + 0.05 * float(torch.randn(1, generator=g))
            f.write(f"{x0:.5f},{x1:.5f},{lab}\n")
    # registry API
    assert load_plugins([plugin]) and "tiny_mlp" in MODEL_REGISTRY and "two_moons_csv" in DATASET_REGISTRY
    assert build_model("tiny_mlp").spec.dims == (2, 16, 16, 2)
    assert len(load_dataset("two_moons_csv", str(csv_path))) == 200
    with pytest.raises(ValueError):
        register_model("tiny_mlp", lambda: None)                       # duplicate without overwrite
    with pytest.raises(ValueError):
        register_dataset("unsw", lambda p: None)
    with pytest.raises(ValueError):
        load_dataset("nope", "x")
    # coordinator CLI: VirtualWorker mode on the plugin's model + dataset, driven by two bus events
    ckpt = tmp_path / "plug.pth"
    import socket
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    coord = subprocess.Popen([sys.executable, os.path.join(root, "federated_coordinator.py"), "-t", "topic/state", "-w", "1", "-p", str(port),
                              "--host", "127.0.0.1", "--embedded-broker", "--exit-after", "1", "--plugin", plugin, "--model", "tiny_mlp",
                              "--dataset", "two_moons_csv", "--test-path", str(csv_path), "--checkpoint", str(ckpt), "--no-cuda", "--lr", "0.05"],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        from colearn_federated_learning_b200.control.bus import BusClient
        import time
        deadline = time.time() + 60
        pub = BusClient("plug-pub", transport="tcp")
        while True:
            try:
                pub.connect("127.0.0.1", port)
                break
            except OSError:
                assert time.time() < deadline and coord.poll() is None, "coordinator did not come up"
                time.sleep(0.2)
        pub.loop_start()
        pub.publish("topic/state", "(192.168.1.7, TRAINING)")
        pub.publish("topic/state", "(192.168.1.8, TRAINING)")
        out, _ = coord.communicate(timeout=120)
        pub.loop_stop()
    finally:
        if coord.poll() is None:
            coord.kill()
    assert coord.returncode == 0, out[-3000:]
    sd = torch.load(str(ckpt))
    assert list(sd) == ["fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc3.weight", "fc3.bias"] and sd["fc1.weight"].shape == (16, 2)
    # worker CLI accepts the same plugin / dataset flags
    import remote_worker
    ns = remote_worker.build_parser().parse_args(["--host", "127.0.0.1", "-b", "x", "-t", "t", "--plugin", plugin, "--dataset", "two_moons_csv",
                                                  "-dt", str(csv_path)])
    ds = remote_worker.pick_dataset(ns)
    assert len(ds) == 200 and ds.data.shape[1] == 2


def test_worker_reannounce_joins_consecutive_trainings(tmp_path):
    """``remote_worker.py --reannounce S``: the coordinator deregisters a device after each training (fc.py:386-392), so
    a device that announces once only ever takes part in one; with ``--reannounce`` it is back for the next window.  Two
    trainings complete with one long-running worker process and nobody publishing by hand."""
    bport, wport = _free_port(), _free_port()
    ckpt = str(tmp_path / "test.pth")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=ROOT)
    coord = subprocess.Popen([sys.executable, os.path.join(ROOT, "federated_coordinator.py"), "-t", "topic/state", "-r", "-w", "1",
                              "-p", str(bport), "--host", "127.0.0.1", "--embedded-broker", "--exit-after", "2", "--no-cuda",
                              "--checkpoint", ckpt], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    worker = subprocess.Popen([sys.executable, os.path.join(ROOT, "remote_worker.py"), "--host", "127.0.0.1", "-p", str(wport), "-b", "127.0.0.1",
                               "--broker-port", str(bport), "-t", "topic/state", "-w", "3", "--reannounce", "1.5", "--synthetic", "64",
                               "--no-cuda"], env=env, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    try:
        out, _ = coord.communicate(timeout=120)
    finally:
        worker.terminate()
        worker.wait(timeout=10)
        if coord.poll() is None:
            coord.kill()
    assert coord.returncode == 0, out[-3000:]
    assert out.count("Total training time") == 2 and os.path.exists(ckpt)
