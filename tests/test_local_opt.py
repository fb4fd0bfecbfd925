"""Local optimizers of the device fit (fl/local_opt.py, ops/csrc/local_opt.cuh, the optimizer instances of
ops/csrc/mlp_persistent_opt.cu): the per-element step against ``reference.local_opt_step`` bit for bit; the reference against
``torch.optim``; the optimizer instances on the SIMT build and the host executor's generic loop against a float64 replay of
the reference, at the edges test_mlp_kernel_edges.py uses; plain SGD routed to the kernels of before; the wire form; every
refusal; and local and remote trainings with Adam.

The float64 bound is test_mlp_kernel_edges.py's bound for long fits: ``‖Δ − Δ64‖∞ ≤ C·‖Δ32 − Δ64‖∞ + 2⁻²⁰·‖Δ64‖∞`` with Δ32 the
float32 reference, which runs the same optimizer recurrence in float32 and differs from the kernel only in the order of the
additions inside the gradient.
"""
import math

import numpy as np
import pytest
import torch

import test_class_weight as CWT
import test_mlp_kernel_edges as E
from colearn_federated_learning_b200.fl.local_opt import LocalOpt, from_request
from colearn_federated_learning_b200.ops import reference as R

simt = E.simt
LR = E.LR
LR_ADAM = float(np.float32(0.005))   # Adam steps every parameter by about lr: 0.05 would make a fit of a few hundred steps chaotic


def _lr(lo):
    return LR_ADAM if lo.kind == "Adam" else LR
# name -> (net kind, dims, output activation, loss)
NETS = {"ffnn": (0, (10, 50, 30, 10, 1), "sigmoid", "bce"), "mlp": (1, (10, 64, 64, 2), "none", "xent"),
        "testing_remote": (2, (2, 50, 10, 1), "none", "sse"), "autoencoder": (3, (10, 32, 4, 32, 10), "none", "mse"),
        "ffnn_category": (4, (10, 50, 30, 10, 5), "none", "xent")}
OPTS = {"momentum": LocalOpt("SGD", momentum=0.9), "nesterov_wd": LocalOpt("SGD", momentum=0.5, nesterov=True, weight_decay=0.01),
        "wd": LocalOpt("SGD", weight_decay=0.05), "adam": LocalOpt("Adam"),
        "adam_wd": LocalOpt("Adam", betas=(0.8, 0.99), eps=1e-6, weight_decay=0.02)}
# The whole fits against the float64 replay run Adam at eps 1e-3.  Adam's step is scale-invariant: a gradient entry that sums to
# 0 in one order of additions and to a rounding residue in another moves its parameter by a full lr step in one executor and
# not at all in the other, which no rounding bound covers.  At eps 1e-3 such a residue moves it by about lr · residue / eps.
# The step itself, at every eps, is held to the bit by test_step_bits_match_the_reference.
FIT_OPTS = {**OPTS, "adam": LocalOpt("Adam", eps=1e-3), "adam_wd": LocalOpt("Adam", betas=(0.8, 0.99), eps=1e-3, weight_decay=0.02)}


def _theta0(net):
    from colearn_federated_learning_b200.models import build_model, flatten_params
    torch.manual_seed(NETS[net][0] + 3)
    return flatten_params(build_model(net)).clone()


def _data(net, n, seed=0):
    _, dims, _, loss = NETS[net]
    g = torch.Generator().manual_seed(700 + 19 * n + seed)
    x = torch.rand(n, dims[0], generator=g)
    if loss == "xent":
        y = torch.randint(0, dims[-1], (n, 1), generator=g).float()
    elif loss == "mse":
        y = x.clone()
    else:
        y = (torch.rand(n, dims[-1], generator=g) > 0.5).float()
    return x, y


def _replay(net, theta0, x, y, perm, B, epochs, max_b, lo, dtype):
    """The reference fit step by step: (θ, [loss of every step])"""
    _, dims, act, loss = NETS[net]
    th = theta0.to(dtype).clone()
    x, y = x.to(dtype), y.to(dtype)
    state = R.local_opt_state(th)
    losses, it = [], 0
    for e in range(epochs):
        order = perm[e % perm.shape[0]].long()
        for s in range(0, x.shape[0], B):
            idx = order[s:s + B]
            value, g = R.mlp_grad(th, dims, x[idx], y[idx], loss, act)
            R.local_opt_step(th, g, lo, _lr(lo), state)
            losses.append(float(value))
            it += 1
            if 0 < max_b <= it:
                return th, losses
    return th, losses


def _check(tag, net, got, got_losses, theta0, x, y, perm, B, epochs, max_b, lo):
    if x.shape[0] == 0:
        assert torch.equal(got, theta0) and got_losses.tolist() == [0.0, 0.0], tag
        return
    o64 = _replay(net, theta0, x, y, perm, B, epochs, max_b, lo, torch.float64)
    r32 = _replay(net, theta0, x, y, perm, B, epochs, max_b, lo, torch.float32)
    CWT._check(tag, got, got_losses, theta0, o64, r32)


def _simt_fit(sim, net, clients, B, epochs, max_b, lo, out_scales=None, delta=False, flags=None, perm_seed=0, perm_row0=0):
    kind, _, _, loss = NETS[net]
    theta_in = clients[0]["theta_in"]
    outs = [torch.full_like(theta_in, 7.0) for _ in clients]
    losses = sim.m.mlp_local_sgd_opt(kind, theta_in, outs, [c["x"] for c in clients], [c["y"] for c in clients],
                                     [c.get("perm") for c in clients], B, epochs, max_b, E.LOSS_CODES[loss], _lr(lo),
                                     out_scales or [1.0] * len(clients), delta, flags, perm_seed, perm_row0, lo.launch_args())
    return torch.stack(outs), losses


def _client(net, n, epochs, seed=0):
    x, y = _data(net, n, seed)
    return dict(x=x, y=y, perm=E._perm(n, epochs, seed=11 + seed), theta_in=_theta0(net))


# ---- the per-element step ------------------------------------------------------------------------------------------------
SPECIAL = [0.0, -0.0, 1e-40, -1e-40, 1.4e-45, 3e38, -3e38, 1e-20, 0.5, -2.0, float("nan"), float("inf"), 1e30]


@pytest.mark.parametrize("name", sorted(OPTS) + ["plain"])
def test_step_bits_match_the_reference(simt, name):
    """local_opt.cuh (SIMT build, over arrays) equals reference.local_opt_step bit for bit over 6 steps, from the first one,
    for 0, ±0, subnormal, large, NaN and infinite gradients and parameters"""
    lo = OPTS.get(name, LocalOpt())
    rng = np.random.default_rng(4)
    n = 600
    theta = torch.tensor(rng.standard_normal(n) * 0.3, dtype=torch.float32)
    theta[:len(SPECIAL)] = torch.tensor(SPECIAL)
    g = torch.tensor(rng.standard_normal((6, n)), dtype=torch.float32)
    sp = torch.tensor(SPECIAL, dtype=torch.float32)
    for s in range(6):
        g[s, 20:20 + len(SPECIAL)] = sp.roll(s)
        g[s, 40:40 + len(SPECIAL)] = sp
    th_k, m_k, v_k = theta.clone(), torch.zeros(n), torch.zeros(n)
    simt.m.local_opt_steps(th_k, g, m_k, v_k, LR, lo.launch_args())
    th_r = theta.clone()
    state = R.local_opt_state(th_r)
    for s in range(6):
        R.local_opt_step(th_r, g[s], lo, LR, state)

    def same(a, b):
        return bool(((a.view(torch.int32) == b.view(torch.int32)) | (torch.isnan(a) & torch.isnan(b))).all())
    assert same(th_k, th_r), (name, (th_k - th_r).abs().nan_to_num().max())
    if lo.kind == "Adam" or lo.momentum:
        assert same(m_k, state["m"]), name
    if lo.kind == "Adam":
        assert same(v_k, state["v"]), name


@pytest.mark.parametrize("name,opt_cls,kw", [
    ("momentum", torch.optim.SGD, dict(momentum=0.9)),
    ("nesterov_wd", torch.optim.SGD, dict(momentum=0.5, nesterov=True, weight_decay=0.01)),
    ("wd", torch.optim.SGD, dict(weight_decay=0.05)),
    ("adam", torch.optim.Adam, dict()),
    ("adam_wd", torch.optim.Adam, dict(betas=(0.8, 0.99), eps=1e-6, weight_decay=0.02))])
def test_reference_agrees_with_torch_optim(name, opt_cls, kw):
    """reference.mlp_local_sgd(local_opt=...) against torch.optim on an MLPNet over 300 batch-4 steps (Adam at lr 1e-3, where
    its steps are not sign-like): within 1e-3 of the largest update (float32; the two differ in how they round the bias
    corrections, the moment updates and the gradient)"""
    lr = 1e-3 if opt_cls is torch.optim.Adam else LR
    from colearn_federated_learning_b200.models import build_model, flatten_params
    torch.manual_seed(1)
    model = build_model("mlp")
    flat = flatten_params(model).clone()
    x, y = _data("mlp", 1200, 1)
    perm = R.make_permutation(1200, 1, 3)
    theta0 = flat.clone()
    R.mlp_local_sgd(flat, (10, 64, 64, 2), x, y, perm, 4, lr, 1, -1, "xent", "none", None, OPTS[name])
    opt = opt_cls(model.parameters(), lr=lr, **kw)
    order = perm[0].long()
    for s in range(0, 1200, 4):
        idx = order[s:s + 4]
        opt.zero_grad()
        torch.nn.functional.cross_entropy(model(x[idx]), y[idx].view(-1).long()).backward()
        opt.step()
    ref = flatten_params(model)
    err = (ref - flat).abs().max().item()
    upd = (flat - theta0).abs().max().item()
    assert upd > 1e-2 and err <= 1e-3 * upd, (name, err, upd)


# ---- the optimizer instances on the SIMT build ---------------------------------------------------------------------------
@pytest.mark.parametrize("net", sorted(NETS))
@pytest.mark.parametrize("opt", ["nesterov_wd", "adam_wd"])
@pytest.mark.parametrize("B,n", [(1, 65), (1, 129), (7, 30), (4, 9)])
def test_instances_match_the_reference_cpu(simt, net, opt, B, n):
    """batch 1 across CHUNK boundaries, batches that end short, two epochs"""
    c = _client(net, n, 2)
    outs, losses = _simt_fit(simt, net, [c], B, 2, -1, FIT_OPTS[opt])
    _check(f"simt {net} {opt} B{B} n{n}", net, outs[0], losses[0], c["theta_in"], c["x"], c["y"], c["perm"], B, 2, -1, FIT_OPTS[opt])


@pytest.mark.parametrize("opt", ["momentum", "adam"])
@pytest.mark.parametrize("B,n,epochs,max_b", [(1, 20, 3, 13), (7, 30, 3, 6), (3, 10, 2, 100)])
def test_max_batches_cpu(simt, opt, B, n, epochs, max_b):
    for net in ("ffnn", "mlp"):
        c = _client(net, n, epochs)
        outs, losses = _simt_fit(simt, net, [c], B, epochs, max_b, FIT_OPTS[opt])
        _check(f"simt max_b {net} {opt}", net, outs[0], losses[0], c["theta_in"], c["x"], c["y"], c["perm"], B, epochs, max_b, FIT_OPTS[opt])


def test_in_kernel_shuffle_cpu(simt):
    """perm_seed / perm_row0: the kernel's own keyed order, the rows simt.table tabulates"""
    net, n, epochs, seed, row0 = "mlp", 70, 2, 987654321, 3
    c = _client(net, n, epochs)
    del c["perm"]
    outs, losses = _simt_fit(simt, net, [c], 1, epochs, -1, FIT_OPTS["adam"], perm_seed=seed, perm_row0=row0)
    perm = simt.m.feistel_permutation(n, row0 + epochs, seed)[row0:]
    _check("simt perm_seed", net, outs[0], losses[0], c["theta_in"], c["x"], c["y"], perm, 1, epochs, -1, FIT_OPTS["adam"])


@pytest.mark.parametrize("opt", ["momentum", "adam_wd"])
def test_out_scale_delta_empty_and_many_clients_cpu(simt, opt):
    """out_scale × delta_mode give fl(s·θ) / fl(s·(θ − θ_in)) of the scale-1 result; an empty shard writes s·θ_in (0 in delta
    mode) and {0, 0}; every flag is raised; every client of a launch is bit-identical to itself alone"""
    lo = FIT_OPTS[opt]
    for net in ("ffnn", "ffnn_category"):
        clients = [_client(net, n, 1, seed=i) for i, n in enumerate((0, 1, 64, 65))]
        base, base_l = _simt_fit(simt, net, clients, 3, 1, -1, lo)
        for k, c in enumerate(clients):
            alone, alone_l = _simt_fit(simt, net, [c], 3, 1, -1, lo)
            assert torch.equal(alone[0], base[k]) and torch.equal(alone_l[0], base_l[k]), (net, k)
            _check(f"simt clients {net}", net, base[k], base_l[k], c["theta_in"], c["x"], c["y"], c["perm"], 3, 1, -1, lo)
        theta0 = clients[0]["theta_in"]
        for delta in (False, True):
            for s in (0.37, -1.0):
                flags = torch.zeros(len(clients), dtype=torch.int32)
                outs, losses = _simt_fit(simt, net, clients, 3, 1, -1, lo, out_scales=[s] * len(clients), delta=delta, flags=flags)
                want = (base - theta0) if delta else base
                assert torch.equal(outs, torch.tensor(s, dtype=torch.float32) * want), (net, delta, s)
                assert torch.equal(losses, base_l)
                assert flags.tolist() == [7 + i for i in range(len(clients))]


# ---- host executor, routing ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", sorted(NETS))
@pytest.mark.parametrize("opt", ["nesterov_wd", "adam_wd"])
def test_host_executor_matches_the_reference(net, opt):
    from colearn_federated_learning_b200.ops import host
    if not host.available():
        pytest.skip("host executor not built")
    _, dims, act, loss = NETS[net]
    for B, n in ((1, 40), (5, 23)):
        c = _client(net, n, 2)
        th = c["theta_in"].clone()
        lo = FIT_OPTS[opt]
        res = host.mlp_local_sgd_multi(dims, act, [th], [c["x"]], [c["y"]], [c["perm"]], B, _lr(lo), 2, -1, loss, threads=1,
                                       local_opt=lo)
        _check(f"host {net} {opt} B{B}", net, th, res[0], c["theta_in"], c["x"], c["y"], c["perm"], B, 2, -1, lo)


def test_plain_sgd_routes_to_the_kernels_of_before(monkeypatch):
    """No optimizer, SGD with no arguments and SGD with explicit zeros all launch the plain binding with the same arguments,
    and train to the same bits on the CPU paths"""
    from colearn_federated_learning_b200.ops import fused_mlp
    calls = []

    class Ext:
        def mlp_local_sgd(self, *a):
            calls.append(("plain", a[0], a[3:]))

        def mlp_local_sgd_opt(self, *a):
            calls.append(("opt", a[0], a[3:]))
    monkeypatch.setattr(fused_mlp._ext, "require", lambda: Ext())
    for lo in (None, LocalOpt(), from_request("SGD", {}), from_request("SGD", {"momentum": 0.0, "weight_decay": 0.0, "nesterov": False,
                                                                           "dampening": 0, "maximize": False})):
        fused_mlp.mlp_local_sgd_multi((10, 50, 30, 10, 1), "sigmoid", None, 3, 1, 0.05, loss="bce", local_opt=lo)
    assert len(calls) == 4 and all(c == calls[0] for c in calls) and calls[0][0] == "plain"
    fused_mlp.mlp_local_sgd_multi((10, 50, 30, 10, 1), "sigmoid", None, 3, 1, 0.05, loss="bce", local_opt=OPTS["adam"])
    assert calls[-1][0] == "opt" and calls[-1][2][-1] == OPTS["adam"].launch_args()
    monkeypatch.undo()
    from colearn_federated_learning_b200 import ops
    c = _client("ffnn", 30, 1)
    outs = []
    for lo in (None, LocalOpt("SGD", momentum=0.0, weight_decay=0.0)):
        th = c["theta_in"].clone()
        ops.mlp_local_sgd(th, (10, 50, 30, 10, 1), c["x"], c["y"], c["perm"], 1, LR, 1, -1, "bce", "sigmoid", local_opt=lo)
        outs.append(th)
    assert torch.equal(outs[0], outs[1])


# ---- semantics, wire, refusals ------------------------------------------------------------------------------------------
def test_wire_form_and_default_request():
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    d = FitConfig().to_dict()
    assert "optimizer_args" not in d and d["optimizer"] == "SGD"
    assert FitConfig().with_local_opt(LocalOpt()).to_dict() == d
    cfg = FitConfig().with_local_opt(OPTS["adam_wd"])
    wire = cfg.to_dict()
    assert wire["optimizer"] == "Adam" and wire["optimizer_args"] == {"betas": [0.8, 0.99], "eps": 1e-6, "weight_decay": 0.02}
    assert FitConfig.from_dict(wire).local_opt() == OPTS["adam_wd"]
    assert FitConfig().with_local_opt(OPTS["nesterov_wd"]).local_opt() == OPTS["nesterov_wd"]
    assert LocalOpt().is_plain() and not OPTS["wd"].is_plain() and not OPTS["momentum"].is_plain() and not LocalOpt("Adam").is_plain()
    assert OPTS["adam"].record() == {"kind": "Adam", "betas": [0.9, 0.999], "eps": 1e-8, "weight_decay": 0.0}


@pytest.mark.parametrize("name,args,match", [
    ("RMSprop", {}, "unknown local optimizer"), ("sgd", {}, "unknown local optimizer"),
    ("SGD", {"lr": 0.1}, "unknown argument"), ("SGD", {"betas": [0.9, 0.9]}, "unknown argument"),
    ("Adam", {"momentum": 0.9}, "unknown argument"), ("SGD", {"momentum": 1.0}, r"\[0, 1\)"),
    ("SGD", {"momentum": -0.1}, r"\[0, 1\)"), ("SGD", {"momentum": float("nan")}, "finite"),
    ("SGD", {"nesterov": True}, "nesterov needs momentum"), ("SGD", {"weight_decay": -1e-3}, ">= 0"),
    ("SGD", {"weight_decay": float("inf")}, "finite"), ("SGD", {"dampening": 0.1}, "dampening"),
    ("SGD", {"maximize": True}, "maximize"), ("Adam", {"amsgrad": True}, "amsgrad"), ("Adam", {"betas": [0.9, 1.0]}, r"\[0, 1\)"),
    ("Adam", {"betas": [0.9]}, "two numbers"), ("Adam", {"eps": 0.0}, "> 0"), ("Adam", {"eps": "1e-8"}, "number"),
    ("SGD", {"momentum": True}, "number"), ("SGD", [0.9], "mapping"), (["SGD"], {}, "unknown local optimizer"),
    ({"kind": "Adam"}, {}, "unknown local optimizer"), (1, {}, "unknown local optimizer")])
def test_refusals(name, args, match):
    with pytest.raises(ValueError, match=match):
        from_request(name, args)


def test_trainers_without_optimizer_instances_refuse(monkeypatch):
    """The layer-wise MLP trainer, the conv-net trainer, the two-shot engine path and class weights refuse a non-plain
    optimizer before any launch"""
    from colearn_federated_learning_b200.fl import local_opt as L
    with pytest.raises(ValueError, match="layer-wise trainer of mlp_wide"):
        L.refuse_non_plain(OPTS["adam"], "the layer-wise trainer of mlp_wide")
    L.refuse_non_plain(LocalOpt(), "anything")
    from colearn_federated_learning_b200 import ops
    c = _client("ffnn", 10, 1)
    with pytest.raises(ValueError, match="class weights together with a local optimizer"):
        ops.mlp_local_sgd(c["theta_in"].clone(), (10, 50, 30, 10, 1), c["x"], c["y"], c["perm"], 1, LR, 1, -1, "bce", "sigmoid",
                          class_weights=[1.0, 2.0], local_opt=OPTS["adam"])
    from colearn_federated_learning_b200.parallel.engine import FederatedEngine
    with pytest.raises(ValueError, match="two-shot"):
        FederatedEngine("mlp", backend="cpu", device=torch.device("cpu"), algo="twoshot", local_opt=OPTS["adam"])


def test_conv_trainer_refuses_before_any_launch(monkeypatch):
    from colearn_federated_learning_b200.fl import convnet, trainer
    from colearn_federated_learning_b200.models import build_model, flatten_params
    monkeypatch.setattr(trainer, "conv_path", lambda device: "native")
    monkeypatch.setattr(convnet.ConvNetTrainer, "supports", staticmethod(lambda *a: True))
    monkeypatch.setattr(convnet.ConvNetTrainer, "cached", staticmethod(lambda *a: pytest.fail("launched")))
    model = build_model("resnet18")
    cfg = trainer.FitConfig(model="resnet18", loss="xent", batch_size=128).with_local_opt(OPTS["momentum"])
    with pytest.raises(ValueError, match="conv-net trainer of resnet18"):
        trainer.local_fit(flatten_params(model), model, torch.zeros(128, 3, 32, 32), torch.zeros(128, 1), cfg)


def test_torch_fit_builds_torch_optim():
    """A user-registered module trains through torch_fit with the torch.optim optimizer the config names"""
    from colearn_federated_learning_b200.fl.trainer import FitConfig, torch_fit
    torch.manual_seed(0)
    a = torch.nn.Sequential(torch.nn.Linear(4, 3))
    b = torch.nn.Sequential(torch.nn.Linear(4, 3))
    b.load_state_dict(a.state_dict())
    x, y = torch.rand(12, 4), torch.randint(0, 3, (12, 1)).float()
    cfg = FitConfig(model="custom", loss="xent", batch_size=3, lr=0.05).with_local_opt(OPTS["adam_wd"])
    torch_fit(a, x, y, cfg, None)
    opt = torch.optim.Adam(b.parameters(), lr=0.05, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.02)
    for s in range(0, 12, 3):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(b(x[s:s + 3]), y[s:s + 3].view(-1).long()).backward()
        opt.step()
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.equal(p, q)


def test_device_refuses_with_the_reason():
    from colearn_federated_learning_b200.control.workers import RemoteWorkerClient, WorkerServer
    from colearn_federated_learning_b200.data import BaseDataset, synthetic_unsw
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    from colearn_federated_learning_b200.models import build_model, flatten_params
    from test_fit_wire import _free_port
    w = WorkerServer("dev", "127.0.0.1", _free_port(), device=torch.device("cpu"))
    w.add_dataset(BaseDataset(*synthetic_unsw(32, seed=1)))
    w.start(block=False)
    try:
        c = RemoteWorkerClient("dev", "127.0.0.1", w.port)
        flat = flatten_params(build_model("ffnn"))
        for name, args, match in (("Adagrad", None, "unknown local optimizer"), ("SGD", {"momentum": 2.0}, r"\[0, 1\)"),
                                  (["SGD"], None, "unknown local optimizer"), ({"k": 1}, None, "unknown local optimizer"),
                                  ("Adam", {"amsgrad": True}, "amsgrad")):
            with pytest.raises(RuntimeError, match=match):
                c.fit(flat, FitConfig(model="ffnn", loss="bce", max_nr_batches=2, optimizer=name, optimizer_args=args))
        with pytest.raises(RuntimeError, match="class weights together"):
            c.fit(flat, FitConfig(model="ffnn", loss="bce", max_nr_batches=2, class_weights=[1.0, 2.0], optimizer="Adam"))
        assert w.fits_served == 0
        new, _, _ = c.fit(flat, FitConfig(model="ffnn", loss="bce", max_nr_batches=2, optimizer="Adam"))
        assert w.fits_served == 1 and not torch.equal(new, flat)
    finally:
        w.stop()


def test_cli_refusals_and_flags():
    import federated_coordinator as fc
    ns = fc.parse_cli(["-t", "t", "--local-optimizer", "Adam", "--local-betas", "0.8,0.95", "--local-eps", "1e-6", "--local-weight-decay", "0.01"])
    assert fc.arguments_from_cli(ns).local_opt() == LocalOpt("Adam", betas=(0.8, 0.95), eps=1e-6, weight_decay=0.01)
    ns = fc.parse_cli(["-t", "t", "--local-momentum", "0.9", "--local-nesterov"])
    assert fc.arguments_from_cli(ns).local_opt() == LocalOpt("SGD", momentum=0.9, nesterov=True)
    assert fc.arguments_from_cli(fc.parse_cli(["-t", "t"])).local_opt().is_plain()
    for argv in (["--local-optimizer", "Adam", "-e"], ["--local-momentum", "0.9", "--class-weight", "1,2"],
                 ["--local-momentum", "1.5"], ["--local-nesterov"], ["--local-optimizer", "Adam", "--local-betas", "0.9"],
                 ["--local-optimizer", "Adagrad"], ["--local-optimizer", "Adam", "--local-momentum", "0.9"],
                 ["--local-optimizer", "Adam", "--local-momentum", "0.5", "--local-nesterov"], ["--local-betas", "0.8,0.99"],
                 ["--local-eps", "1e-6"], ["--local-momentum", "0.9", "--local-eps", "1e-6"]):
        with pytest.raises(SystemExit):
            fc.parse_cli(["-t", "t"] + argv)


# ---- trainings ----------------------------------------------------------------------------------------------------------
def test_local_mode_round_is_the_reference_fits():
    """train_virtual_workers with Adam on a CPU box: every worker's model is the reference fit of its shard (the host executor
    within the float64 bound), so the round's FedAvg is the FedAvg of the per-device reference fits"""
    from types import SimpleNamespace
    from colearn_federated_learning_b200.control.coordinator import train_virtual_workers
    from colearn_federated_learning_b200.fl.trainer import FitConfig, make_perm
    from colearn_federated_learning_b200.models import build_model
    model = build_model("ffnn")
    theta = _theta0("ffnn")
    shards = {f"w{i}": SimpleNamespace(x=_data("ffnn", n, i)[0], y=_data("ffnn", n, i)[1]) for i, n in enumerate((23, 0, 40))}

    class _Shard:
        def __init__(self, s):
            self.x, self.y = s.x, s.y

        def __len__(self):
            return self.x.shape[0]

    class Fed:
        workers = list(shards)

        def __getitem__(self, k):
            return _Shard(shards[k])
    lo = FIT_OPTS["adam_wd"]
    cfg = FitConfig(model="ffnn", loss="bce", batch_size=4, epochs=2, lr=LR_ADAM, seed=5).with_local_opt(lo)
    flats, losses, counts = train_virtual_workers(theta.clone(), model, Fed(), cfg, 0)
    assert counts == [23, 0, 40]
    for i, wid in enumerate(Fed.workers):
        sh = shards[wid]
        if sh.x.shape[0] == 0:
            assert torch.equal(flats[i], theta)
            continue
        perm = make_perm(sh.x.shape[0], cfg.with_seed(cfg.seed + 31 * i), torch.device("cpu"), 0)
        o64 = _replay("ffnn", theta, sh.x, sh.y, perm, 4, 2, -1, lo, torch.float64)
        r32 = _replay("ffnn", theta, sh.x, sh.y, perm, 4, 2, -1, lo, torch.float32)
        err = (flats[i].double() - o64[0]).abs().max().item()
        bound = E.C_LONG * (r32[0].double() - o64[0]).abs().max().item() + 2.0 ** -20 * (o64[0] - theta.double()).abs().max().item()
        assert err <= bound, (wid, err, bound)
        assert math.isclose(losses[i], r32[1][-1], rel_tol=1e-4, abs_tol=1e-6), (wid, losses[i], r32[1][-1])


ADAM_WIRE = {"betas": [0.9, 0.999], "eps": 1e-3, "weight_decay": 0.01}


def _remote_adam(tmp_path, n_rounds, **kw):
    """CWT._remote (two loopback devices with 128 synthetic rows each) with Adam at eps 1e-3 (see FIT_OPTS): (result, frames,
    round records, the saved model)"""
    from colearn_federated_learning_b200.models import build_model, flatten_params
    res, frames, recs = CWT._remote(tmp_path, local_optimizer="Adam", local_weight_decay=0.01, local_eps=1e-3, n_rounds=n_rounds,
                                    **kw)
    model = build_model(kw.get("model", "ffnn"))
    model.load_state_dict(torch.load(str(tmp_path / "test.pth"), weights_only=True))
    return res, frames, recs, flatten_params(model)


def _check_adam_training(res, frames, recs, final, n_rounds):
    want = {"kind": "Adam", **ADAM_WIRE}
    assert res["local_opt"] == want
    assert len(recs) == n_rounds and recs[0]["local_opt"] == want and all("local_opt" not in r for r in recs[1:])
    for fr in frames.values():
        fits = [(req, reply) for req, reply in fr if req.get("op") == "fit"]
        assert fits
        for req, reply in fits:
            assert req["config"]["optimizer"] == "Adam" and req["config"]["optimizer_args"] == ADAM_WIRE
            assert reply.get("ok"), reply
    assert bool(torch.isfinite(final).all())


def test_remote_round0_is_the_fedavg_of_reference_fits(tmp_path):
    """Two loopback devices train one round with Adam: every device's reply is the reference fit (reference.mlp_local_sgd with
    the request's optimizer) of its rows, in its order, from the model the request carries, and the coordinator's model is
    their FedAvg, both within the float64 bound.  The device path is the whole of it: fit request -> FitConfig.local_opt() ->
    local_fit -> ops.mlp_local_sgd(local_opt=...)."""
    from colearn_federated_learning_b200.control.workers import _from_bytes
    from colearn_federated_learning_b200.data import BaseDataset, dataset_tensors, synthetic_unsw
    from colearn_federated_learning_b200.fl.trainer import FitConfig, make_perm, resolve_loss
    res, frames, recs, final = _remote_adam(tmp_path, 1)
    _check_adam_training(res, frames, recs, final, 1)
    fits64, bounds = [], []
    for i in range(2):
        req, reply = [(q, r) for q, r in frames[f"dev-{i}"] if q.get("op") == "fit"][0]
        x, y = dataset_tensors(BaseDataset(*synthetic_unsw(128, seed=i + 1)), torch.device("cpu"))
        cfg = FitConfig.from_dict(req["config"])
        lo = cfg.local_opt()
        assert lo == LocalOpt("Adam", eps=1e-3, weight_decay=0.01)
        theta0 = _from_bytes(req["params"])
        perm = make_perm(x.shape[0], cfg, torch.device("cpu"), 0)
        got = _from_bytes(reply["params"])
        fits = {}
        for dt in (torch.float64, torch.float32):
            th = theta0.to(dt).clone()
            R.mlp_local_sgd(th, (10, 50, 30, 10, 1), x.to(dt), y.to(dt).view(x.shape[0], -1), perm, cfg.batch_size, cfg.lr,
                            cfg.epochs, cfg.max_nr_batches, resolve_loss(cfg.model, cfg.loss), "sigmoid", None, lo)
            fits[dt] = th
        d64 = fits[torch.float64] - theta0.double()
        bound = E.C_LONG * (fits[torch.float32].double() - fits[torch.float64]).abs().max().item() + 2.0 ** -20 * d64.abs().max().item()
        err = (got.double() - fits[torch.float64]).abs().max().item()
        assert err <= bound, (i, err, bound)
        assert d64.abs().max().item() > cfg.lr                       # it trained: Adam moves parameters by about lr per step
        plain = theta0.clone()                                       # and not as plain SGD
        R.mlp_local_sgd(plain, (10, 50, 30, 10, 1), x, y.view(x.shape[0], -1), perm, cfg.batch_size, cfg.lr, cfg.epochs,
                        cfg.max_nr_batches, resolve_loss(cfg.model, cfg.loss), "sigmoid")
        assert (plain.double() - fits[torch.float64]).abs().max().item() > 100 * bound
        fits64.append(fits[torch.float64])
        bounds.append(bound)
    avg = (fits64[0] + fits64[1]) / 2
    err = (final.double() - avg).abs().max().item()
    assert err <= sum(bounds) / 2 + 2.0 ** -23 * avg.abs().max().item(), (err, bounds)


@pytest.mark.parametrize("kw", [{"uplink": "int8"}, {"uplink": "topk"}, {"uplink": "int4", "downlink": "int8"},
                                {"aggregator": "median"}, {"aggregator": "geomed"}, {"server_opt": "adam", "server_lr": 0.01},
                                {"secure_agg": True}, {"async_buffer": 2}, {"model": "ffnn_category"}],
                         ids=["uplink-int8", "uplink-topk", "downlink", "median", "geomed", "server-adam", "secagg", "fedbuff",
                              "category"])
def test_remote_adam_composes(tmp_path, kw):
    """A two-round remote training with Adam next to every family of option: codecs, aggregators, server optimizers, secure
    aggregation, FedBuff and the category target.  Every fit request names Adam, every device trains, the records carry
    local_opt and the model stays finite and moves."""
    from colearn_federated_learning_b200.models import build_model, flatten_params
    res, frames, recs, final = _remote_adam(tmp_path, 2, **kw)
    _check_adam_training(res, frames, recs, final, 2)
    torch.manual_seed(0)
    assert not torch.equal(final, flatten_params(build_model(kw.get("model", "ffnn"))))


@pytest.mark.parametrize("target", ["autoencoder", "category"])
def test_local_adam_with_fed_eval_and_targets(tmp_path, target):
    """Local mode with Adam, a federated evaluation after every round, for the autoencoder (input target) and the attack-category
    FFNN: every round is evaluated and the first record carries local_opt"""
    import test_anomaly
    import test_category
    run = test_anomaly.local_run if target == "autoencoder" else test_category.local_run
    _, recs, _ = run(tmp_path, local_optimizer="Adam", local_eps=1e-3)
    assert recs and all("fed_eval" in r for r in recs)
    assert recs[0]["local_opt"]["kind"] == "Adam" and all("local_opt" not in r for r in recs[1:])


def test_coordinator_refuses_class_weights_next_to_an_optimizer():
    from colearn_federated_learning_b200.control.coordinator import _local_opt_field
    from colearn_federated_learning_b200.fl.trainer import FitConfig
    cfg = FitConfig().with_local_opt(OPTS["momentum"])
    with pytest.raises(ValueError, match="class weights together"):
        _local_opt_field(cfg, "balanced")
    assert _local_opt_field(cfg, None) == {"local_opt": OPTS["momentum"].record()}
    assert _local_opt_field(FitConfig(), "balanced") == {}


def test_plain_remote_requests_are_unchanged(tmp_path):
    res0, frames0, _ = CWT._remote(tmp_path / "plain", n_rounds=1)
    assert "local_opt" not in res0
    for fr in frames0.values():
        assert all("optimizer_args" not in req["config"] and req["config"]["optimizer"] == "SGD" for req, _ in fr if req.get("op") == "fit")
