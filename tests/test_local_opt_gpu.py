"""Local optimizers on the H100: the optimizer instances of mlp_persistent_opt.cu for all five persistent nets against the
float64 replay of the reference (test_local_opt.py's bound), several clients in one launch bit-identical to each client alone,
two launches agreeing, plain SGD launching the kernels of before with the same bits, and a one-GPU FederatedEngine star round
with Adam."""
import pytest
import torch

import test_local_opt as T
from colearn_federated_learning_b200.fl.local_opt import LocalOpt

gpu = pytest.mark.gpu
SIZES = [37, 0, 129, 1, 64, 203]


def _fit(net, clients, B, epochs, lo, max_b=-1):
    """(outs [K, P], losses [K, 2]) of one launch of K clients on cuda:0"""
    from colearn_federated_learning_b200 import ops
    dev = torch.device("cuda", 0)
    _, dims, act, loss = T.NETS[net]
    theta = clients[0]["theta_in"].to(dev)
    K, P = len(clients), theta.numel()
    slots = torch.full((K, P), 7.0, device=dev)
    lo_out = torch.full((K, 2), 7.0, device=dev)
    keep, tasks = [], []
    for i, c in enumerate(clients):
        x, y, perm = c["x"].to(dev), c["y"].to(dev), c["perm"].to(dev, torch.int32).contiguous()
        keep += [x, y, perm]
        tasks.append(ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=slots[i], perm=perm, loss_out=lo_out[i]))
    descs = ops.build_client_descs(tasks, dev)
    lr = T.LR if lo is None else T._lr(lo)
    ops.mlp_local_sgd_multi(dims, act, descs, K, batch_size=B, lr=lr, epochs=epochs, max_nr_batches=max_b, loss=loss,
                            local_opt=lo)
    torch.cuda.synchronize()
    return slots.cpu(), lo_out.cpu()


@gpu
@pytest.mark.parametrize("net", sorted(T.NETS))
@pytest.mark.parametrize("opt", ["momentum", "nesterov_wd", "adam", "adam_wd"])
@pytest.mark.parametrize("B", [1, 7])
def test_instances_match_the_reference_gpu(net, opt, B):
    lo = T.FIT_OPTS[opt]
    clients = [T._client(net, n, 2, seed=i) for i, n in enumerate(SIZES)]
    outs, losses = _fit(net, clients, B, 2, lo)
    for k, c in enumerate(clients):
        T._check(f"gpu {net} {opt} B{B} client {k}", net, outs[k], losses[k], c["theta_in"], c["x"], c["y"], c["perm"], B, 2, -1, lo)
    for k in (0, 2):                                   # each client alone: the same bits
        alone, alone_l = _fit(net, [clients[k]], B, 2, lo)
        assert torch.equal(alone[0], outs[k]) and torch.equal(alone_l[0], losses[k]), (net, opt, B, k)
    again, again_l = _fit(net, clients, B, 2, lo)      # two launches agree
    assert torch.equal(again, outs) and torch.equal(again_l, losses)


@gpu
def test_max_batches_gpu():
    lo = T.FIT_OPTS["adam_wd"]
    for net in ("ffnn", "mlp"):
        c = T._client(net, 300, 3)
        outs, losses = _fit(net, [c], 4, 3, lo, max_b=100)
        T._check(f"gpu max_b {net}", net, outs[0], losses[0], c["theta_in"], c["x"], c["y"], c["perm"], 4, 3, 100, lo)


@gpu
@pytest.mark.parametrize("net", sorted(T.NETS))
def test_plain_sgd_is_the_default_kernel_gpu(net):
    """No optimizer and SGD with explicit zeros give the same bits (variant 5, the default)"""
    clients = [T._client(net, n, 2, seed=i) for i, n in enumerate(SIZES)]
    a, la = _fit(net, clients, 1, 2, None)
    b, lb = _fit(net, clients, 1, 2, LocalOpt("SGD", momentum=0.0, weight_decay=0.0))
    assert torch.equal(a, b) and torch.equal(la, lb)


@gpu
def test_engine_star_round_with_adam_gpu():
    """One-GPU FederatedEngine with Adam: verify_round's fused round equals the library round of the same local fit, the
    model moves, and the local fit is the optimizer instances' (not plain SGD's)"""
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel.engine import FederatedEngine
    dev = torch.device("cuda", 0)
    res = {}
    for name, lo in (("adam", LocalOpt("Adam")), ("sgd", None)):
        eng = FederatedEngine("ffnn", backend="fused", device=dev, batch_size=1, lr=0.01, seed=3, local_opt=lo)
        x, y = synthetic_unsw(256, seed=0)
        eng.set_local_data(x.to(dev), y.to(dev))
        assert eng.algo == "star"
        out = eng.verify_round()
        assert out["ok"], out
        res[name] = eng.global_flat().clone()
    assert not torch.equal(res["adam"], res["sgd"])
