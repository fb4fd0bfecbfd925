"""Class-weighted training on the H100: the weighted instances of mlp_persistent_cw.cu with several clients in one launch, held
to the same three checks as the SIMT build in test_class_weight.py (w ≡ 1 gives the unweighted bits, a zero weight leaves θ
bit for bit, mixed weights match the float64 oracle within the bounds of test_mlp_kernel_edges.py), and one short local-mode
ffnn_category training with balanced weights."""
import math

import pytest
import torch

import test_class_weight as T

gpu = pytest.mark.gpu


def _fit(net, loss, clients, B, epochs, w=None):
    """(outs [K, P], losses [K, 2]) of one launch of K clients on cuda:0, unweighted (w None) or weighted"""
    from colearn_federated_learning_b200 import ops
    dev = torch.device("cuda", 0)
    _, dims, act, _ = T.NETS[net]
    theta = T._theta0(net).to(dev)
    K, P = len(clients), theta.numel()
    slots = torch.full((K, P), 7.0, device=dev)
    lo = torch.full((K, 2), 7.0, device=dev)
    keep, tasks = [], []
    for i, c in enumerate(clients):
        x, y, perm = c["x"].to(dev), c["y"].to(dev), c["perm"].to(dev, torch.int32).contiguous()
        keep += [x, y, perm]
        tasks.append(ops.ClientTask(x=x, y=y, theta_in=theta, theta_out=slots[i], perm=perm, loss_out=lo[i]))
    descs = ops.build_client_descs(tasks, dev)
    ops.mlp_local_sgd_multi(dims, act, descs, K, batch_size=B, lr=T.LR, epochs=epochs, loss=loss, class_weights=w)
    torch.cuda.synchronize()
    return slots.cpu(), lo.cpu()


SIZES = [10, 37, 1, 203, 64, 0, 129, 5]


@gpu
@pytest.mark.parametrize("net,loss", T.CASES + [("ffnn", "mse")])
@pytest.mark.parametrize("B", [1, 4])
def test_unit_weights_are_the_unweighted_bits_gpu(net, loss, B):
    clients = T._clients(net, SIZES)
    outs, losses = _fit(net, loss, clients, B, 2)
    outs_w, losses_w = _fit(net, loss, clients, B, 2, [1.0] * T.NETS[net][3])
    assert torch.equal(outs, outs_w), (net, loss, B)
    assert torch.equal(losses, losses_w), (net, loss, B)


@gpu
@pytest.mark.parametrize("net,loss", T.CASES)
@pytest.mark.parametrize("B", [1, 4])
def test_zero_weight_leaves_theta_gpu(net, loss, B):
    clients = T._clients(net, SIZES)
    outs, losses = _fit(net, loss, clients, B, 2, [0.0] * T.NETS[net][3])
    theta0 = T._theta0(net)
    for k in range(len(clients)):
        assert torch.equal(outs[k], theta0), (net, loss, B, k)
    assert torch.equal(losses, torch.zeros_like(losses))


@gpu
@pytest.mark.parametrize("net,loss", T.CASES + [("ffnn", "mse")])
@pytest.mark.parametrize("B", [1, 4])
def test_mixed_weights_match_the_oracle_gpu(net, loss, B):
    w = T.MIXED[net]
    clients = T._clients(net, [37, 10, 64, 203, 1], seed=3)
    outs, losses = _fit(net, loss, clients, B, 2, w)
    theta0 = T._theta0(net)
    for k, c in enumerate(clients):
        o64 = T._oracle(net, loss, theta0, c["x"], c["y"], c["perm"], B, 2, w)
        r32 = T._reference32(net, loss, theta0, c["x"], c["y"], c["perm"], B, 2, w)
        T._check(f"gpu {net} {loss} B{B} client {k}", outs[k], losses[k], theta0, o64, r32)


@gpu
def test_local_training_balanced_gpu(tmp_path):
    import test_category as TC
    _, recs, _ = TC.local_run(tmp_path, device=torch.device("cuda", 0), class_weight="balanced")
    cw = recs[0]["class_weights"]
    assert cw["mode"] == "balanced" and len(cw["weights"]) == 5 and sum(cw["counts"]) == 3000
    assert all(r.get("fed_eval") for r in recs) and all(math.isfinite(v) for r in recs for v in r["loss_k"])
    # well above the majority class alone (macro F1 ~0.11); the same training on the CPU's host executor reaches 0.75
    assert recs[-1]["fed_eval"]["total"]["macro_f1"] >= 0.5
