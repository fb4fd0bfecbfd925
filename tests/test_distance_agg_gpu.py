"""Distance-based robust aggregation on the H100: ``ops.fedavg_apply`` / ``ops.fedavg_apply_quantized`` with ``geomed`` and
``norm_clip`` against the reference (tolerance of tests/test_distance_agg.py), over fp32 / int8 / int4 rows, K from 1 to
100, P across chunk boundaries, with and without a server optimizer; two calls give the same bits, and ``agg_weights_out``
matches the reference weights."""
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.fl.uplink import UplinkCodec
from colearn_federated_learning_b200.ops import reference

pytestmark = pytest.mark.gpu
TOL = dict(atol=2e-5, rtol=2e-5)
AGGS = {"geomed": Aggregator("geomed", iters=3), "geomed1": Aggregator("geomed", iters=1), "norm_clip": Aggregator("norm_clip", clip_norm=2.0)}
CASES = [(1, 1001), (2, 2048), (5, 2401), (8, 1001), (16, 3 * 4096), (32, 2401), (33, 2048), (100, 1001)]


def _rows(K, P, seed):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(P, generator=g)
    x = theta + 0.1 * torch.randn(K, P, generator=g)
    if K > 2:
        x[1] = float("nan")
        x[2] = theta + 1000 * (x[2] - theta)
    alpha = torch.rand(K, generator=g) + 0.5
    return theta, x, alpha / alpha.sum()


def _run(theta, apply, opt_kind, P):
    if opt_kind is None:
        apply(theta, None)
        return theta, None
    st = ServerOpt(opt_kind, lr=0.01).init_state(P, theta.device)
    apply(theta, st)
    return theta, st


@pytest.mark.parametrize("opt_kind", [None, "adam"])
@pytest.mark.parametrize("agg", list(AGGS))
@pytest.mark.parametrize("K,P", CASES)
def test_fp32_matches_reference(K, P, agg, opt_kind):
    agg = AGGS[agg]
    theta, x, alpha = _rows(K, P, K * 7 + P)
    dev = torch.device("cuda")
    outs = []
    for _ in range(2):
        w = torch.zeros(K, device=dev)
        t, st = _run(theta.to(dev), lambda t, st: ops.fedavg_apply(t, x.to(dev), alpha, opt=st, aggregator=agg, agg_weights_out=w), opt_kind, P)
        outs.append((t.cpu(), w.cpu(), st))
    w_ref = torch.zeros(K)
    ref, st_ref = _run(theta.clone(), lambda t, st: ops.fedavg_apply(t, x, alpha, opt=st, aggregator=agg, agg_weights_out=w_ref), opt_kind, P)
    torch.testing.assert_close(outs[0][0], ref, **TOL)
    torch.testing.assert_close(outs[0][1], w_ref, atol=1e-6, rtol=1e-5)
    if st_ref is not None:
        torch.testing.assert_close(outs[0][2].m.cpu(), st_ref.m, **TOL)
    assert torch.equal(outs[0][0].view(torch.int32), outs[1][0].view(torch.int32))
    assert torch.equal(outs[0][1].view(torch.int32), outs[1][1].view(torch.int32))


@pytest.mark.parametrize("opt_kind", [None, "adam"])
@pytest.mark.parametrize("agg", list(AGGS))
@pytest.mark.parametrize("bits", [8, 4])
@pytest.mark.parametrize("K,P", CASES)
def test_quantized_matches_reference(K, P, bits, agg, opt_kind):
    agg = AGGS[agg]
    theta, x, alpha = _rows(K, P, K * 11 + P + bits)
    x = torch.where(torch.isfinite(x), x, theta)
    codec = UplinkCodec(f"int{bits}")
    payload, scales = reference.encode_delta(x, theta, bits, list(range(1, K + 1)))
    if K > 2:
        scales[1, 0] = float("nan")
    dev = torch.device("cuda")
    outs = []
    for _ in range(2):
        w = torch.zeros(K, device=dev)
        t, _ = _run(theta.to(dev), lambda t, st: ops.fedavg_apply_quantized(t, payload, scales, alpha, codec, opt=st, aggregator=agg,
                                                                           agg_weights_out=w), opt_kind, P)
        outs.append((t.cpu(), w.cpu()))
    w_ref = torch.zeros(K)
    ref, _ = _run(theta.clone(), lambda t, st: ops.fedavg_apply_quantized(t, payload, scales, alpha, codec, opt=st, aggregator=agg,
                                                                         agg_weights_out=w_ref), opt_kind, P)
    torch.testing.assert_close(outs[0][0], ref, **TOL)
    torch.testing.assert_close(outs[0][1], w_ref, atol=1e-6, rtol=1e-5)
    assert torch.equal(outs[0][0].view(torch.int32), outs[1][0].view(torch.int32))


@pytest.mark.parametrize("agg", list(AGGS))
def test_misaligned_theta(agg):
    agg = AGGS[agg]
    K, P = 7, 2401
    theta, x, alpha = _rows(K, P + 1, 3)
    dev = torch.device("cuda")
    buf = theta.to(dev)
    t = buf[1:]
    ops.fedavg_apply(t, x[:, 1:].contiguous().to(dev), alpha, aggregator=agg)
    ref = theta[1:].clone()
    ops.fedavg_apply(ref, x[:, 1:].contiguous(), alpha, aggregator=agg)
    torch.testing.assert_close(t.cpu(), ref, **TOL)
    assert float(buf[0].cpu()) == float(theta[0])


def test_all_rows_nonfinite_keep_theta():
    dev = torch.device("cuda")
    theta = torch.randn(5000, device=dev)
    x = torch.full((4, 5000), float("nan"), device=dev)
    for agg in AGGS.values():
        t = theta.clone()
        w = torch.ones(4, device=dev)
        ops.fedavg_apply(t, x, torch.full((4,), 0.25), aggregator=agg, agg_weights_out=w)
        assert torch.equal(t, theta) and not bool(w.any())
