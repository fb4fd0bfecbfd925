"""``ops.fedavg_apply_based`` on the H100 (``fedavg_based_kernel``, ``fedavg_based_robust_kernel`` and the distance passes on
``BasedRows``) against ``ops.reference`` on the CPU: bit for bit for the mean and the coordinate-wise kinds under sgd / adam /
yogi, K in {1, 3, 40}, P in {1, 255, 2401, 4096, 2^20, 2^20 + 3} with random base slots in a ring of 5; geomed / norm_clip within their
tolerance, their agg_weights_out too; the write slot holds the new theta and the other slots are untouched."""
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.server_opt import ServerOpt

from test_async_apply import AGGS, case, same

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")


def cuda_state(st):
    st.m = st.m.to(DEV) if st.m is not None else None
    st.v = st.v.to(DEV) if st.v is not None else None
    return st


@pytest.mark.parametrize("P", [1, 255, 2401, 4096, 2 ** 20, 2 ** 20 + 3])   # P % 4 == 0: the 16-byte path
@pytest.mark.parametrize("K", [1, 3, 40])
@pytest.mark.parametrize("opt_kind", ["sgd", "adam", "yogi"])
@pytest.mark.parametrize("agg_name", ["mean", "median", "trimmed_mean"])
def test_cuda_matches_reference_bit_for_bit(agg_name, opt_kind, K, P):
    theta, ring, models, w, bases = case(K, P, seed=K * 131 + P)
    agg = AGGS[agg_name]
    opt = ServerOpt(opt_kind, lr=0.05) if opt_kind != "sgd" else None
    st_ref, st = (opt.init_state(P), cuda_state(opt.init_state(P))) if opt else (None, None)
    step_ref = dict(opt=st_ref) if opt else dict(server_lr=0.7)
    step = dict(opt=st) if opt else dict(server_lr=0.7)
    want, ring_want = theta.clone(), ring.clone()
    ops.fedavg_apply_based(want, models, ring_want, bases, w, 2, aggregator=agg, **step_ref)
    got, ring_got = theta.to(DEV), ring.to(DEV)
    ops.fedavg_apply_based(got, models.to(DEV), ring_got, bases, w.to(DEV), 2, aggregator=agg, **step)
    got, ring_got = got.cpu(), ring_got.cpu()
    assert same(got, want)
    assert same(ring_got[2], got)
    keep = [s for s in range(5) if s != 2]
    assert same(ring_got[keep], ring[keep])
    if opt:
        assert same(st.m.cpu(), st_ref.m) and same(st.v.cpu(), st_ref.v)


@pytest.mark.parametrize("P", [2401, 4096, 2 ** 20, 2 ** 20 + 3])
@pytest.mark.parametrize("K", [3, 40])
@pytest.mark.parametrize("agg_name", ["geomed", "norm_clip"])
def test_cuda_distance_aggregators_within_tolerance(agg_name, K, P):
    theta, ring, models, w, bases = case(K, P, seed=K + P)
    agg = AGGS[agg_name]
    w_ref, w_got = torch.zeros(K), torch.zeros(K, device=DEV)
    want, ring_want = theta.clone(), ring.clone()
    ops.fedavg_apply_based(want, models, ring_want, bases, w, 2, server_lr=0.7, aggregator=agg, agg_weights_out=w_ref)
    got, ring_got = theta.to(DEV), ring.to(DEV)
    ops.fedavg_apply_based(got, models.to(DEV), ring_got, bases, w.to(DEV), 2, server_lr=0.7, aggregator=agg, agg_weights_out=w_got)
    torch.testing.assert_close(got.cpu(), want, atol=2e-5, rtol=2e-5)
    torch.testing.assert_close(w_got.cpu(), w_ref, atol=1e-6, rtol=1e-5)
    assert same(ring_got[2].cpu(), got.cpu())
    keep = [s for s in range(5) if s != 2]
    assert same(ring_got[keep].cpu(), ring[keep])


def test_cuda_every_base_current_is_the_synchronous_step_in_float64():
    theta, ring, models, w, _ = case(16, 2401, seed=3)
    got = theta.to(DEV)
    ops.fedavg_apply_based(got, models.to(DEV), ring.to(DEV), [1] * 16, w.to(DEV), 3)
    want = theta.double() + (w.double().view(-1, 1) * (models.double() - theta.double())).sum(0)
    torch.testing.assert_close(got.cpu().double(), want, atol=1e-6, rtol=1e-6)


def test_cuda_launcher_refuses_the_write_slot_as_a_base():
    theta, ring, models, w, _ = case(3, 300, seed=5)
    from colearn_federated_learning_b200.ops import _ext
    got, ring_got = theta.to(DEV), ring.to(DEV)
    with pytest.raises(RuntimeError):
        _ext.require().fedavg_apply_based(got, models.to(DEV), ring_got, torch.tensor([0, 2, 3], dtype=torch.int32), w.to(DEV), 2, 1.0)
    assert same(got.cpu(), theta) and same(ring_got.cpu(), ring)
