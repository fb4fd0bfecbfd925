"""The asynchronous apply (``ROWS_F32_BASED``: fp32 models read as deltas to their base version in a ring, the new theta
also stored to the ring's write slot) through the SIMT CPU build of ``elementwise.cu``, against ``ops.reference``:
bit for bit for the mean and the coordinate-wise kinds under sgd / adam / yogi, within the distance-aggregator tolerance for
geomed / norm_clip; and the launcher's refusal of a base slot that is out of range or equal to the write slot."""
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt

SLOTS = 5
AGGS = {"mean": Aggregator("mean"), "median": Aggregator("median"), "trimmed_mean": Aggregator("trimmed_mean", 0.2),
        "geomed": Aggregator("geomed", iters=3), "norm_clip": Aggregator("norm_clip", clip_norm=2.0)}


@pytest.fixture(scope="module")
def simt():
    import importlib.util
    import os
    import shutil

    from colearn_federated_learning_b200.ops import build
    if shutil.which("g++") is None or not os.path.exists(os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include", "cuda_runtime.h")):
        pytest.skip("no g++ / CUDA headers on this box: the SIMT emulator cannot be built")
    path = build.build_simt_emul()
    spec = importlib.util.spec_from_file_location("_colearn_simt", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def case(K, P, seed, write_slot=2):
    """theta, ring [SLOTS, P] (theta in slot 1), models trained from random bases (never the write slot), weights, bases"""
    g = torch.Generator().manual_seed(seed)
    ring = torch.randn(SLOTS, P, generator=g)
    theta = ring[1].clone()
    bases = [b for b in torch.randint(0, SLOTS, (4 * K,), generator=g).tolist() if b != write_slot][:K]
    bases += [1] * (K - len(bases))
    models = ring[bases] + 0.1 * torch.randn(K, P, generator=g)
    if K > 1:
        models[K // 2] += 3.0                                     # one far row for the robust kinds to act on
    w = (torch.rand(K, generator=g) + 0.5) / K
    return theta, ring, models, w, bases


def same(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def tail(agg, opt, st, w_out):
    t = [float(opt.lr), opt.code, opt.hyper, st.m, st.v] if opt else [0.7, 0, [], None, None]
    return t + [agg.code, agg.trim, agg.iters, agg.eps, agg.clip, w_out, 0]


@pytest.mark.parametrize("P", [1, 255, 1001, 1024])       # 1024: the 16-byte loads and ring stores
@pytest.mark.parametrize("K", [1, 3, 40])
@pytest.mark.parametrize("opt_kind", ["sgd", "adam", "yogi"])
@pytest.mark.parametrize("agg_name", ["mean", "median", "trimmed_mean"])
def test_simt_matches_reference_bit_for_bit(simt, agg_name, opt_kind, K, P):
    theta, ring, models, w, bases = case(K, P, seed=K * 131 + P)
    agg = AGGS[agg_name]
    opt = ServerOpt(opt_kind, lr=0.05) if opt_kind != "sgd" else None
    st_ref, st = (opt.init_state(P), opt.init_state(P)) if opt else (None, None)
    want, ring_want = theta.clone(), ring.clone()
    ops.fedavg_apply_based(want, models, ring_want, bases, w, 2, aggregator=agg, **(dict(opt=st_ref) if opt else dict(server_lr=0.7)))
    got, ring_got = theta.clone(), ring.clone()
    simt.fedavg_apply_based(got, models, ring_got, torch.tensor(bases, dtype=torch.int32), w, 2, *tail(agg, opt, st, None))
    assert same(got, want)
    assert same(ring_got, ring_want)
    assert same(ring_got[2], got)                                     # the write slot holds the new theta
    keep = [s for s in range(SLOTS) if s != 2]
    assert same(ring_got[keep], ring[keep])                           # the other slots are untouched
    if opt:
        assert same(st.m, st_ref.m) and same(st.v, st_ref.v)
    assert not same(got, theta) or P == 1


@pytest.mark.parametrize("K", [3, 40])
@pytest.mark.parametrize("agg_name", ["geomed", "norm_clip"])
def test_simt_distance_aggregators_match_within_tolerance(simt, agg_name, K):
    P = 2100                                                          # partial last 2048-chunk
    theta, ring, models, w, bases = case(K, P, seed=K + 7)
    agg = AGGS[agg_name]
    w_ref, w_got = torch.zeros(K), torch.zeros(K)
    want, ring_want = theta.clone(), ring.clone()
    ops.fedavg_apply_based(want, models, ring_want, bases, w, 2, server_lr=0.7, aggregator=agg, agg_weights_out=w_ref)
    got, ring_got = theta.clone(), ring.clone()
    simt.fedavg_apply_based(got, models, ring_got, torch.tensor(bases, dtype=torch.int32), w, 2, *tail(agg, None, None, w_got))
    torch.testing.assert_close(got, want, atol=2e-5, rtol=2e-5)
    torch.testing.assert_close(w_got, w_ref, atol=1e-6, rtol=1e-5)
    assert same(ring_got[2], got)
    assert float(w_ref.min()) < float(w_ref.max())                    # the far row was weighted down


@pytest.mark.parametrize("bases,write", [([0, 2, 3], 2), ([0, 5, 3], 2), ([0, -1, 3], 2), ([0, 1, 3], 5)])
def test_launcher_refuses_a_base_on_the_write_slot_or_out_of_range(simt, bases, write):
    theta, ring, models, w, _ = case(3, 300, seed=5)
    got, ring_got = theta.clone(), ring.clone()
    with pytest.raises(RuntimeError, match="launch failed"):
        simt.fedavg_apply_based(got, models, ring_got, torch.tensor(bases, dtype=torch.int32), w, write, *tail(AGGS["mean"], None, None, None))
    assert same(got, theta) and same(ring_got, ring)
    with pytest.raises(ValueError, match="must lie in"):
        ops.fedavg_apply_based(theta.clone(), models, ring.clone(), bases, w, write)


def test_every_base_the_current_theta_is_the_synchronous_fedavg_step():
    """with every row trained from theta the apply is theta + sum w_k (x_k - theta), within fp32 rounding of float64"""
    theta, ring, models, w, _ = case(6, 2401, seed=11)
    got = theta.clone()
    ops.fedavg_apply_based(got, models, ring, [1] * 6, w, 3)
    want = theta.double() + (w.double().view(-1, 1) * (models.double() - theta.double())).sum(0)
    torch.testing.assert_close(got.double(), want, atol=1e-6, rtol=1e-6)
