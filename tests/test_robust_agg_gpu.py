"""Byzantine-robust aggregation (coordinate-wise median / trimmed mean) in the sm_90a kernels, against the PyTorch definition
(ops.reference.robust_aggregate): ops.fedavg_apply on its register and general paths, and the star / two-shot kernels on ONE
GPU with W emulated ranks (separate local buffers, raw pointers, arrive flags preset, the ranks' kernels launched one after
another), as the SIMT CPU build does it in test_robust_agg.py.

"Bit for bit" is for every value but NaN: the GPU writes its canonical NaN where arithmetic produces one, so a NaN must meet
a NaN and every other value must carry the same 32 bits."""
import pytest
import torch

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.fl.aggregate import Aggregator
from colearn_federated_learning_b200.fl.server_opt import ServerOpt
from colearn_federated_learning_b200.ops import _ext, reference

from test_robust_agg import models_with_outliers, same_bits

pytestmark = pytest.mark.gpu

AGGS = [Aggregator("median"), Aggregator("trimmed_mean", 0.2)]


@pytest.mark.parametrize("K", [1, 2, 5, 8, 16, 33, 100])
@pytest.mark.parametrize("n", [4096 * 3, 1001])
def test_fedavg_apply_robust(K, n):
    dev = torch.device("cuda", 0)
    models = models_with_outliers(K, n, seed=K * 7 + n)
    theta = torch.randn(n, generator=torch.Generator().manual_seed(n))
    w = torch.full((K,), 1.0 / K)
    for agg in AGGS + [Aggregator("trimmed_mean", 0.0)]:
        th = theta.to(dev)
        ops.fedavg_apply(th, models.to(dev), w.to(dev), aggregator=agg)
        want = reference.fedavg_apply(theta.clone(), models, w, aggregator=agg)
        assert same_bits(th.cpu(), want), (agg, K, n)


def test_fedavg_apply_robust_with_adam():
    dev = torch.device("cuda", 0)
    n, K = 4096 + 3, 9
    opt = ServerOpt("adam", lr=0.05)
    st, ref = opt.init_state(n, dev), opt.init_state(n)
    theta = torch.randn(n)
    th = theta.to(dev)
    agg = Aggregator("median")
    for i in range(3):
        models = theta + 0.5 * torch.randn(K, n)
        models[i] = float("nan")                                # one client sends NaN everywhere
        models[i + 3] = -1e6
        ops.fedavg_apply(th, models.to(dev), torch.full((K,), 1.0 / K, device=dev), opt=st, aggregator=agg)
        reference.server_opt_apply(theta, models, None, "adam", opt.lr, ref.m, ref.v, *opt.hyper, aggregator=agg)
        torch.cuda.synchronize()
        torch.testing.assert_close(th.cpu(), theta, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(st.m.cpu(), ref.m, rtol=1e-5, atol=1e-5)
        theta, ref.m, ref.v = th.cpu(), st.m.cpu(), st.v.cpu()
    assert bool(theta.isfinite().all())


@pytest.mark.parametrize("W", [4, 8])
@pytest.mark.parametrize("agg", AGGS, ids=lambda a: a.kind)
def test_star_round_robust_one_gpu(W, agg):
    ext = _ext.require()
    dev = torch.device("cuda", 0)
    P, P4 = 4099, 4100                                         # float4 body + scalar tail; rows 16-byte aligned as in the engine
    theta = torch.randn(P, device=dev)
    slots = torch.zeros(W, P4, device=dev)
    slots[:, :P] = models_with_outliers(W, P, seed=W).to(dev)
    inbox = torch.zeros(W, P4, device=dev)
    bflag = torch.zeros(W, dtype=torch.int32, device=dev)
    arrive = torch.full((W,), 5, dtype=torch.int32, device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    decision = torch.zeros(2, dtype=torch.int32, device=dev)
    mask = ((1 << W) - 1) & ~0b10                              # worker 1 not selected
    want = reference.fedavg_apply(theta.cpu(), slots[:, :P].cpu()[[k for k in range(W) if (mask >> k) & 1]], None, aggregator=agg)
    ext.star_round(theta.data_ptr(), slots.data_ptr(), P4, arrive.data_ptr(), 5, [inbox[k].data_ptr() for k in range(W)],
                   [bflag[k:].data_ptr() for k in range(W)], 6, 0, mask, 1.0, P, True, True, counter.data_ptr(), 8, 0.0,
                   [1.0 / W] * W, decision.data_ptr(), 0, [], 0, 0, agg.code, agg.trim)
    torch.cuda.synchronize()
    assert same_bits(theta.cpu(), want)
    for k in range(W):
        assert int(bflag[k]) == (6 if (mask >> k) & 1 else 0)
        if (mask >> k) & 1:
            assert same_bits(inbox[k, :P].cpu(), want)
    # a deadline at which worker 0 is late: the aggregate covers the others
    theta2 = torch.randn(P, device=dev)
    arrive[0] = 4
    want2 = reference.fedavg_apply(theta2.cpu(), slots[:, :P].cpu()[[k for k in range(W) if (mask >> k) & 1 and k != 0]], None, aggregator=agg)
    ext.star_round(theta2.data_ptr(), slots.data_ptr(), P4, arrive.data_ptr(), 5, [inbox[k].data_ptr() for k in range(W)],
                   [bflag[k:].data_ptr() for k in range(W)], 7, 0, mask, 1.0, P, True, False, counter.data_ptr(), 8, 2.0,
                   [1.0 / W] * W, decision.data_ptr(), 0, [], 0, 0, agg.code, agg.trim)
    torch.cuda.synchronize()
    assert int(decision[1]) == mask & ~1
    assert same_bits(theta2.cpu(), want2)


@pytest.mark.parametrize("W", [4, 8])
@pytest.mark.parametrize("agg", AGGS, ids=lambda a: a.kind)
def test_twoshot_robust_one_gpu(W, agg):
    ext = _ext.require()
    dev = torch.device("cuda", 0)
    n, chunk = 4 * 4096 + 4 * 96, 1024                         # the last chunk is short
    n_chunks = (n + chunk - 1) // chunk
    trained = models_with_outliers(W, n, seed=100 + W)
    works = trained.to(dev)
    shadows = torch.zeros(W, n, dtype=torch.bfloat16, device=dev)
    flags = torch.zeros(W, n_chunks, dtype=torch.int32, device=dev)
    epoch = 3
    arrive = torch.full((W, W), epoch, dtype=torch.int32, device=dev)   # row r: rank r's arrive flags
    weights = torch.full((W,), 1.0 / W, device=dev)
    mask = ((1 << W) - 1) & ~0b100                              # rank 2 not selected (it still owns chunks)
    for r in range(W):
        ext.twoshot_fedavg([works[k].data_ptr() for k in range(W)], [shadows[k].data_ptr() for k in range(W)],
                           [flags[k].data_ptr() for k in range(W)], arrive[r].data_ptr(), weights.data_ptr(), 0, epoch, mask, 1.0,
                           n, chunk, r, 16, [], False, 0, 0, 0, 0.0, 0, [], 0, 0, agg.code, agg.trim)
    torch.cuda.synchronize()
    want = reference.robust_aggregate(trained, mask, agg.kind, agg.trim)
    for k in range(W):
        assert same_bits(works[k].cpu(), want), k
        assert same_bits(shadows[k].cpu(), works[k].cpu().to(torch.bfloat16)), k
    assert int(flags.min()) == epoch


@pytest.mark.parametrize("agg", AGGS, ids=lambda a: a.kind)
def test_twoshot_robust_with_deadline_one_gpu(agg):
    """rank 3 misses the deadline; chunk ownership is dealt among ranks 0..2, every rank's second arena gets the result"""
    ext = _ext.require()
    dev = torch.device("cuda", 0)
    W, n, chunk = 4, 4 * 2048, 512
    n_chunks = n // chunk
    trained = models_with_outliers(W, n, seed=200)
    works = trained.to(dev)
    globals_ = torch.zeros(W, n, device=dev)
    flags = torch.zeros(W, n_chunks, dtype=torch.int32, device=dev)
    decisions = torch.zeros(W, 16, dtype=torch.int32, device=dev)
    epoch = 5
    arrive = torch.zeros(W, W, dtype=torch.int32, device=dev)
    arrive[:, :3] = epoch
    weights = torch.full((W,), 1.0 / W, device=dev)
    for r in range(3):                                          # the coordinator (which decides) first
        ext.twoshot_fedavg_deadline([works[k].data_ptr() for k in range(W)], [], [flags[k].data_ptr() for k in range(W)],
                                    arrive[r].data_ptr(), weights.data_ptr(), 0, epoch, 0b1111, 1.0, n, chunk, r, 8, [], False, 0, 0,
                                    2.0, [decisions[k].data_ptr() for k in range(W)], [globals_[k].data_ptr() for k in range(W)],
                                    agg.code, agg.trim)
    torch.cuda.synchronize()
    assert int(decisions[0, 2 * (epoch % 8) + 1]) == 0b0111
    want = reference.robust_aggregate(trained, 0b0111, agg.kind, agg.trim)
    for k in range(W):
        assert same_bits(globals_[k].cpu(), want), k
    for k in range(3):
        assert same_bits(works[k].cpu(), want), k


# ---- FederatedEngine ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("agg", AGGS, ids=lambda a: a.kind)
def test_star_engine_verify_round_robust(agg):
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=7, aggregator=agg)
    x, y = synthetic_unsw(200, seed=3)
    eng.set_local_data(x, y)
    for _ in range(3):
        res = eng.verify_round()
        assert res["ok"] and res["max_abs_err"] == 0.0 and res["moved"] > 0, res
    rep = eng.run_rounds(2)
    assert rep.extra["aggregator"] == agg.kind and torch.isfinite(eng.global_flat()).all()


def test_twoshot_engine_robust_one_rank():
    """world 1: the median of one model is that model, so a round gives what a plain FedAvg engine gives, bit for bit"""
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    xs, ys = synthetic_unsw(256, seed=21)
    kw = dict(backend="fused", device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096, bf16_shadow=True, shuffle=False,
              model_kwargs={"width": 256, "depth": 3})
    outs = []
    for agg in (None, Aggregator("median")):
        eng = FederatedEngine("wide_mlp", aggregator=agg, **kw)
        eng.set_local_data(xs, ys)
        rep = eng.run_rounds(2)
        torch.cuda.synchronize()
        assert rep.extra["nvls"] is False and rep.extra["aggregator"] == (agg.kind if agg else "mean")
        outs.append(eng.global_flat().clone())
    assert torch.equal(outs[0], outs[1])


def _rank_main(rank, world, port, out_path):
    import os

    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from colearn_federated_learning_b200.data import shard_bounds, synthetic_unsw
        from colearn_federated_learning_b200.parallel import FederatedEngine
        dev = torch.device("cuda", rank)
        x, y = synthetic_unsw(80 * world, seed=4)
        lo, hi = list(shard_bounds(80 * world, world))[rank]
        x, y = x[lo:hi], y[lo:hi]
        if rank == 1:
            x, y = x * 1e3, 1.0 - y                                # rank 1 trains on poisoned data
        eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=3, aggregator=Aggregator("median"))
        eng.set_local_data(x, y)
        oks = [eng.verify_round() for _ in range(3)]
        if rank == 0:
            torch.save({"oks": oks}, out_path)
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
def test_star_engine_robust_multi_rank_with_a_poisoned_rank(tmp_path):
    import socket

    import torch.multiprocessing as mp
    world = min(torch.cuda.device_count(), 8)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    out = str(tmp_path / "out.pt")
    mp.spawn(_rank_main, args=(world, port, out), nprocs=world, join=True)
    res = torch.load(out, weights_only=False)
    assert all(r["ok"] and r["max_abs_err"] == 0.0 for r in res["oks"]), res
