"""Fused NVLink collectives + engine on real GPUs (1 GPU: single-rank paths; >= 2 GPUs: spawned ranks).

Each multi-rank case runs in spawned processes (one per GPU, NCCL only for bootstrap) and compares
the fused result with a plain PyTorch recomputation of the same round semantics."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_engine_star_single_gpu_matches_reference_round():
    from colearn_federated_learning_b200 import ops
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.ops import reference as R
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=7, shuffle=False)
    x, y = synthetic_unsw(300, seed=2)
    eng.set_local_data(x, y)
    theta0 = eng.global_flat().cpu().clone()
    rep = eng.run_rounds(3)
    ref = theta0.clone()
    for _ in range(3):
        R.mlp_local_sgd(ref, eng.spec.dims, x, y, R.make_permutation(300, 1, 0, shuffle=False), 1, 0.05, 1, -1, "xent")
    assert torch.allclose(eng.global_flat().cpu(), ref, atol=5e-4, rtol=5e-3)
    assert rep.launches == 3 * 2 + 1 and rep.losses.shape == (3, 1, 2)
    # second call continues from the stored epoch counters; e2e path with host inputs + read back
    hx, hy = x.pin_memory(), y.pin_memory()
    rep2 = eng.run_rounds(2, host_inputs=[(hx, hy)] * 2, read_back=True, barrier=False)
    for _ in range(2):
        R.mlp_local_sgd(ref, eng.spec.dims, x, y, R.make_permutation(300, 1, 0, shuffle=False), 1, 0.05, 1, -1, "xent")
    assert torch.allclose(eng.global_flat().cpu(), ref, atol=1e-3, rtol=1e-2)
    assert abs(float(eng.loss_host[0]) - float(rep2.losses[-1, 0, 0])) < 1e-6


def test_engine_single_round_calls_use_cached_plan_and_match_multi_round():
    from colearn_federated_learning_b200.data import synthetic_unsw
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    x, y = synthetic_unsw(200, seed=5)
    a = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=9, shuffle=False)
    b = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=9, shuffle=False)
    a.set_local_data(x, y)
    b.set_local_data(x, y)
    for _ in range(4):
        a.run_rounds(1)
    assert a._star_plan["used"] == 4                      # one plan, four single-round calls
    b.run_rounds(4)
    assert torch.allclose(a.global_flat(), b.global_flat(), atol=1e-6)
    a.run_rounds(2)                                       # a multi-round call in between invalidates nothing it should not
    a.run_rounds(1)
    b.run_rounds(3)
    assert torch.allclose(a.global_flat(), b.global_flat(), atol=1e-6)


def test_engine_many_clients_per_gpu():
    """100 federated devices do not need 100 GPUs: C virtual clients per rank, one CTA each, summed on-GPU."""
    from colearn_federated_learning_b200.data import shard_bounds, synthetic_unsw
    from colearn_federated_learning_b200.ops import reference as R
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    C, n = 13, 650
    eng = FederatedEngine("ffnn", backend="fused", device=dev, batch_size=1, lr=0.05, seed=2, shuffle=False, weighted=True,
                          clients_per_rank=C)
    x, y = synthetic_unsw(n, seed=4)
    eng.set_local_data(x, y)
    theta0 = eng.global_flat().cpu().clone()
    rep = eng.run_rounds(2)
    ref = theta0.clone()
    for _ in range(2):
        acc = torch.zeros_like(ref)
        for lo, hi in shard_bounds(n, C):
            loc = ref.clone()
            R.mlp_local_sgd(loc, eng.spec.dims, x[lo:hi], y[lo:hi], R.make_permutation(hi - lo, 1, 0, shuffle=False), 1, 0.05, 1,
                            -1, "bce", "sigmoid")
            acc += loc * ((hi - lo) / n)
        ref = acc
    assert torch.allclose(eng.global_flat().cpu(), ref, atol=5e-4, rtol=5e-3), (eng.global_flat().cpu() - ref).abs().max()
    assert rep.launches == 2 * 3 + 1 and torch.isfinite(rep.losses).all()


def test_engine_twoshot_single_gpu_resnet_round():
    from colearn_federated_learning_b200.data import synthetic_images
    from colearn_federated_learning_b200.parallel import FederatedEngine
    dev = torch.device("cuda", 0)
    eng = FederatedEngine("resnet18", backend="fused", device=dev, batch_size=128, lr=0.05, seed=1)
    x, y = synthetic_images(256, seed=0)
    eng.set_local_data(x, y.float().view(-1, 1))
    t0 = eng.global_flat().clone()
    rep = eng.run_rounds(2)
    assert rep.algo == "twoshot" and torch.isfinite(eng.global_flat()).all() and not torch.equal(eng.global_flat(), t0)
    assert rep.extra["train_path"] == "convnet"                  # this repo's conv / BatchNorm kernels + wgmma GEMMs, not cuDNN
    assert float(rep.losses[1, 0, 0]) < float(rep.losses[0, 0, 0]) * 1.5
    # a shape the conv kernels do not cover raises instead of switching to cuDNN (fl/trainer.py: _library_path_guard)
    eng32 = FederatedEngine("resnet18", backend="fused", device=dev, batch_size=32, lr=0.05, seed=1)
    eng32.set_local_data(x[:64], y[:64].float().view(-1, 1))
    import pytest as _pytest
    with _pytest.raises(RuntimeError, match="no sm_90a kernel path"):
        eng32.run_rounds(1)


# ------------------------------------------------------------------------------------------------------------
def _rank_main(rank, world, port, out_path, case):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), LOCAL_RANK=str(rank),
                      WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        from colearn_federated_learning_b200 import ops
        from colearn_federated_learning_b200.data import synthetic_unsw
        from colearn_federated_learning_b200.ops import reference as R
        from colearn_federated_learning_b200.parallel import FederatedEngine
        dev = torch.device("cuda", rank)
        sizes = [200, 120, 80, 160, 90, 70, 110, 130][:world]
        x, y = synthetic_unsw(sizes[rank], seed=10 + rank)
        if case == "star":
            eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=3, shuffle=False, weighted=True)
            eng.set_local_data(x, y)
            theta0 = eng.global_flat().clone()
            masks = [(1 << world) - 1, 0b01 if world == 2 else 0b0101, (1 << world) - 1]
            rep = eng.run_rounds(3, masks=masks)
            # recompute on this rank with the reference: gather everything we need
            gathered = [None] * world
            dist.all_gather_object(gathered, (x, y))
            if rank == 0:
                theta = theta0.cpu()
                for m in masks:
                    sel = [k for k in range(world) if (m >> k) & 1]
                    tot = sum(sizes[k] for k in sel)
                    acc = torch.zeros_like(theta)
                    for k in sel:
                        loc = theta.clone()
                        xs, ys = gathered[k]
                        R.mlp_local_sgd(loc, eng.spec.dims, xs, ys, R.make_permutation(len(xs), 1, 0, shuffle=False), 1, 0.05, 1, -1, "xent")
                        acc += loc * (sizes[k] / tot)
                    theta = acc
                err = (eng.global_flat().cpu() - theta).abs().max().item()
                torch.save({"err": err, "provider": rep.extra["provider"], "multicast": rep.extra["multicast"],
                            "losses": rep.losses.cpu()}, out_path)
        elif case == "twoshot":
            # wide-ish MLP through the generic torch path: checks the in-place all-reduce-with-apply + chunk flags
            eng = FederatedEngine("net", backend="fused", device=dev, batch_size=16, lr=0.05, seed=4, chunk_elems=8192,
                                  bf16_shadow=True)
            xs = torch.rand(64, 784, generator=torch.Generator().manual_seed(rank))
            ys = torch.randint(0, 10, (64, 1), generator=torch.Generator().manual_seed(100 + rank)).float()
            eng.set_local_data(xs, ys)
            theta0 = eng.global_flat().clone()
            rep = eng.run_rounds(2)
            flat = eng.global_flat().clone()
            allf = [torch.zeros_like(flat) for _ in range(world)]
            dist.all_gather(allf, flat)
            same = all(torch.equal(allf[0], f) for f in allf)             # every rank holds the new global model
            shadow_ok = torch.equal(eng.arena.tensor("shadow")[: eng.P], flat.to(torch.bfloat16))
            if rank == 0:
                torch.save({"same": same, "shadow_ok": bool(shadow_ok), "moved": not torch.equal(flat, theta0),
                            "finite": bool(torch.isfinite(flat).all()), "n_chunks": rep.extra["n_chunks"]}, out_path)
        elif case == "twoshot_nvls_weighted":
            # n_k-weighted and subset rounds on the NVLS path (every rank pre-scales its arena by its weight, 0 when it was not
            # selected, then the switch sums all members) against the P2P path of the same rounds
            sizes2 = [256, 128, 384, 128, 256, 128, 384, 128][:world]
            xs, ys = synthetic_unsw(sizes2[rank], seed=30 + rank)
            masks = [(1 << world) - 1, (0b01 if world == 2 else 0b0110), (1 << world) - 1]
            outs, nvls_flags = [], []
            for use in ("1", "0"):
                os.environ["COLEARN_NVLS"] = use
                eng = FederatedEngine("wide_mlp", backend="fused", device=dev, batch_size=128, lr=0.05, seed=9, chunk_elems=4096,
                                      bf16_shadow=True, weighted=True, model_kwargs={"width": 256, "depth": 3})
                eng.set_local_data(xs, ys)
                per_round = []
                for m in masks:
                    rep = eng.run_rounds(1, masks=m)
                    per_round.append(bool(rep.extra["nvls"]))
                torch.cuda.synchronize()
                outs.append(eng.global_flat().clone())
                nvls_flags.append(per_round)
                multicast = eng.arena.has_multicast
            os.environ.pop("COLEARN_NVLS", None)
            allf = [torch.zeros_like(outs[0]) for _ in range(world)]
            dist.all_gather(allf, outs[0])
            if rank == 0:
                scale = float(outs[1].abs().max())
                torch.save({"err": float((outs[0] - outs[1]).abs().max()) / scale, "same": all(torch.equal(allf[0], f) for f in allf),
                            "nvls_rounds": nvls_flags[0], "p2p_rounds": nvls_flags[1], "multicast": bool(multicast),
                            "finite": bool(torch.isfinite(outs[0]).all())}, out_path)
        elif case == "twoshot_deadline":
            # failure detection on the large-model path: rank 1's shard is 24x bigger, it misses the coordinator's deadline in
            # round 1, the round completes on the ranks that arrived (weights renormalised, chunk ownership dealt among them);
            # before round 2 the late rank restores its arena from the second arena and — with a generous deadline — takes part
            n_r = 3072 if rank == 1 else 128
            xs, ys = synthetic_unsw(n_r, seed=40 + rank)
            eng = FederatedEngine("wide_mlp", backend="fused", device=dev, batch_size=128, lr=0.05, seed=11, chunk_elems=4096,
                                  bf16_shadow=True, weighted=False, round_deadline_ms=1.0, model_kwargs={"width": 512, "depth": 3})
            eng.set_local_data(xs, ys)
            theta0 = eng.global_flat().clone()
            rep1 = eng.run_rounds(1)
            torch.cuda.synchronize()
            after1 = eng.arena.tensor("global")[: eng.P].clone()           # what the owners pushed (the late rank's work arena is garbage)
            # reference of round 1 on every arrived rank: same trainer class, same data, from theta0
            from colearn_federated_learning_b200.fl.layerwise import LayerwiseMLPTrainer
            loc = theta0.clone()
            tr = LayerwiseMLPTrainer(eng.spec, loc, 128)
            from colearn_federated_learning_b200.fl.trainer import make_perm
            tr.fit(loc, xs.to(dev), ys.to(dev), eng.cfg, make_perm(n_r, eng.cfg, dev, 0))
            locs = [torch.zeros_like(loc) for _ in range(world)]
            dist.all_gather(locs, loc)
            eng.round_deadline_ms = 5000.0                                  # round 2: everybody makes it
            rep2 = eng.run_rounds(1)
            torch.cuda.synchronize()
            flat2 = eng.global_flat().clone()
            allf = [torch.zeros_like(flat2) for _ in range(world)]
            dist.all_gather(allf, flat2)
            alla = [torch.zeros_like(after1) for _ in range(world)]
            dist.all_gather(alla, after1)
            if rank == 0:
                arrived = rep1.extra["arrived_masks"][0]
                sel = [k for k in range(world) if (arrived >> k) & 1]
                want = sum(locs[k] for k in sel) / len(sel)
                torch.save({"arrived1": arrived, "arrived2": rep2.extra["arrived_masks"][0], "world": world,
                            "err1": float((after1 - want).abs().max() / want.abs().max()),
                            "global_same": all(torch.equal(alla[0], a) for a in alla),
                            "same2": all(torch.equal(allf[0], f) for f in allf), "finite": bool(torch.isfinite(flat2).all()),
                            "moved2": not torch.equal(flat2, after1)}, out_path)
        elif case == "twoshot_kernel":
            # direct numerics of twoshot_fedavg_kernel: P2P path (non-uniform weights, subset mask) and NVLS path
            from colearn_federated_learning_b200.parallel.symm import SymmetricArena
            ext = ops._ext.require()
            P4, chunk = 40000, 2048
            n_chunks = (P4 + chunk - 1) // chunk
            arena = SymmetricArena({"work": (P4, torch.float32), "shadow": (P4, torch.bfloat16),
                                    "chunk_flags": (n_chunks, torch.int32), "flags": (64, torch.int32)}, dev)
            base = torch.arange(P4, dtype=torch.float32, device=dev) * 1e-3
            arrive = [arena.ptr("flags", k, 1 + rank) for k in range(world)]
            results = {}
            epoch = 0
            for name, mask, wts, nvls in (("p2p_weighted", (1 << world) - 1, [float(k + 1) for k in range(world)], False),
                                          ("p2p_subset", 0b01 if world == 2 else 0b0110, None, False),
                                          ("nvls_uniform", (1 << world) - 1, None, True)):
                epoch += 1
                sel = [k for k in range(world) if (mask >> k) & 1]
                w = torch.zeros(16)
                if wts is None:
                    for k in sel:
                        w[k] = 1.0 / len(sel)
                else:
                    tot = sum(wts[k] for k in sel)
                    for k in sel:
                        w[k] = wts[k] / tot
                arena.tensor("work").copy_(base * (rank + 1) + rank)
                torch.cuda.synchronize()
                dist.barrier()
                use_nvls = nvls and arena.has_multicast
                ext.twoshot_fedavg(arena.peer_ptrs("work"), arena.peer_ptrs("shadow"), arena.peer_ptrs("chunk_flags"),
                                   arena.ptr("flags", None, 1), w.to(dev).data_ptr(), 0, epoch, mask, 1.0, P4, chunk, rank,
                                   8, arrive, True, arena.mc_ptr("work") if use_nvls else 0,
                                   arena.mc_ptr("shadow") if use_nvls else 0, 0, 0.0)
                torch.cuda.synchronize()
                dist.barrier()
                want = sum(float(w[k]) * (base * (k + 1) + k) for k in sel)
                got = arena.tensor("work")
                results[name] = {"err": float((got - want).abs().max() / want.abs().max()), "nvls": bool(use_nvls),
                                 "shadow_ok": bool(torch.equal(arena.tensor("shadow"), got.to(torch.bfloat16)))}
            allr = [None] * world
            dist.all_gather_object(allr, results)
            if rank == 0:
                torch.save(allr, out_path)
        elif case == "deadline":
            # failure detection: rank 1 is ~60x slower than the coordinator's deadline allows -> dropped from the
            # round, its weight renormalised away, the round completes with the workers that did arrive
            n = 64 if rank != 1 else 4096
            xs, ys = synthetic_unsw(n, seed=30 + rank)
            eng = FederatedEngine("mlp", backend="fused", device=dev, batch_size=1, lr=0.05, seed=3, shuffle=False,
                                  weighted=False, round_deadline_ms=0.5)
            eng.set_local_data(xs, ys)
            theta0 = eng.global_flat().clone()
            rep = eng.run_rounds(1)
            gathered = [None] * world
            dist.all_gather_object(gathered, (xs, ys))
            if rank == 0:
                arrived = rep.extra["arrived_masks"][0]
                sel = [k for k in range(world) if (arrived >> k) & 1]
                acc = torch.zeros_like(theta0.cpu())
                for k in sel:
                    loc = theta0.cpu().clone()
                    xk, yk = gathered[k]
                    R.mlp_local_sgd(loc, eng.spec.dims, xk, yk, R.make_permutation(len(xk), 1, 0, shuffle=False), 1, 0.05, 1, -1, "xent")
                    acc += loc / len(sel)
                err = (eng.global_flat().cpu() - acc).abs().max().item()
                torch.save({"arrived": arrived, "err": err, "world": world}, out_path)
            torch.cuda.synchronize()
        elif case == "wide":
            # wide MLP on the wgmma layer-wise trainer; rounds >= 2 consume the two-shot broadcast through the
            # bf16 shadow arena with the GEMM's TMA producer polling per-chunk flags (fused broadcast -> GEMM)
            eng = FederatedEngine("wide_mlp", backend="fused", device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096,
                                  bf16_shadow=True, model_kwargs={"width": 256, "depth": 2})
            xs, ys = synthetic_unsw(256, seed=20 + rank)
            eng.set_local_data(xs, ys)
            rep = eng.run_rounds(4)
            flat = eng.global_flat().clone()
            allf = [torch.zeros_like(flat) for _ in range(world)]
            dist.all_gather(allf, flat)
            same = all(torch.equal(allf[0], f) for f in allf)
            shadow_ok = torch.equal(eng.arena.tensor("shadow")[: eng.P], flat.to(torch.bfloat16))
            if rank == 0:
                # device perms differ from CPU perms, so compare the loss trajectory, not the weights
                torch.save({"same": same, "shadow_ok": bool(shadow_ok), "finite": bool(torch.isfinite(flat).all()),
                            "path": rep.extra["train_path"], "loss_first": float(rep.losses[0, :, 0].mean()),
                            "loss_last": float(rep.losses[-1, :, 0].mean())}, out_path)
        elif case == "wide_overlap":
            # fused wgrad GEMM -> FedAvg reduce (opt-in): the two-shot kernel runs next to the last backward and takes chunks
            # as the wgrad epilogues report them.  Same kernels, same summation order => bit-identical to the serial round.
            flats, paths = [], []
            for overlap in (False, True):
                eng = FederatedEngine("wide_mlp", backend="fused", device=dev, batch_size=128, lr=0.05, seed=6, chunk_elems=4096,
                                      bf16_shadow=True, model_kwargs={"width": 256, "depth": 2}, overlap_reduce=overlap)
                xs, ys = synthetic_unsw(384, seed=20 + rank)
                eng.set_local_data(xs, ys)
                rep = eng.run_rounds(4, masks=[(1 << world) - 1, (1 << world) - 1, (1 << world) - 2 if world > 1 else 1, (1 << world) - 1])
                flats.append(eng.global_flat().clone())
                paths.append(rep.extra["train_path"])
                shadow_ok = torch.equal(eng.arena.tensor("shadow")[: eng.P], flats[-1].to(torch.bfloat16))
                idle = overlap is False or bool((eng.prod_count == 0).all())
            allf = [torch.zeros_like(flats[1]) for _ in range(world)]
            dist.all_gather(allf, flats[1])
            if rank == 0:
                torch.save({"same": all(torch.equal(allf[0], f) for f in allf), "identical": bool(torch.equal(flats[0], flats[1])),
                            "shadow_ok": bool(shadow_ok), "idle": idle, "paths": paths,
                            "finite": bool(torch.isfinite(flats[1]).all())}, out_path)
    finally:
        dist.destroy_process_group()


@pytest.mark.multigpu
@pytest.mark.parametrize("case", ["star", "twoshot", "twoshot_kernel", "twoshot_nvls_weighted", "twoshot_deadline", "wide", "deadline", "wide_overlap"])
def test_fused_collectives_multi_rank(tmp_path, case):
    world = min(torch.cuda.device_count(), 8)
    out = str(tmp_path / "out.pt")
    mp.spawn(_rank_main, args=(world, _free_port(), out, case), nprocs=world, join=True)
    res = torch.load(out, weights_only=False)
    if case == "star":
        assert res["err"] < 2e-3, res
        assert torch.isfinite(res["losses"]).all()
    elif case == "twoshot_kernel":
        for per_rank in res:
            for name, r in per_rank.items():
                assert r["err"] < 1e-5 and r["shadow_ok"], (name, r)
    elif case == "deadline":
        assert (res["arrived"] >> 1) & 1 == 0 and res["arrived"] & 1 == 1, res     # slow rank 1 dropped, rank 0 kept
        assert res["err"] < 2e-3, res
    elif case == "wide_overlap":
        assert res["same"] and res["identical"] and res["shadow_ok"] and res["idle"] and res["finite"], res
        assert res["paths"][1].endswith("+overlap_reduce") and not res["paths"][0].endswith("+overlap_reduce"), res
    elif case == "twoshot_deadline":
        assert (res["arrived1"] >> 1) & 1 == 0 and res["arrived1"] & 1 == 1, res       # the slow rank 1 was dropped from round 1 ...
        assert res["err1"] < 2e-3 and res["global_same"], res                          # ... which is the mean over those that arrived
        assert res["arrived2"] == (1 << res["world"]) - 1 and res["same2"] and res["finite"] and res["moved2"], res
    elif case == "twoshot_nvls_weighted":
        assert res["same"] and res["finite"] and res["err"] < 2e-3, res         # bf16 shadows + switch-defined reduction order
        assert res["p2p_rounds"] == [False, False, False], res
        if res["multicast"]:
            assert res["nvls_rounds"] == [True, True, True], res                 # weighted AND subset rounds take the in-switch reduce
    elif case == "twoshot":
        assert res["same"] and res["shadow_ok"] and res["moved"] and res["finite"], res
    else:
        assert res["same"] and res["shadow_ok"] and res["finite"], res
        assert res["path"].startswith("layerwise+fused_bcast") and res["loss_last"] < res["loss_first"], res
