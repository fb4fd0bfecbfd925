"""Broadcast + FedAvg-reduce bandwidth sweep (BASELINE.json: "broadcast+FedAvg-reduce GB/s vs 450 GB/s/dir").

Run under torchrun on N GPUs.  For each message size P (fp32 elements) it times, with CUDA events and
max over ranks:
  * ours   — ``twoshot_fedavg_kernel`` (reduce + weight + apply + re-broadcast, fp32 [+ bf16 shadow]) and,
             for small P, the coordinator-centric ``star_round_kernel`` path;
  * nccl   — ``dist.all_reduce`` (the library collective the comparator would use for the same job).
Reported bandwidth is algorithmic per-GPU traffic: every rank must receive (W-1)/W·P (reduce leg) and
(W-1)/W·P (broadcast leg) fp32 → bus_bytes = 2·(W-1)/W·4P, the same convention as nccl-tests' busbw.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from colearn_federated_learning_b200 import ops
from colearn_federated_learning_b200.parallel import init_distributed, shutdown
from colearn_federated_learning_b200.parallel.symm import SymmetricArena
from colearn_federated_learning_b200.utils.monitors import NvlinkCounters

NVL = {"counters": None}


def timed(fn, iters, world, device, nvlink=None):
    """ms per call (CUDA events, max over ranks).  ``nvlink``: a dict that receives this GPU's NVLink payload bytes per call
    as the hardware counted them (NVML), next to the time — a second, untimed loop so the NVML reads never sit inside the
    event bracket."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device=device, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    c = NVL["counters"]
    if nvlink is not None and c is not None and c.ok:
        import time
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        time.sleep(0.3)                                   # let the counters settle (barrier traffic, NVML's own sampling)
        a = c.read()
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()                                # every peer's stores into this GPU have landed
        torch.cuda.synchronize()
        time.sleep(0.3)
        d = c.delta(a, c.read())
        if d is not None:
            nvlink.update({"tx_bytes_per_call": d["tx_bytes"] / iters, "rx_bytes_per_call": d["rx_bytes"] / iters, "calls": iters})
    return float(t.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/comm_sweep.json")
    ap.add_argument("--sizes", default="4994,109386,1048576,11181644,50397188")
    ap.add_argument("--chunk-elems", type=int, default=0, help="0 = adaptive")
    ap.add_argument("--shadow", action="store_true")
    ap.add_argument("--blocks", type=int, default=0, help="CTAs for the two-shot kernel (0 = auto)")
    ap.add_argument("--tag", default="")
    ap.add_argument("--nvls", type=int, default=1, help="use multimem.ld_reduce/st when a multicast mapping exists")
    ap.add_argument("--nvlink-counters", action="store_true",
                    help="also report each kernel's NVLink payload bytes per call from the GPU's own counters (NVML field values)")
    args = ap.parse_args()
    rank, world, device = init_distributed()
    if args.nvlink_counters:
        NVL["counters"] = NvlinkCounters(index=device.index or 0, uuid=str(torch.cuda.get_device_properties(device).uuid))
        if rank == 0 and not NVL["counters"].ok:
            print("NVLink counters unavailable:", NVL["counters"].err, flush=True)
    ext = ops._ext.require()
    results = []
    for P in [int(s) for s in args.sizes.split(",")]:
        P4 = (P + 3) // 4 * 4
        chunk = args.chunk_elems
        if not chunk:
            chunk, target = 2048, max(1, P4 // (world * 296))
            while chunk < target and chunk < 65536:
                chunk *= 2
        n_chunks = (P4 + chunk - 1) // chunk
        layout = {"work": (P4, torch.float32), "chunk_flags": (n_chunks, torch.int32), "flags": (64, torch.int32)}
        if args.shadow:
            layout["shadow"] = (P4, torch.bfloat16)
        arena = SymmetricArena(layout, device)
        arena.tensor("work").normal_()
        weights = torch.full((16,), 1.0 / world, device=device)
        use_nvls = bool(args.nvls and arena.has_multicast and world > 1)
        arrive = [arena.ptr("flags", k, 1 + rank) for k in range(world)]
        state = {"e": 0}
        n_blocks = args.blocks or max(1, min(132 * 2, (n_chunks + world - 1) // world))

        def ours():
            state["e"] += 1
            e = state["e"]
            ext.twoshot_fedavg(arena.peer_ptrs("work"), arena.peer_ptrs("shadow") if args.shadow else [],
                               arena.peer_ptrs("chunk_flags"), arena.ptr("flags", None, 1), weights.data_ptr(), 0, e,
                               (1 << world) - 1, 1.0, P4, chunk, rank, n_blocks, arrive, True,
                               arena.mc_ptr("work") if use_nvls else 0,
                               arena.mc_ptr("shadow") if (use_nvls and args.shadow) else 0, 0, 0.0)

        iters = 20 if P4 < (1 << 22) else 8
        nvl_ours, nvl_nccl = ({}, {}) if args.nvlink_counters else (None, None)
        ms = timed(ours, iters, world, device, nvl_ours)
        buf = torch.randn(P4, device=device)
        ms_nccl = timed(lambda: dist.all_reduce(buf), iters, world, device, nvl_nccl) if world > 1 else float("nan")
        bus = 2.0 * (world - 1) / world * 4.0 * P4
        rec = {"P": P, "bytes": 4 * P4, "world": world, "provider": arena.provider, "multicast": arena.has_multicast,
               "twoshot_ms": ms, "twoshot_busbw_GBps": bus / ms / 1e6 if world > 1 else None,
               "nccl_allreduce_ms": ms_nccl, "nccl_busbw_GBps": bus / ms_nccl / 1e6 if world > 1 else None,
               "shadow_bf16": args.shadow, "chunk_elems": chunk, "nvls": use_nvls, "blocks": n_blocks, "tag": args.tag,
               # fraction of the H100's NVLink 4 450 GB/s per direction (data sheet); busbw is directly comparable with it
               "twoshot_frac_of_450GBps": (bus / ms / 1e6 / 450.0) if world > 1 else None,
               "nccl_frac_of_450GBps": (bus / ms_nccl / 1e6 / 450.0) if world > 1 else None}
        if args.nvlink_counters:
            # what the algorithm says this GPU must move per call: pull (W-1)/W of the vector for its reduce share + push its
            # reduced share to W-1 peers (P2P form) = (W-1)/W * 4P each way; with NVLS the switch reduces and multicasts, so
            # the GPU receives 1/W of the vector once (already reduced) and sends its share once.
            rec["nvlink"] = {"ours": nvl_ours, "nccl_allreduce": nvl_nccl,
                             "algorithmic_bytes_each_way_p2p": (world - 1) / world * 4.0 * P4,
                             "counter": "NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX/RX summed over links (payload, KiB granularity), rank 0's GPU"}
            if nvl_ours and ms > 0:
                rec["nvlink"]["ours_tx_GBps"] = nvl_ours.get("tx_bytes_per_call", 0) / ms / 1e6
                rec["nvlink"]["ours_rx_GBps"] = nvl_ours.get("rx_bytes_per_call", 0) / ms / 1e6
        results.append(rec)
        if rank == 0:
            print(json.dumps(rec), flush=True)
        arena.close()
        del arena
    if rank == 0:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)
    shutdown()


if __name__ == "__main__":
    main()
