"""How much does a collective running on a side stream slow down the wgmma GEMM?  (2+ GPUs)

    torchrun --nproc-per-node 2 benchmarks/overlap_bench.py

For each collective implementation (16-byte-load kernels vs TMA bulk-copy kernels, selected through
TORCHACC_B200_COMM_TMA_MIN) the script times a train of gate_up GEMMs alone and with all-gathers / reduce-scatters of
one Llama-3-8B layer (436 MB bf16) looping on a second stream, and reports the collective's own bandwidth.
"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
    world = dist.get_world_size()
    dev = torch.device("cuda", rank)
    from torchacc_b200 import _native as nat
    from torchacc_b200.ops.linear import gemm
    from torchacc_b200.parallel.collectives import make_collectives
    coll = make_collectives(dist.group.WORLD, dev, True)
    nat.set_gemm_scheduler(os.environ.get("OVERLAP_SCHED", "dynamic") == "dynamic")
    n_layer = 218_112_000 // (8 * world) * (8 * world)
    shard = coll.alloc(n_layer // world, torch.bfloat16) if hasattr(coll, "alloc") else torch.empty(n_layer // world, dtype=torch.bfloat16, device=dev)
    full = torch.empty(n_layer, dtype=torch.bfloat16, device=dev)
    gfull = coll.alloc(n_layer, torch.bfloat16) if hasattr(coll, "alloc") else torch.empty(n_layer, dtype=torch.bfloat16, device=dev)
    gshard = torch.empty(n_layer // world, dtype=torch.float32, device=dev)
    shard.normal_(); gfull.normal_()
    x = torch.randn(8192, 4096, device=dev, dtype=torch.bfloat16)
    w = torch.randn(28672, 4096, device=dev, dtype=torch.bfloat16) * 0.02
    y = torch.empty(8192, 28672, device=dev, dtype=torch.bfloat16)
    side = torch.cuda.Stream(dev, priority=-1)
    reps = 12

    def gemm_train():
        for _ in range(reps):
            gemm(x, w, out=y)

    def timed(fn, with_comm):
        dist.barrier()
        torch.cuda.synchronize()
        if with_comm is not None:
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(with_comm[1]):
                    with_comm[0]()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        t = torch.tensor(a.elapsed_time(b), device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    def comm_time(fn, n):
        dist.barrier()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        t = torch.tensor(a.elapsed_time(b) / n, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    ag = lambda: coll.all_gather(shard, full)
    rs = lambda: coll.reduce_scatter(gfull, gshard, 1.0 / world)
    for _ in range(2):
        gemm_train(); ag(); rs()
    res = {"world": world, "tma_min": os.environ.get("TORCHACC_B200_COMM_TMA_MIN", "default"),
           "sched": os.environ.get("OVERLAP_SCHED", "dynamic")}
    res["gemm_alone_ms"] = timed(gemm_train, None) / reps
    res["ag_alone_ms"] = comm_time(ag, 8)
    res["rs_alone_ms"] = comm_time(rs, 8)
    remote = n_layer * 2 * (world - 1) / world
    res["ag_GBps"] = remote / res["ag_alone_ms"] / 1e6
    res["rs_GBps"] = remote / res["rs_alone_ms"] / 1e6
    n_ag = int(reps * res["gemm_alone_ms"] / res["ag_alone_ms"]) + 2
    n_rs = int(reps * res["gemm_alone_ms"] / res["rs_alone_ms"]) + 2
    res["gemm_with_ag_ms"] = timed(gemm_train, (ag, n_ag)) / reps
    res["gemm_with_rs_ms"] = timed(gemm_train, (rs, n_rs)) / reps
    res["slowdown_ag"] = res["gemm_with_ag_ms"] / res["gemm_alone_ms"]
    res["slowdown_rs"] = res["gemm_with_rs_ms"] / res["gemm_alone_ms"]
    if dist.get_rank() == 0:
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
