#!/usr/bin/env python
"""Peer-memory collectives checked against values every rank can compute locally -- NO NCCL collective in the timed /
checked region, so the script can run under compute-sanitizer (NCCL's own kernels are not synccheck-clean and abort the
run: the 2-GPU sanitizer run):

    torchrun --nproc-per-node 2 --master-addr 127.0.0.1 --no-python \
        compute-sanitizer --tool synccheck python tools/symm_selfcheck.py

Every rank seeds a generator per source rank, so it knows all ranks' inputs and can form the expected all-gather,
reduce-scatter, all-reduce and all-to-all results by itself.  Ends with the collective teardown of the domain
(SymmDomain.close)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def inputs(world, n, dtype, device, salt):
    out = []
    for r in range(world):
        g = torch.Generator(device="cpu").manual_seed(1000 * salt + r)
        out.append((torch.randn(n, generator=g) * 0.5).to(dtype).to(device))
    return out


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)           # bootstrap / barriers only
    from torchacc_b200.parallel.symm_mem import SymmCollectives, SymmDomain, symm_available
    assert symm_available(dist.group.WORLD), "symmetric memory unavailable on this box"
    coll = SymmCollectives(dist.group.WORLD, world, rank, dev)
    worst = 0.0
    for salt, n in enumerate([4096, 1 << 20, (1 << 22) + 8 * world]):       # 16-byte-load path, TMA path, ragged TMA path
        n -= n % (8 * world)
        xs = inputs(world, n, torch.bfloat16, dev, salt)
        # all-gather
        full = torch.empty(n * world, dtype=torch.bfloat16, device=dev)
        coll.all_gather(xs[rank], full)
        torch.cuda.synchronize()
        assert torch.equal(full, torch.cat(xs)), f"all_gather n={n}"
        # reduce-scatter (bf16 wire, fp32 accumulate)
        shard = n // world
        out = torch.empty(shard, dtype=torch.float32, device=dev)
        coll.reduce_scatter(xs[rank].clone(), out, 1.0 / world)
        torch.cuda.synchronize()
        want = sum(x[rank * shard:(rank + 1) * shard].float() for x in xs) / world
        worst = max(worst, float((out - want).abs().max()))
        # all-reduce (in place)
        t = xs[rank].float().clone()
        coll.all_reduce(t)
        torch.cuda.synchronize()
        worst = max(worst, float((t - sum(x.float() for x in xs)).abs().max()))
        # all-to-all
        a2a = torch.empty(n, dtype=torch.bfloat16, device=dev)
        coll.all_to_all(xs[rank], a2a)
        torch.cuda.synchronize()
        want = torch.cat([x[rank * shard:(rank + 1) * shard] for x in xs])
        assert torch.equal(a2a, want), f"all_to_all n={n}"
    assert worst < 1e-4, worst
    SymmDomain.close_all()
    if rank == 0:
        print(f"symm selfcheck ok on {world} ranks (max abs err {worst:.2e}); domain closed")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
