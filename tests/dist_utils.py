"""Multi-process test harness: N gloo ranks on this host (the reference's harness needs GPUs + NCCL,
reference tests/utils/distributed.py:14-64; ours runs the same plumbing on CPU)."""
import os
import socket
import sys
import traceback

import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, fn, args, errq):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port), TORCHACC_B200_FORCE_CPU="1")
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    torch.set_num_threads(1)
    try:
        import torch.distributed as dist
        dist.init_process_group("gloo", rank=rank, world_size=world)
        fn(rank, world, *args)
        # drain every group this rank belongs to (in creation order, the same on every rank) before any socket closes:
        # a rank that tears down while a peer still has traffic on a subgroup (TP, FSDP shard groups) can abort both
        # processes in gloo's teardown
        for pg in list(dist.distributed_c10d._world.pg_map):
            dist.barrier(group=pg)
        dist.destroy_process_group()
    except Exception:
        errq.put((rank, traceback.format_exc()))
        raise


def run_distributed(fn, world: int = 2, args=(), timeout: float = 240.0):
    """Run ``fn(rank, world, *args)`` in ``world`` processes; re-raises the first failure with its traceback."""
    ctx = mp.get_context("spawn")
    errq = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, fn, args, errq)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout)
    failed = []
    for r, p in enumerate(procs):
        if p.is_alive():
            p.kill()   # exact child handle, not a pattern
            failed.append((r, "timeout"))
        elif p.exitcode != 0:
            failed.append((r, f"exit code {p.exitcode}"))
    msgs = []
    while not errq.empty():
        msgs.append(errq.get())
    if failed or msgs:
        detail = "\n".join(f"--- rank {r} ---\n{tb}" for r, tb in msgs) or str(failed)
        raise AssertionError(f"distributed test failed: {failed}\n{detail}")
