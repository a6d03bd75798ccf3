"""Collectives carried inside the GEMM kernels (csrc/fused/carry.cuh / carry.cu) -- the FSDP hot path.

Instead of launching the parameter all-gather and the gradient reduce-scatter of a unit as their own kernels on side
streams, the sharding engine *enqueues* them here.  Every wgmma GEMM launched afterwards (forward, recomputation,
dgrad, wgrad, the chunked lm_head) takes a slice of the pending jobs proportional to its FLOPs, and warp 3 of each of
its CTAs moves that slice over NVLink with TMA bulk copies while the tile pipeline of the same CTA runs:

* all-gather: peer shards -> private smem ring -> the local gathered flat-parameter buffer;
* reduce-scatter: this rank's slice of all peers' flat gradient buffers -> smem -> fp32 sum -> 1/world scale ->
  gradient shard, and the sum of squares of the result for ``clip_grad_norm_`` (no separate norm pass).

Foreground jobs (the next unit's gather) get a launch's byte budget first; background jobs (reduce-scatters, the
lm_head gather) use the rest.  Whatever no GEMM carried by the time it is needed runs as one stand-alone kernel
(``flush``) -- in a Llama-3-8B step that is the first gather of the step and the last reductions of the backward.
Everything is on the compute stream: there are no communication streams and no events in this mode.

Reference parity: torchacc/dist/fsdp.py:196-230 (torch FSDP / XLA-FSDP all-gather + reduce-scatter per unit).
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from .. import _native as nat

nat.register_signatures({
    "tb_carry_push": ([nat.i32, ctypes.POINTER(nat.u64), nat.u64, ctypes.POINTER(nat.u64), nat.i64, nat.i32, nat.i32,
                       nat.i32, ctypes.c_uint32, nat.u64, nat.f32, nat.i32, nat.i32, nat.i32, nat.u64, nat.i32, nat.i32,
                       ctypes.c_uint32], nat.i64),
    "tb_symm_signal": ([ctypes.POINTER(nat.u64), nat.i32, nat.i32, nat.i32, ctypes.c_uint32, nat.u64], nat.i32),
    "tb_carry_pending": ([nat.i64, nat.i32], nat.i64),
    "tb_carry_take_probe": ([ctypes.c_double, ctypes.POINTER(nat.i64)], nat.i32),
    "tb_carry_flush": ([nat.i64, nat.i32, nat.i32, nat.u64], nat.i32),
    "tb_carry_bytes_per_flop": ([ctypes.c_double], ctypes.c_double),
    "tb_carry_stats": ([ctypes.POINTER(nat.i64), nat.i32], nat.i32),
    "tb_carry_set_debug": ([nat.u64, nat.i64], nat.i64),
    "tb_symm_wait_done": ([ctypes.POINTER(nat.u64), nat.i32, nat.i32, nat.i32, ctypes.c_uint32, nat.u64], nat.i32),
})

# signal-pad channels (parallel/symm_mem.py uses 0-3, fused TP 8+).  CH_PARAMS carries only ENTRY flags: "my parameter
# shards of this step are final" -- one epoch per step, every gather job of the step waits for it.
CH_GATHER, CH_REDUCE, CH_GATHER_BG, CH_PARAMS = 4, 5, 6, 7
FOREGROUND, BACKGROUND, ALL_QUEUES = 0, 1, -1


def available() -> bool:
    L = nat.lib()
    return L is not None and hasattr(L, "tb_carry_push")


class CarryRuntime:
    """Job submission for one symmetric-memory domain (= one FSDP shard group)."""

    def __init__(self, coll, device: torch.device):
        self.coll = coll                      # SymmCollectives
        self.domain = coll.domain
        self.device = device
        self.world, self.rank = self.domain.world, self.domain.rank
        # [sum of squares of every reduced gradient shard of this backward pass, non-finite flag]
        self.stats = torch.zeros(2, dtype=torch.float32, device=device)
        self.reduce_jobs = 0                  # reduce-scatters pushed since the statistics were armed
        self.stats_exact = True               # False once a job accumulated into an existing shard (micro-batching)
        self.last_epoch = {CH_GATHER: 0, CH_REDUCE: 0, CH_GATHER_BG: 0}
        self.params_epoch = 0

    # ---- submission ---------------------------------------------------------------------------------------
    def _buf(self, t: torch.Tensor):
        buf = self.domain.find(t)
        if buf is None:
            raise RuntimeError("carried collectives need their peer-visible operand inside the symmetric domain")
        return buf

    def _signal(self, channel: int, epoch: int) -> None:
        d = self.domain
        nat.check(nat.require().tb_symm_signal(d.pad_ptrs, self.rank, self.world, channel, epoch, nat.stream()),
                  "tb_symm_signal")
        nat.count_launch()

    def publish_params(self) -> int:
        """Tell every peer that ALL parameter shards of this rank are final for the coming step (call once per step,
        after the optimizer / the bf16 refresh of every unit).  Gather jobs pushed afterwards wait for this epoch on
        every rank -- they never depend on how far a peer has progressed inside the step."""
        self.params_epoch = self.domain.next_epoch(CH_PARAMS)
        self._signal(CH_PARAMS, self.params_epoch)
        return self.params_epoch

    def publish_grads(self) -> int:
        """Tell every peer that the flat gradient buffer of the unit whose backward just ended is final.  Returns the
        epoch the (possibly later enqueued) reduce job has to be pushed with."""
        epoch = self.domain.next_epoch(CH_REDUCE)
        self._signal(CH_REDUCE, epoch)
        return epoch

    def push_gather(self, shard: torch.Tensor, full: torch.Tensor, background: bool = False):
        """``full[r * n:(r + 1) * n] = shard of rank r`` for every r (own shard included, copied first).
        Needs ``publish_params()`` of this step.  Returns ``(job_id, channel, epoch)``."""
        d = self.domain
        buf = self._buf(shard)
        nbytes = shard.numel() * shard.element_size()
        assert nbytes % 16 == 0 and full.numel() == shard.numel() * self.world and full.is_contiguous()
        off = shard.data_ptr() - buf.ptr
        src = (nat.u64 * self.world)(*[buf.peer_ptrs[r] + off for r in range(self.world)])
        ch = CH_GATHER_BG if background else CH_GATHER
        epoch = d.next_epoch(ch)
        L = nat.require()
        job = L.tb_carry_push(1, src, full.data_ptr(), d.pad_ptrs, nbytes, self.rank, self.world, ch, epoch,
                              d.counter_ptr(ch), 1.0, 0, 0, 0, 0, int(background), CH_PARAMS, self.params_epoch)
        if job <= 0:
            raise nat.NativeError("tb_carry_push (gather) rejected the job")
        self.last_epoch[ch] = epoch
        return job, ch, epoch

    def push_reduce(self, full: torch.Tensor, out: torch.Tensor, scale: float, accumulate: bool, epoch: int):
        """``out (+)= scale * sum_r full_of_rank_r[rank * n:(rank + 1) * n]`` with fp32 accumulation; the sum of
        squares of the new ``out`` is added to ``self.stats``.  ``epoch`` comes from ``publish_grads()`` (called when
        the buffer became final; the job itself may be enqueued later).  Returns ``(job_id, channel, epoch)``."""
        d = self.domain
        buf = self._buf(full)
        n = out.numel()
        assert full.numel() == n * self.world and full.is_contiguous() and out.is_contiguous()
        assert full.dtype in (torch.bfloat16, torch.float32) and out.dtype in (torch.bfloat16, torch.float32)
        slice_bytes = n * full.element_size()
        assert slice_bytes % 256 == 0, "shard sizes are multiples of 128 elements"
        off = full.data_ptr() - buf.ptr
        src = (nat.u64 * self.world)(*[buf.peer_ptrs[r] + off for r in range(self.world)])
        L = nat.require()
        job = L.tb_carry_push(2, src, out.data_ptr(), d.pad_ptrs, slice_bytes, self.rank, self.world, CH_REDUCE, epoch,
                              d.counter_ptr(CH_REDUCE), float(scale), int(full.dtype == torch.bfloat16),
                              int(out.dtype == torch.float32), int(accumulate), self.stats.data_ptr(), 1,
                              CH_REDUCE, epoch)
        if job <= 0:
            raise nat.NativeError("tb_carry_push (reduce) rejected the job")
        self.last_epoch[CH_REDUCE] = epoch
        self.reduce_jobs += 1
        if accumulate:
            self.stats_exact = False
        return job, CH_REDUCE, epoch

    def arm_stats(self):
        """Start of a backward pass: forget the previous pass' gradient statistics."""
        self.stats.zero_()
        self.reduce_jobs = 0
        self.stats_exact = True

    # ---- completion ---------------------------------------------------------------------------------------
    def pending(self, job: int = 0, queue: int = ALL_QUEUES) -> int:
        return int(nat.require().tb_carry_pending(job, queue))

    def flush(self, job: int = 0, queue: int = ALL_QUEUES) -> None:
        """Issue whatever is still queued (up to ``job``) as a stand-alone kernel on the current stream."""
        L = nat.require()
        if L.tb_carry_pending(job, queue) > 0:
            nat.check(L.tb_carry_flush(job, queue, nat.num_sms(), nat.stream()), "tb_carry_flush")
            nat.count_launch()

    def wait_done(self, channel: int, epoch: int) -> None:
        """Current stream waits until EVERY rank finished the job ``epoch`` of ``channel`` (its source buffers may
        then be overwritten)."""
        if epoch <= 0:
            return
        d = self.domain
        nat.check(nat.require().tb_symm_wait_done(d.pad_ptrs, self.rank, self.world, channel, epoch, nat.stream()),
                  "tb_symm_wait_done")
        nat.count_launch()

    @staticmethod
    def counters(reset: bool = False) -> dict:
        out = (nat.i64 * 4)()
        nat.require().tb_carry_stats(out, int(reset))
        return {"chunks_carried": out[0], "chunks_flushed": out[1], "launches_carrying": out[2], "flushes": out[3]}


def make_carry(coll, device: torch.device) -> Optional[CarryRuntime]:
    """A runtime when ``coll`` is the symmetric-memory back-end on a CUDA device and the feature is enabled."""
    import os
    if device.type != "cuda" or not hasattr(coll, "domain") or not available():
        return None
    mode = os.environ.get("TORCHACC_B200_CARRY", "auto")
    if mode == "0":
        return None
    if mode == "auto" and coll.domain.world > 2:
        # with 8 ranks a reduce stage is eight 1 KB bulk loads and every GEMM CTA's copy warp fans in from 7 peers.  Until the copy role uses larger per-peer stages the stand-alone TMA
        # collectives (side streams, communication windows) stay the default beyond 2 ranks; TORCHACC_B200_CARRY=1 forces it.
        return None
    return CarryRuntime(coll, device)
