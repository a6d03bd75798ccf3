"""Throughput / memory observability (the reference has neither a memory-stats API nor device-timed throughput:
its benchmark divides the batch size by rank-0 host wall-clock between log points, benchmarks/transformer.py:186-204;
SURVEY 5.5).

* ``ThroughputMeter``: CUDA-event timing of a window of steps, reduced with MAX over ranks (the number a whole job
  actually achieves), host wall-clock fallback on CPU.
* ``memory_stats()``: allocator + engine view of device memory in GB (what is resident: master/compute shards,
  gradient shards, pooled gather/gradient buffers).
"""
from __future__ import annotations

import time
from typing import Any, Dict, Optional

import torch
import torch.distributed as dist


class ThroughputMeter:
    """``with meter.step(tokens): train_step()`` ... ``meter.summary()`` -> tokens/s of the whole job."""

    def __init__(self, device: Optional[torch.device] = None, group=None):
        self.device = device if device is not None else (
            torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu"))
        self.group = group
        self.reset()

    def reset(self):
        self._tokens = 0
        self._steps = 0
        self._start = None
        self._end = None

    class _Step:
        def __init__(self, meter, tokens):
            self.m, self.tokens = meter, tokens

        def __enter__(self):
            m = self.m
            if m._start is None:
                if m.device.type == "cuda":
                    m._start = torch.cuda.Event(enable_timing=True)
                    m._start.record()
                else:
                    m._start = time.perf_counter()
            return self

        def __exit__(self, *exc):
            m = self.m
            m._tokens += self.tokens
            m._steps += 1
            if m.device.type == "cuda":
                m._end = torch.cuda.Event(enable_timing=True)
                m._end.record()
            else:
                m._end = time.perf_counter()
            return False

    def step(self, tokens: int) -> "ThroughputMeter._Step":
        return ThroughputMeter._Step(self, int(tokens))

    def summary(self) -> Dict[str, float]:
        """tokens counted on THIS rank x world / max-over-ranks elapsed time."""
        if self._start is None or self._end is None:
            return {"steps": 0, "tokens_per_s": 0.0, "ms_per_step": 0.0}
        if self.device.type == "cuda":
            self._end.synchronize()
            ms = self._start.elapsed_time(self._end)
        else:
            ms = (self._end - self._start) * 1e3
        world = 1
        if dist.is_available() and dist.is_initialized():
            world = dist.get_world_size(self.group)
            t = torch.tensor([ms], dtype=torch.float64, device=self.device if self.device.type == "cuda" else "cpu")
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
            ms = float(t)
        return {"steps": self._steps, "ms_per_step": ms / max(self._steps, 1),
                "tokens_per_s": self._tokens * world / (ms / 1e3) if ms > 0 else 0.0, "world": world}


def memory_stats(model: Any = None, device: Optional[int] = None) -> Dict[str, float]:
    """Device memory in GB: torch allocator counters plus, for an accelerated model, what the sharding engine holds."""
    gb = 1.0 / (1 << 30)
    out: Dict[str, float] = {}
    if torch.cuda.is_available():
        free, total = torch.cuda.mem_get_info(device)
        out.update(allocated=torch.cuda.memory_allocated(device) * gb, reserved=torch.cuda.memory_reserved(device) * gb,
                   peak_allocated=torch.cuda.max_memory_allocated(device) * gb, device_free=free * gb,
                   device_total=total * gb)
    eng = getattr(model, "engine", None)
    if eng is not None:
        master = sum(u.flat_param.numel() * u.flat_param.element_size() for u in eng.units)
        lp = sum(u.lp_shard.numel() * u.lp_shard.element_size() for u in eng.units
                 if getattr(u, "lp_shard", None) is not None and u.lp_shard is not u.flat_param.data)
        gshard = sum(u._grad_shard.numel() * u._grad_shard.element_size() for u in eng.units
                     if getattr(u, "_grad_shard", None) is not None)
        gpers = sum(u._grad_persistent.numel() * u._grad_persistent.element_size() for u in eng.units
                    if getattr(u, "_grad_persistent", None) is not None)
        pools = 0
        for pool in (eng.lp_pool, eng.grad_pool):
            for lst in pool._bufs.values():
                pools += sum(b.numel() * b.element_size() for b in lst)
        out.update(engine_master_shards=master * gb, engine_compute_shards=lp * gb,
                   engine_grad_shards=(gshard + gpers) * gb, engine_pooled_buffers=pools * gb,
                   engine_units=float(len(eng.units)))
    return out
