"""Flat-parameter sharding engine: FSDP (ZeRO-3), HSDP and bucketed DP in one implementation.

Capability parity: reference torchacc/dist/fsdp.py:135-241 (which delegates to torch FSDP1 / XLA-FSDP) and
dist/dp.py:20-89 (torch DDP).  This is our own runtime, not a wrapper:

* every wrapped module ("unit", chosen by ``wrap_layer_cls``) owns ONE flat vector holding all of its parameters,
  padded to a multiple of ``128 * world`` (the reference's checkpoint padding rule, state_dict_utils.py:355-357);
* the optimizer sees one fp32 ``flat_param`` shard per unit (``model.parameters()``); compute uses a bf16 copy:
  ``lp_shard`` (own slice) gathered into ``lp_full`` right before the unit runs.  ``FusedAdamW`` writes the bf16
  shard in the same kernel as the update, so no separate cast pass exists;
* gradients: the wgrad GEMM epilogue writes straight into the unit's flat bf16 gradient buffer
  (``ops.linear`` + ``_tb_grad_view``); after the unit's backward the buffer is reduce-scattered with fp32
  accumulation into the fp32 gradient shard (bf16 on the wire, half the reference's fp32 reduce traffic);
* schedule: all-gathers are prefetched one unit ahead on a high-priority communication stream, reduce-scatters run
  on a second one behind the backward; on a GPU both are *queued* at unit boundaries and *started* at the next
  communication window (the MLP of the running / recomputed layer, ``ShardingEngine.comm_window``) so they overlap
  large GEMMs instead of flash-attention and the small projections; the wgmma GEMM switches to dynamic
  scheduling (one CTA per tile) while collectives share the GPU.  Gather / gradient buffers come from small
  rotating pools so memory stays at ``2 units`` regardless of depth;
* strategies: ``FULL_SHARD`` (fsdp), ``HYBRID`` (fsdp x dp replicas), ``NO_SHARD`` (pure DP: units act as
  gradient all-reduce buckets overlapped with backward -- this is the DataParallel engine);
* gradient checkpointing (``gc``) happens INSIDE the unit, so recomputation reuses the gathered parameters
  (the reference silently drops GC on its eager FSDP path, SURVEY Appendix B #1).
"""
from __future__ import annotations

import math
from contextlib import contextmanager
from typing import Dict, Iterable, List, Optional, Sequence, Set

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.utils.checkpoint import checkpoint as torch_checkpoint

from .collectives import Collectives, make_collectives

PAD_MULTIPLE = 128


class _ParamInfo:
    __slots__ = ("module", "name", "fqn", "shape", "numel", "offset", "tensor", "is_gemm_weight")

    def __init__(self, module, name, fqn, shape, numel, offset):
        self.module, self.name, self.fqn = module, name, fqn
        self.shape, self.numel, self.offset = shape, numel, offset
        self.tensor = None
        self.is_gemm_weight = False


class _BufferPool:
    """Rotating pool of equally sized device buffers keyed by (numel, dtype)."""

    def __init__(self, device, depth: int = 2, allocator=None):
        self.device, self.depth = device, depth
        self.allocator = allocator
        self._bufs: Dict[tuple, List[torch.Tensor]] = {}
        self._events: Dict[int, Optional[torch.cuda.Event]] = {}
        self._next: Dict[tuple, int] = {}

    def acquire(self, numel: int, dtype: torch.dtype, zero: bool = False) -> torch.Tensor:
        key = (numel, dtype)
        lst = self._bufs.setdefault(key, [])
        i = self._next.get(key, 0)
        if len(lst) < self.depth:
            buf = (self.allocator(numel, dtype) if self.allocator is not None
                   else torch.zeros(numel, dtype=dtype, device=self.device))
            lst.append(buf)
            self._next[key] = len(lst) % self.depth
            return buf
        buf = lst[i]
        self._next[key] = (i + 1) % self.depth
        ev = self._events.pop(buf.data_ptr(), None)
        if ev is not None:
            torch.cuda.current_stream().wait_event(ev)
        if zero:
            buf.zero_()
        return buf

    def release(self, buf: torch.Tensor, stream=None) -> None:
        """Mark ``buf`` reusable once work queued so far on ``stream`` finishes."""
        if buf.is_cuda:
            ev = torch.cuda.Event()
            ev.record(stream if stream is not None else torch.cuda.current_stream())
            self._events[buf.data_ptr()] = ev


class FlatParamUnit:
    """All parameters of one wrapped module as a single flat, padded, sharded vector."""

    def __init__(self, engine: "ShardingEngine", module: nn.Module, prefix: str, index: int,
                 exclude: Optional[Set[int]] = None, include: Optional[Set[int]] = None):
        self.engine = engine
        self.module = module
        self.prefix = prefix
        self.index = index
        world = engine.shard_world
        infos: List[_ParamInfo] = []
        seen: Dict[int, _ParamInfo] = {}
        self.shared: List[tuple] = []  # (module, name, info) for tied parameters
        off = 0
        for mname, sub in module.named_modules():
            for pname, p in list(sub._parameters.items()):
                if p is None or (exclude and id(p) in exclude) or (include is not None and id(p) not in include):
                    continue
                if id(p) in seen:
                    self.shared.append((sub, pname, seen[id(p)]))
                    continue
                fqn = (mname + "." if mname else "") + pname
                info = _ParamInfo(sub, pname, fqn, tuple(p.shape), p.numel(), off)
                info.is_gemm_weight = ((isinstance(sub, nn.Linear) and pname == "weight")
                                       or getattr(p, "_tb_gemm_weight", False))   # MoE expert weights (ops/moe.py)
                # keep every parameter 16-byte aligned inside the flat buffer (TMA / vector loads)
                off += (p.numel() + 7) // 8 * 8
                infos.append(info)
                seen[id(p)] = info
        self.infos = infos
        self.numel = off
        mult = PAD_MULTIPLE * world
        self.padded = max(mult, (off + mult - 1) // mult * mult)
        self.shard_numel = self.padded // world
        self.param_ids = set(seen.keys())
        self._build(seen)
        # runtime state
        self.lp_full: Optional[torch.Tensor] = None
        self.grad_full: Optional[torch.Tensor] = None
        self.gathered = False
        self.gather_event = None
        self.lp_version = -1
        self._gathered_version = -1
        self.needs_post_backward = False

    @property
    def grad_accumulated(self) -> bool:
        """True while the optimizer-visible gradient of this unit holds earlier micro-batches.  Derived from the
        gradient tensors themselves (not a sticky flag), so ``optimizer.zero_grad()`` -- the reference's canonical
        loop, docs/quick_start.md / benchmarks/transformer.py:170 -- starts a fresh accumulation exactly like
        ``model.zero_grad()`` does."""
        fp = self.flat_param
        return fp.grad is not None or getattr(fp, "_tb_grad", None) is not None

    # ---- construction ---------------------------------------------------------------------------------
    @torch.no_grad()
    def _build(self, seen):
        eng = self.engine
        dev = eng.device
        world, rank = eng.shard_world, eng.shard_rank
        full = torch.zeros(self.padded, dtype=torch.float32, device=dev)
        originals = {}
        for sub in self.module.modules():
            for pname, p in sub._parameters.items():
                if p is not None and id(p) in seen:
                    originals[id(p)] = p
        for pid, info in seen.items():
            p = originals[pid]
            if p.is_meta:
                raise RuntimeError(f"parameter {info.fqn} is on the meta device; materialise the module first "
                                   "(accelerate() does this per unit when LOW_CPU_MEM_USAGE=1)")
            full[info.offset:info.offset + info.numel].copy_(p.detach().reshape(-1).to(dev, torch.float32))
        if eng.sync_module_states and eng.world_all > 1:
            dist.broadcast(full, src=dist.get_global_rank(eng.all_group, 0) if eng.all_group is not None else 0,
                           group=eng.all_group)
        shard = full[rank * self.shard_numel:(rank + 1) * self.shard_numel].clone()
        self.flat_param = nn.Parameter(shard, requires_grad=True)       # fp32 master shard (optimizer-visible)
        self.flat_param._tb_unit = self
        lp_dtype = eng.compute_dtype
        if lp_dtype == torch.float32:
            self.lp_shard = self.flat_param.data                        # fp32 training: no separate copy
        else:
            # the bf16 shard is what peers pull during the all-gather: allocate it where they can reach it
            self.lp_shard = eng.shard_coll.alloc(self.shard_numel, lp_dtype, dev) if hasattr(eng.shard_coll, "domain") \
                else torch.empty(self.shard_numel, dtype=lp_dtype, device=dev)
            self.lp_shard.copy_(shard)
            self.flat_param._tb_lp_shard = self.lp_shard
        self.lp_version = self.flat_param._version
        if world == 1:
            self.persistent_full = self.lp_shard                        # already the full vector
        elif not eng.reshard or eng.keep_gathered:
            self.persistent_full = full.to(lp_dtype)
        else:
            self.persistent_full = None
        # replace module parameters by plain leaf tensors that view the (current) full buffer
        for pid, info in seen.items():
            p = originals[pid]
            t = torch.empty(0, dtype=lp_dtype, device=dev).requires_grad_(p.requires_grad)
            info.tensor = t
            del info.module._parameters[info.name]
            setattr(info.module, info.name, t)
        for sub, pname, info in self.shared:
            if pname in sub._parameters:
                del sub._parameters[pname]
            setattr(sub, pname, info.tensor)
        del full
        if self.persistent_full is not None:
            self._point_views(self.persistent_full)

    def _point_views(self, full: torch.Tensor) -> None:
        for info in self.infos:
            info.tensor.data = full[info.offset:info.offset + info.numel].view(info.shape)

    def _drop_views(self) -> None:
        empty = self.engine._empty
        for info in self.infos:
            info.tensor.data = empty

    # ---- parameter all-gather -------------------------------------------------------------------------
    def refresh_lp_shard(self) -> None:
        """Re-cast the master shard if an optimizer other than FusedAdamW updated it."""
        fp = self.flat_param
        if self.engine.compute_dtype != torch.float32 and getattr(fp, "_tb_lp_version", self.lp_version) != fp._version:
            with torch.no_grad():
                self.lp_shard.copy_(fp.data)
        self.lp_version = fp._version
        fp._tb_lp_version = fp._version

    def gather(self, prefetch: bool = False, background: bool = False) -> None:
        """Make ``lp_full`` valid (asynchronously on the gather stream when sharded; as a job carried by the following
        GEMM kernels when the engine runs carried collectives)."""
        eng = self.engine
        if self.gathered and eng.keep_gathered and eng.shard_world > 1 and \
                self._gathered_version != self.flat_param._version:
            self.gathered = False          # an optimizer rewrote the shard since the kept copy was gathered
        if self.gathered:
            return
        self.refresh_lp_shard()
        self._gathered_version = self.flat_param._version
        if eng.carry is not None and (self.persistent_full is None or eng.keep_gathered):
            eng.publish_params_once()
            buf = self.persistent_full if self.persistent_full is not None else \
                eng.lp_pool.acquire(self.padded, eng.compute_dtype)
            self._gather_job = eng.carry.push_gather(self.lp_shard, buf, background=background)
            self.gather_event = None
            self.lp_full = buf
            self.gathered = True
            if not prefetch:
                self.finish_gather()
            return
        if self.persistent_full is not None:
            if eng.shard_world > 1:   # NO_SHARD-after-forward mode keeps a full copy: refresh it by all-gather
                with eng.on_gather_stream():
                    eng.shard_coll.all_gather(self.lp_shard, self.persistent_full)
                    self.gather_event = eng.record_gather_event()
            self.lp_full = self.persistent_full
            self.gathered = True
            return
        with eng.on_gather_stream():
            buf = eng.lp_pool.acquire(self.padded, eng.compute_dtype)
            eng.shard_coll.all_gather(self.lp_shard, buf)
            self.gather_event = eng.record_gather_event()
        self.lp_full = buf
        self.gathered = True

    def mark_params_updated(self) -> None:
        """The optimizer rewrote this unit's shard: a kept gathered copy (``keep_gathered``) is stale now."""
        if self.engine.keep_gathered and self.engine.shard_world > 1:
            self.finish_gather()
            self.gathered = False

    def finish_gather(self) -> None:
        """Carried mode: whatever part of this unit's gather no GEMM has taken yet runs now (stand-alone kernel)."""
        job = getattr(self, "_gather_job", None)
        if job is not None:
            self._gather_job = None
            jid, ch, _epoch = job
            from .carry import BACKGROUND, FOREGROUND
            left = self.engine.carry.pending(jid, BACKGROUND if ch != 4 else FOREGROUND)
            if left:
                self.engine.stats["gather_chunks_flushed"] = self.engine.stats.get("gather_chunks_flushed", 0) + left
                self.engine.carry.flush(jid, BACKGROUND if ch != 4 else FOREGROUND)

    def wait_gather(self) -> None:
        self.finish_gather()
        if self.gather_event is not None:
            torch.cuda.current_stream().wait_event(self.gather_event)
            self.gather_event = None
        if self.lp_full is not None and getattr(self, "_views_ptr", None) != self.lp_full.data_ptr():
            self._point_views(self.lp_full)
            self._views_ptr = self.lp_full.data_ptr()

    def reshard(self) -> None:
        """Free the gathered parameters (no-op when the unit keeps a persistent full copy)."""
        if not self.gathered:
            return
        if self.persistent_full is None:
            self._drop_views()
            self._views_ptr = None
            self.engine.lp_pool.release(self.lp_full)
            self.lp_full = None
            self.gathered = False
        elif self.engine.shard_world > 1:
            self.finish_gather()
            self.gathered = False  # contents go stale after the next optimizer step

    # ---- gradients ------------------------------------------------------------------------------------
    def prepare_grad_buffer(self) -> None:
        eng = self.engine
        if self.grad_full is not None:
            return
        if eng.world_data == 1:
            if getattr(self, "_grad_persistent", None) is None:
                self._grad_persistent = torch.zeros(self.padded, dtype=eng.grad_wire_dtype, device=eng.device)
            self.grad_full = self._grad_persistent
        else:
            self.grad_full = eng.grad_pool.acquire(self.padded, eng.grad_wire_dtype)
            if eng.carry is not None:
                # the previous user's reduce-scatter reads this buffer from EVERY rank: it must have been issued here
                # and finished everywhere before the wgrad epilogues write into it again
                if any(p[1].data_ptr() == self.grad_full.data_ptr() for p in eng._carry_pending_reduces):
                    eng.enqueue_delayed_reduces(0)     # pool too shallow for the configured delay: enqueue now
                prev = eng._carry_reduce_of.pop(self.grad_full.data_ptr(), None)
                if prev is not None:
                    from .carry import BACKGROUND
                    jid, ch, epoch = prev
                    left = eng.carry.pending(jid, BACKGROUND)
                    if left:
                        eng.stats["reduce_chunks_flushed"] = eng.stats.get("reduce_chunks_flushed", 0) + left
                        eng.carry.flush(jid, BACKGROUND)
                    eng.carry.wait_done(ch, epoch)
        keep = self.grad_accumulated and eng.accumulate_in_flat
        for info in self.infos:
            t = info.tensor
            if info.is_gemm_weight and t.requires_grad and eng.compute_dtype == torch.bfloat16:
                t._tb_grad_view = self.grad_full[info.offset:info.offset + info.numel].view(info.shape)
                t._tb_grad_ready = keep
            else:
                t._tb_grad_view = None

    def collect_autograd_grads(self) -> None:
        """Copy ``.grad`` of non-GEMM parameters (norm weights, biases, embeddings) into the flat buffer and
        zero whatever received no gradient at all."""
        g = self.grad_full
        accumulate = self.grad_accumulated and self.engine.accumulate_in_flat
        for info in self.infos:
            t = info.tensor
            dst = g[info.offset:info.offset + info.numel]
            if getattr(t, "_tb_grad_view", None) is not None:
                if not getattr(t, "_tb_grad_ready", False):
                    dst.zero_()
                if t.grad is not None:  # e.g. the weight was also used through a non-fused path
                    dst.add_(t.grad.reshape(-1).to(dst.dtype))
                    t.grad = None
                    self.engine.stats["wgrad_fallbacks"] = self.engine.stats.get("wgrad_fallbacks", 0) + 1
                t._tb_grad_ready = False
                continue
            if t.grad is not None:
                if accumulate:
                    dst.add_(t.grad.reshape(-1).to(dst.dtype))
                else:
                    dst.copy_(t.grad.reshape(-1))
                t.grad = None
            elif not accumulate:
                dst.zero_()
        if self.padded > self.numel and not accumulate:
            g[self.numel:].zero_()

    def reduce_grads(self) -> None:
        """Turn this unit's flat gradient buffer into the optimizer-visible gradient shard:
        single device -> the buffer itself; otherwise reduce-scatter over the shard group with fp32 accumulation
        (+ all-reduce over replicas for HSDP / DP), overlapped with the rest of backward on the reduce stream."""
        if self.stage_reduce():
            self.launch_reduce()

    def stage_reduce(self) -> bool:
        """First half of ``reduce_grads``: finish the flat buffer on the compute stream and record the event the
        collective has to wait for.  Returns False when there is nothing to communicate (single device)."""
        eng = self.engine
        self.collect_autograd_grads()
        fp = self.flat_param
        if eng.world_data == 1:
            if eng.grad_mode == "fused":
                fp._tb_grad = self.grad_full        # persistent per-unit buffer, accumulates across micro-batches
            else:
                if fp.grad is None:
                    fp.grad = self.grad_full.to(torch.float32, copy=True)   # never alias the reusable flat buffer
                else:
                    fp.grad.add_(self.grad_full)
            self.grad_full = None
            return False
        self._reduce_ready = None
        if eng.device.type == "cuda":
            self._reduce_ready = torch.cuda.Event()
            self._reduce_ready.record()
        self._reduce_src, self.grad_full = self.grad_full, None
        return True

    def launch_reduce(self) -> None:
        """Second half: the collective itself, on the reduce stream (may run long after ``stage_reduce``)."""
        eng = self.engine
        fp = self.flat_param
        src, self._reduce_src = self._reduce_src, None
        first = not self.grad_accumulated
        if getattr(self, "_grad_shard", None) is None:
            self._grad_shard = torch.empty(self.shard_numel, dtype=eng.grad_shard_dtype, device=eng.device)
        if eng.carry is not None:
            # carried by the GEMMs of the units whose backward follows: fp32 sum over ranks, 1/world scale, (+= for
            # later micro-batches) and the sum of squares for the gradient norm, all in the reducing warp
            if not eng._carry_stats_armed:
                eng.carry.arm_stats()
                eng._carry_stats_armed = True
            # the gradients are final NOW (flag to the peers); the job is enqueued `reduce_delay` units later so that
            # a peer whose backward runs a few percent slower is not waited for inside our next GEMM
            epoch = eng.carry.publish_grads()
            eng._carry_pending_reduces.append((self, src, not first, epoch))
            eng.enqueue_delayed_reduces(eng.reduce_delay)
            eng.grad_pool.release(src, torch.cuda.current_stream())
            self._reduce_ready = None
            if eng.grad_mode == "fused" or self._grad_shard.dtype != fp.dtype:
                fp._tb_grad = self._grad_shard
            else:
                fp.grad = self._grad_shard
            return
        out = self._grad_shard if first else torch.empty_like(self._grad_shard)
        scale = 1.0 / eng.world_data
        if eng.device.type == "cuda":
            # start no earlier than the point the compute stream has reached NOW (the communication window this is
            # launched from), not merely when the gradients were complete: the host runs far ahead of the device
            self._reduce_ready = torch.cuda.Event()
            self._reduce_ready.record()
        with eng.on_reduce_stream(self._reduce_ready):
            if eng.shard_world > 1:
                eng.shard_coll.reduce_scatter(src, out, scale)
            else:
                out.copy_(src)
                out.mul_(scale)
            if eng.replica_world > 1:
                eng.replica_coll.all_reduce(out)
            if not first:
                self._grad_shard.add_(out)
            if eng.device.type == "cuda":
                eng.grad_pool.release(src, torch.cuda.current_stream())
                out.record_stream(torch.cuda.current_stream())
            eng.note_reduce_done()
        self._reduce_ready = None
        if eng.grad_mode == "fused" or self._grad_shard.dtype != fp.dtype:
            fp._tb_grad = self._grad_shard
        else:
            fp.grad = self._grad_shard


class _PostBackward(torch.autograd.Function):
    """Identity on the unit's inputs; its backward runs after every gradient of the unit has been produced."""

    @staticmethod
    def forward(ctx, unit_runner, *inputs):
        ctx.runner = unit_runner
        return inputs if len(inputs) > 1 else inputs[0]

    @staticmethod
    def backward(ctx, *grads):
        ctx.runner._post_backward()
        return (None, *grads)


def _find_window_module(module: nn.Module) -> Optional[nn.Module]:
    """The sub-module of a transformer block whose start marks the "GEMM-only" part of the layer (the MLP)."""
    for name in ("mlp", "feed_forward", "ffn", "block_sparse_moe"):
        m = getattr(module, name, None)
        if isinstance(m, nn.Module):
            return m
    return None


class ShardedUnit(nn.Module):
    """Wrapper installed in place of each unit module: gather -> (checkpointed) forward -> reshard, plus the
    autograd hooks that drive backward prefetch and gradient reduction."""

    def __init__(self, engine: "ShardingEngine", module: nn.Module, unit: FlatParamUnit, use_gc: bool):
        super().__init__()
        self.__dict__["_engine"] = engine
        self.module = module
        self.__dict__["_unit"] = unit
        self.use_gc = use_gc
        unit.recomputes = bool(use_gc)
        unit.window_module = None
        if engine.comm_windows:
            win = _find_window_module(module)
            if win is not None:
                # fires in the forward AND in the checkpoint recomputation: the point after attention, where only
                # GEMM-bound work (MLP) follows -- the engine starts deferred collectives here (see comm_window)
                win.register_forward_pre_hook(lambda _m, _a, _e=engine, _u=unit: _e.comm_window(_u))
                unit.window_module = win

    @property
    def unit(self) -> FlatParamUnit:
        return self.__dict__["_unit"]

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(self.__dict__["_modules"]["module"], name)

    def forward(self, *args, **kwargs):
        eng: ShardingEngine = self.__dict__["_engine"]
        unit = self.unit
        eng.pre_forward(unit)
        grad_on = torch.is_grad_enabled()
        if grad_on:
            tensor_idx = [i for i, a in enumerate(args) if isinstance(a, torch.Tensor) and a.requires_grad]
            if tensor_idx:
                wrapped = _PostBackward.apply(self, *[args[i] for i in tensor_idx])
                if len(tensor_idx) == 1:
                    wrapped = (wrapped,)
                args = list(args)
                for i, w in zip(tensor_idx, wrapped):
                    args[i] = w
                args = tuple(args)
                unit.needs_post_backward = True
            else:
                unit.needs_post_backward = False   # root-like unit: finalised by the end-of-backward callback
                eng.register_final_callback_unit(unit)
        if self.use_gc and grad_on:
            from ..ops.swiglu import activations_recomputed_later
            with activations_recomputed_later():        # nothing saved in this pass survives: ops may skip it
                out = torch_checkpoint(self.module, *args, use_reentrant=False, **kwargs)
        else:
            out = self.module(*args, **kwargs)
        eng.post_forward(unit)
        if grad_on:
            self._hook_outputs(out)
        return out

    def _hook_outputs(self, out):
        fired = [False]

        def pre_backward(_g):
            if not fired[0]:
                fired[0] = True
                self.__dict__["_engine"].pre_backward(self.unit)
            return None

        def visit(o):
            if isinstance(o, torch.Tensor):
                if o.requires_grad:
                    o.register_hook(pre_backward)
            elif isinstance(o, (list, tuple)):
                for x in o:
                    visit(x)
            elif isinstance(o, dict):
                for x in o.values():
                    visit(x)
        visit(out)

    def _post_backward(self):
        self.__dict__["_engine"].post_backward(self.unit)


class ShardingEngine:
    """Owns units, streams, pools and the prefetch schedule for one wrapped model."""

    def __init__(self, device: torch.device, shard_group=None, replica_group=None, compute_dtype=torch.bfloat16,
                 strategy: str = "FULL_SHARD", sync_module_states: bool = False, reduce_dtype: str = "fp32",
                 prefetch: int = 1, prefer_symm: bool = True, grad_mode: str = "compat",
                 reshard_after_forward: Optional[bool] = None, model_numel: int = 0, grad_dtype: str = "compute"):
        self.device = device
        self.compute_dtype = compute_dtype
        self.strategy = strategy
        self.sync_module_states = sync_module_states
        self.prefetch = prefetch
        self.grad_mode = grad_mode          # 'compat': fp32 .grad for any torch optimizer; 'fused': _tb_grad for FusedAdamW
        init = dist.is_available() and dist.is_initialized()
        if strategy == "NO_SHARD":
            # pure DP: parameters replicated, the "replica" group carries the gradient all-reduce
            replica_group = replica_group if replica_group is not None else shard_group
            shard_group = None
        self.shard_group, self.replica_group = shard_group, replica_group
        self.shard_world = dist.get_world_size(shard_group) if (init and shard_group is not None) else 1
        self.shard_rank = dist.get_rank(shard_group) if (init and shard_group is not None) else 0
        self.replica_world = dist.get_world_size(replica_group) if (init and replica_group is not None) else 1
        self.world_data = self.shard_world * self.replica_world
        self.all_group = shard_group if shard_group is not None else replica_group
        self.world_all = self.world_data
        self.reshard = strategy in ("FULL_SHARD", "HYBRID") and self.shard_world > 1
        # keep_gathered: parameters stay sharded (ZeRO-3 memory for master weights / optimizer state / gradients) but
        # the gathered compute copy of every unit lives in its own persistent buffer from the forward until the end
        # of the backward -- one all-gather per unit and step instead of two.  Auto: on when that full copy is at most
        # 20 % of the device memory; a 70 B model falls back to re-gathering.
        self.keep_gathered = False
        if self.reshard:
            if reshard_after_forward is None:
                import os as _os0
                env = _os0.environ.get("TORCHACC_B200_RESHARD_AFTER_FORWARD", "")
                if env in ("0", "1"):
                    reshard_after_forward = env == "1"
            if reshard_after_forward is None:
                total = torch.cuda.get_device_properties(device).total_memory if device.type == "cuda" else (64 << 30)
                item = 4 if compute_dtype == torch.float32 else 2
                reshard_after_forward = not (0 < model_numel * item <= 0.2 * total)
            self.keep_gathered = not reshard_after_forward
        self.root_unit = None
        self.stats = {}                      # diagnostics (e.g. 'wgrad_fallbacks': wgrads that missed the flat buffer)
        self.shard_coll: Collectives = make_collectives(shard_group, device, prefer_symm)
        self.replica_coll: Collectives = make_collectives(replica_group, device, prefer_symm)
        # bf16 on the wire, fp32 accumulation at the destination (our kernels); plain fp32 training keeps fp32
        self.grad_wire_dtype = torch.float32 if compute_dtype == torch.float32 else compute_dtype
        # grad_dtype == "fp32": fp32 flat buffer = fp32 wgrad output, fp32 micro-batch accumulation, fp32 wire
        self.grad_flat_fp32 = grad_dtype == "fp32" and compute_dtype != torch.float32
        if self.grad_flat_fp32:
            self.grad_wire_dtype = torch.float32
        self.grad_shard_dtype = torch.float32 if reduce_dtype == "fp32" else self.grad_wire_dtype
        self.units: List[FlatParamUnit] = []
        self.lp_pool = _BufferPool(device, depth=2 + prefetch)
        symm_grad = hasattr(self.shard_coll, "domain")
        self._empty = torch.empty(0, dtype=compute_dtype, device=device)
        cuda = device.type == "cuda"
        # Carried collectives (parallel/carry.py): parameter all-gathers and gradient reduce-scatters ride inside the
        # GEMM kernels that run anyway (warp 3 of every CTA is the copy / reduce engine) -- no communication kernels
        # next to the GEMMs, no side streams.  Needs the symmetric-memory back-end and a plain FULL_SHARD group.
        self.carry = None
        self._carry_reduce_of: Dict[int, tuple] = {}
        self._carry_stats_armed = False
        self._carry_pending_reduces: List[tuple] = []      # (unit, flat gradient buffer, accumulate, entry epoch)
        self._params_published_for = -1
        import os as _os1
        self.reduce_delay = max(0, int(_os1.environ.get("TORCHACC_B200_REDUCE_DELAY", "2")))
        if cuda and self.reshard and self.replica_world == 1 and not self.grad_flat_fp32:   # carried reduce: bf16 slices
            from .carry import make_carry
            self.carry = make_carry(self.shard_coll, device)
        self.grad_pool = _BufferPool(device, depth=2 + (self.reduce_delay if self.carry is not None else 0),
                                     allocator=(self.shard_coll.alloc if symm_grad else None))
        if cuda and self.world_data > 1:
            # without carried collectives they run on side streams next to the GEMMs: claim GEMM tiles dynamically so
            # SMs that are busy with a collective CTA do not stall a whole GEMM (csrc/gemm/gemm_bf16.cu, "tile
            # iteration").  With them the GEMM owns the GPU: static striping (warp 3 is the copy engine, not a scheduler)
            from .. import _native as nat
            nat.set_gemm_scheduler(self.carry is None)
        # communication windows: on a GPU the flash-attention CTAs need whole SMs (224 KB smem) and small GEMMs are
        # the most sensitive to a concurrent collective, so prefetch all-gathers and gradient reduce-scatters are
        # not started at unit boundaries but at the next "window" = the start of an MLP, where the large GEMMs
        # follow.  TORCHACC_B200_COMM_WINDOWS=0 restores the old timing.
        import os as _os
        _cw = _os.environ.get("TORCHACC_B200_COMM_WINDOWS", "1")           # "0" off, "force" also on CPU (tests)
        self.comm_windows = bool(self.world_data > 1 and (_cw == "force" or (cuda and _cw != "0")))
        if self.carry is not None:
            self.comm_windows = False      # nothing to defer: the jobs are spread over the GEMMs by their FLOPs
        # optional "head" unit (final norm + lm_head split off the root unit, TORCHACC_B200_SPLIT_HEAD=1): its
        # gradients are complete right after the loss backward, so its reduce-scatter hides behind the whole
        # backward pass instead of sitting exposed before the optimizer with the embedding's
        self.split_head = _os.environ.get("TORCHACC_B200_SPLIT_HEAD", "1") == "1"
        self.head_unit: Optional[FlatParamUnit] = None
        self._head_staged = False
        self._deferred_prefetch: Optional[FlatParamUnit] = None
        self._deferred_reduces: List[FlatParamUnit] = []
        self._bwd_unit: Optional[FlatParamUnit] = None
        self.gather_stream = torch.cuda.Stream(device, priority=-1) if (cuda and self.shard_world > 1) else None
        self.reduce_stream = torch.cuda.Stream(device, priority=-1) if (cuda and self.world_data > 1) else None
        self.fwd_order: List[int] = []
        self._fwd_recorded = False
        self._final_units: List[FlatParamUnit] = []
        self._callback_queued = False
        self._pending_reduce = False
        self.training_step = 0

    def publish_params_once(self) -> None:
        """First gather after an optimizer step: bring every unit's bf16 shard up to date, then tell the peers ONCE
        that all shards of this rank are final (entry flag of every gather job of the step)."""
        if self._params_published_for == self.training_step:
            return
        self._params_published_for = self.training_step
        for u in self.units:
            u.refresh_lp_shard()
        self.carry.publish_params()

    def enqueue_delayed_reduces(self, keep: int) -> None:
        """Hand all but the newest ``keep`` finished gradient buffers to the carry queue."""
        while len(self._carry_pending_reduces) > keep:
            unit, src, accumulate, epoch = self._carry_pending_reduces.pop(0)
            job = self.carry.push_reduce(src, unit._grad_shard, 1.0 / self.world_data, accumulate, epoch)
            self._carry_reduce_of[src.data_ptr()] = job

    @property
    def accumulate_in_flat(self) -> bool:
        """Single device + fused optimizer: micro-batch gradients accumulate inside the flat bf16 buffer itself."""
        return self.world_data == 1 and self.grad_mode == "fused"

    def use_fused_optimizer(self, optimizer) -> None:
        """Called by FusedAdamW when it is built over this engine's flat parameters."""
        self.grad_mode = "fused"
        self._fused_optimizer = optimizer

    # ---- streams --------------------------------------------------------------------------------------
    @contextmanager
    def on_gather_stream(self):
        if self.gather_stream is None:
            yield
            return
        self.gather_stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.gather_stream):
            yield

    def record_gather_event(self):
        if self.gather_stream is None:
            return None
        ev = torch.cuda.Event()
        ev.record(self.gather_stream)
        return ev

    @contextmanager
    def on_reduce_stream(self, after_event=None):
        if self.reduce_stream is None:
            yield
            return
        if after_event is not None:
            self.reduce_stream.wait_event(after_event)
        with torch.cuda.stream(self.reduce_stream):
            yield

    def note_reduce_done(self):
        self._pending_reduce = True

    def wait_reductions(self):
        """Make the current stream wait for all queued gradient reductions (called at the end of backward)."""
        if self.reduce_stream is not None and self._pending_reduce:
            torch.cuda.current_stream().wait_stream(self.reduce_stream)
        self._pending_reduce = False

    # ---- schedule hooks -------------------------------------------------------------------------------
    def _neighbor(self, unit: FlatParamUnit, step: int) -> Optional[FlatParamUnit]:
        if not self._fwd_recorded or unit.index not in self.fwd_order:
            return None
        pos = self.fwd_order.index(unit.index) + step
        if 0 <= pos < len(self.fwd_order):
            return self.units[self.fwd_order[pos]]
        return None

    def pre_forward(self, unit: FlatParamUnit):
        if not self._fwd_recorded and unit.index not in self.fwd_order:
            self.fwd_order.append(unit.index)
        unit.gather()
        unit.wait_gather()
        if unit is self.root_unit and self.head_unit is not None:
            head = self.head_unit
            if self.carry is not None and self._fwd_recorded and len(self.fwd_order) > 2:
                # final norm + lm_head are needed after the LAST layer: their gather rides in the background of all
                # layers' GEMMs; post_forward of the last wrapped unit makes sure it is complete
                head.gather(prefetch=True, background=True)
                head._point_views(head.lp_full)
                head._views_ptr = head.lp_full.data_ptr()
            else:
                head.gather()
                head.wait_gather()
            if torch.is_grad_enabled():
                head.prepare_grad_buffer()
        if unit is self.root_unit and torch.is_grad_enabled():
            unit.prepare_grad_buffer()   # the fused linear+CE writes lm_head's wgrad during the forward pass
        for k in range(1, self.prefetch + 1):
            nxt = self._neighbor(unit, k)
            if nxt is not None:
                if k == 1 and self.comm_windows and getattr(unit, "window_module", None) is not None:
                    self._deferred_prefetch = nxt          # started by comm_window(unit)
                else:
                    nxt.gather(prefetch=True)

    def comm_window(self, unit: FlatParamUnit):
        """Start the collectives that were deferred to this unit's GEMM-only phase."""
        if self._deferred_reduces:
            pending, self._deferred_reduces = self._deferred_reduces, []
            for u in pending:
                u.launch_reduce()
            if unit is not None:
                self.stats["window_reduces"] = self.stats.get("window_reduces", 0) + len(pending)
        nxt, self._deferred_prefetch = self._deferred_prefetch, None
        if nxt is not None:
            nxt.gather(prefetch=True)
            if unit is not None:
                self.stats["window_gathers"] = self.stats.get("window_gathers", 0) + 1

    def flush_deferred(self):
        self.comm_window(None)

    def post_forward(self, unit: FlatParamUnit):
        if self.carry is not None and self.head_unit is not None and self._is_last_forward_unit(unit):
            self.head_unit.finish_gather()
        if self.reshard and not self.keep_gathered and unit is not self.root_unit \
                and not self._is_last_forward_unit(unit):
            unit.reshard()

    def _is_last_forward_unit(self, unit):
        # keep the last unit gathered: its backward starts immediately
        return self._fwd_recorded and self.fwd_order and self.fwd_order[-1] == unit.index

    def pre_backward(self, unit: FlatParamUnit):
        if not self._fwd_recorded and self.fwd_order:
            self._fwd_recorded = True
        if self._deferred_prefetch is not None:      # a forward window never came (e.g. last forward unit)
            nxt, self._deferred_prefetch = self._deferred_prefetch, None
            if nxt is not unit:
                nxt.gather(prefetch=True)
        unit.gather()
        unit.wait_gather()
        unit.prepare_grad_buffer()
        # with activation checkpointing the unit's forward is recomputed now and its window hook fires again
        windowed = self.comm_windows and getattr(unit, "window_module", None) is not None and \
            getattr(unit, "recomputes", False)
        if not windowed and self._deferred_reduces:
            self.flush_deferred()
        for k in range(1, self.prefetch + 1):
            prv = self._neighbor(unit, -k)
            if prv is not None:
                if k == 1 and windowed:
                    self._deferred_prefetch = prv
                else:
                    prv.gather(prefetch=True)
        self._queue_final_callback()

    def post_backward(self, unit: FlatParamUnit):
        head = self.head_unit
        if head is not None and not self._head_staged and head.grad_full is not None:
            # the first wrapped unit has finished its backward: the loss / final-norm backward (and their
            # AccumulateGrad nodes) ran long ago, the head's gradients are final
            self._head_staged = True
            if self.comm_windows:
                if head.stage_reduce():
                    self._deferred_reduces.append(head)
            else:
                head.reduce_grads()
        if unit.grad_full is None:
            unit.prepare_grad_buffer()
        if self.comm_windows:
            if unit.stage_reduce():                  # collect + "gradients complete" event now, collective later
                self._deferred_reduces.append(unit)
        else:
            unit.reduce_grads()
        if self.reshard and not self.keep_gathered:
            unit.reshard()

    def register_final_callback_unit(self, unit: FlatParamUnit):
        if unit not in self._final_units:
            self._final_units.append(unit)

    def _queue_final_callback(self):
        if self._callback_queued:
            return
        self._callback_queued = True
        torch.autograd.Variable._execution_engine.queue_callback(self._final_callback)

    def _final_callback(self):
        self._callback_queued = False
        head = self.head_unit
        if head is not None:
            if not self._head_staged and (head.grad_full is not None or
                                          any(i.tensor.grad is not None for i in head.infos)):
                if head.grad_full is None:
                    head.prepare_grad_buffer()
                head.reduce_grads()              # no wrapped unit ran a backward: reduce with the root
            self._head_staged = False
        self.flush_deferred()
        for unit in self._final_units:
            # units whose inputs carry no gradient (embedding/root): reduce now, after the whole backward.
            # The list persists across backward passes (1F1B runs several forwards before the first backward).
            pending = unit.grad_full is not None or any(i.tensor.grad is not None for i in unit.infos)
            if not pending:
                continue
            if unit.grad_full is None:
                unit.prepare_grad_buffer()
            unit.reduce_grads()
            if self.reshard and not self.keep_gathered:
                unit.reshard()
        for unit in self.units:  # anything still gathered from prefetch
            if self.reshard and unit.gathered:
                unit.finish_gather()
                if not self.keep_gathered:       # kept copies stay valid until an optimizer rewrites the shard
                    unit.reshard()
        if self.carry is not None:
            c = self.carry
            self.enqueue_delayed_reduces(0)
            left = c.pending()
            if left:
                self.stats["tail_chunks_flushed"] = self.stats.get("tail_chunks_flushed", 0) + left
            c.flush()                                   # the last reductions of the pass: nothing left to carry them
            # every rank has finished pulling parameter shards: the optimizer may now rewrite them
            from .carry import CH_GATHER, CH_GATHER_BG
            c.wait_done(CH_GATHER, c.last_epoch[CH_GATHER])
            c.wait_done(CH_GATHER_BG, c.last_epoch[CH_GATHER_BG])
            self._carry_stats_armed = False
        self.wait_reductions()
        self.training_step += 1

    # ---- utilities ------------------------------------------------------------------------------------
    def flat_parameters(self) -> List[nn.Parameter]:
        return [u.flat_param for u in self.units]

    def zero_grad(self, set_to_none: bool = True):
        for u in self.units:
            u.flat_param.grad = None
            u.flat_param._tb_grad = None

    def grads(self) -> List[torch.Tensor]:
        out = []
        for u in self.units:
            g = getattr(u.flat_param, "_tb_grad", None)
            if g is None:
                g = u.flat_param.grad
            if g is not None:
                out.append(g)
        return out

    @torch.no_grad()
    def clip_grad_norm_(self, max_norm: float, norm_type: float = 2.0, groups: Sequence = ()) -> torch.Tensor:
        """Global L2 clip over the sharded gradients with NO host synchronisation: per-shard sum of squares (our
        kernel), one all-reduce over the shard group (+ any extra ``groups``), coefficient kept on the device
        and consumed by FusedAdamW (``grad_scale``) or applied in place."""
        from ..ops.optim import grad_sqnorm, scale_
        assert norm_type == 2.0, "only the L2 norm is supported"
        gs = self.grads()
        c = self.carry
        if c is not None and c.stats_exact and c.reduce_jobs == len(gs) and len(gs) == len(self.units):
            stat = c.stats.clone()          # accumulated by the reduce-scatter warps: no pass over the gradients
            self.stats["fused_grad_norm"] = self.stats.get("fused_grad_norm", 0) + 1
        else:
            stat = grad_sqnorm(gs, device=self.device)
        if self.shard_world > 1:
            self.shard_coll.all_reduce(stat)
        for g in groups:
            if g is not None:
                dist.all_reduce(stat, group=g)
        norm = stat[0].sqrt()
        coef = (max_norm / (norm + 1e-6)).clamp(max=1.0).reshape(1).float()
        self.last_clip_coef = coef
        self.last_found_inf = (stat[1] > 0).float().reshape(1)
        if self.grad_mode == "compat" or not getattr(self, "_fused_optimizer", None):
            for g in gs:
                scale_(g, coef)
        else:
            self._fused_optimizer.grad_scale = coef
        return norm


def _resolve_classes(model: nn.Module, names: Iterable[str]):
    """Class names -> the set of class objects present in ``model`` (reference fsdp.py:149-153)."""
    names = set(names or ())
    found = {}
    for m in model.modules():
        if type(m).__name__ in names:
            found[type(m).__name__] = type(m)
    missing = names - set(found)
    if missing:
        raise ValueError(f"wrap/gc class name(s) {sorted(missing)} not found in the model")
    return tuple(found.values())


_HEAD_NAMES = ("lm_head", "norm", "ln_f", "final_layernorm", "final_norm")


def _head_param_ids(model: nn.Module, claimed: Set[int]) -> Set[int]:
    """Parameters of the modules that run AFTER the last wrapped unit (final norm, lm_head), found by name at the top
    levels of the model (``model.lm_head``, ``model.model.norm``, ``model.transformer.ln_f`` ...).  A parameter that is
    also used by another module (tied embeddings) stays in the root unit."""
    cands: Dict[int, nn.Parameter] = {}
    for holder in (model, getattr(model, "model", None), getattr(model, "transformer", None)):
        if not isinstance(holder, nn.Module):
            continue
        for name in _HEAD_NAMES:
            m = holder._modules.get(name)
            if isinstance(m, nn.Module) and not isinstance(m, ShardedUnit):
                for p in m.parameters():
                    if id(p) not in claimed:
                        cands[id(p)] = p
    if not cands:
        return set()
    head_mods = set()
    for holder in (model, getattr(model, "model", None), getattr(model, "transformer", None)):
        if isinstance(holder, nn.Module):
            for name in _HEAD_NAMES:
                m = holder._modules.get(name)
                if isinstance(m, nn.Module):
                    head_mods |= {id(x) for x in m.modules()}
    for sub in model.modules():
        if id(sub) in head_mods:
            continue
        for p in sub._parameters.values():
            if p is not None and id(p) in cands:
                del cands[id(p)]                       # shared with a non-head module (e.g. tied embedding)
    return set(cands)


def shard_model(model: nn.Module, engine: ShardingEngine, wrap_classes: Sequence[type] = (),
                gc_classes: Sequence[type] = (), gc_cnt: Optional[int] = None) -> nn.Module:
    """Wrap every instance of ``wrap_classes`` as its own unit and the remaining parameters as the root unit.
    Returns the root ``ShardedUnit``."""
    dev = engine.device
    idx = 0
    gc_left = [gc_cnt if gc_cnt is not None else math.inf]

    def want_gc(m):
        if gc_classes and isinstance(m, tuple(gc_classes)) and gc_left[0] > 0:
            gc_left[0] -= 1
            return True
        return False

    def recurse(parent: nn.Module, prefix: str):
        nonlocal idx
        for name, child in list(parent.named_children()):
            fq = prefix + name
            if wrap_classes and isinstance(child, tuple(wrap_classes)):
                child.to(dev) if not any(p.is_meta for p in child.parameters()) else None
                unit = FlatParamUnit(engine, child, fq, idx)
                idx += 1
                engine.units.append(unit)
                parent._modules[name] = ShardedUnit(engine, child, unit, want_gc(child))
            else:
                recurse(child, fq + ".")

    recurse(model, "")
    claimed: Set[int] = set()
    for u in engine.units:
        claimed |= u.param_ids
    for b in model.buffers():
        if not b.is_meta:
            b.data = b.data.to(dev)
    if engine.split_head and engine.world_data > 1:
        head_ids = _head_param_ids(model, claimed)
        if head_ids:
            head = FlatParamUnit(engine, model, "", idx, exclude=claimed, include=head_ids)
            idx += 1
            engine.units.append(head)
            engine.head_unit = head
            claimed |= head.param_ids
    root_unit = FlatParamUnit(engine, model, "", idx, exclude=claimed)
    engine.units.append(root_unit)
    engine.root_unit = root_unit
    root = ShardedUnit(engine, model, root_unit, False)
    # non-wrapped gc classes (gc without fsdp wrapping of the same class)
    if gc_classes:
        from ..utils.checkpoint import disable_kv_cache, gradient_checkpoint
        gradient_checkpoint(model, gc_classes, gc_left[0] if gc_left[0] != math.inf else None,
                            skip_types=(ShardedUnit,))
        disable_kv_cache(model)
    return root
