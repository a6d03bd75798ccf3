"""Python side of the symmetric-memory communication runtime (csrc/comm/symm_comm.cu).

``SymmDomain`` (one per process group, <= 8 ranks on one NVSwitch domain):
  * allocates communication buffers with the native allocator, exchanges their CUDA-IPC handles over
    ``torch.distributed`` and maps every peer's buffer locally (peer pointers are what the kernels take);
  * owns the signal pad (epoch flags) and per-channel epoch counters.
``SymmCollectives`` plugs into the sharding engines (parallel/collectives.py): parameter shards and gradient
buffers are *allocated inside* the domain, so all-gather / reduce-scatter are single kernels that pull from peer
memory -- no staging copies and no NCCL.  Anything that does not satisfy the kernels' alignment rules falls back to
NCCL on the same group.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from .. import _native as nat
from .collectives import Collectives, NcclCollectives

nat.register_signatures({
    "tb_symm_alloc": ([nat.i64, ctypes.POINTER(nat.u64)], nat.i32),
    "tb_symm_free": ([nat.u64], nat.i32),
    "tb_symm_get_handle": ([nat.u64, ctypes.c_void_p], nat.i32),
    "tb_symm_open_handle": ([ctypes.c_void_p, ctypes.POINTER(nat.u64)], nat.i32),
    "tb_symm_close_handle": ([nat.u64], nat.i32),
    "tb_symm_all_gather": ([ctypes.POINTER(nat.u64), ctypes.POINTER(nat.u64), nat.i64, nat.u64, nat.i64, nat.i32,
                            nat.i32, nat.i32, ctypes.c_uint32, nat.u64, nat.i32, nat.u64], nat.i32),
    "tb_symm_reduce_scatter": ([ctypes.POINTER(nat.u64), ctypes.POINTER(nat.u64), nat.i64, nat.u64, nat.i64, nat.i32,
                                nat.i32, nat.f32, nat.i32, nat.i32, nat.i32, ctypes.c_uint32, nat.u64, nat.i32,
                                nat.u64], nat.i32),
    "tb_symm_all_to_all": ([ctypes.POINTER(nat.u64), ctypes.POINTER(nat.u64), nat.i64, nat.u64, nat.i64, nat.i32,
                            nat.i32, nat.i32, ctypes.c_uint32, nat.u64, nat.i32, nat.u64], nat.i32),
})

# Channel map of a domain's signal pad (64 channels x 16 slots): 0-3 first SymmCollectives instance (all-gather,
# reduce-scatter, all-reduce, all-to-all), 4-7 carried collectives (parallel/carry.py), 8-9 fused TP GEMMs, 16+4k..19+4k
# the k-th further SymmCollectives instance.  The device protocol requires the collectives of ONE channel to run in the
# same order on every rank; two users that issue from different streams (the engine's gradient all-reduce on its
# reduce stream, ring attention's reduce-scatter on the compute stream) therefore get their own channel block
# (found with the bounded spins on 8 GPUs).
CH_ALL_GATHER, CH_REDUCE_SCATTER, CH_ALL_REDUCE, CH_ALL_TO_ALL, CH_USER0 = 0, 1, 2, 3, 8
_FIRST_EXTRA_BLOCK, _MAX_BLOCKS = 16, 12
_PAD_BYTES = 64 * 16 * 4


class _RawCuda:
    """Exposes a raw device allocation through ``__cuda_array_interface__`` so torch can view it zero-copy."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class SymmBuffer:
    """A buffer that exists at the same logical place on every rank of the domain."""

    def __init__(self, domain: "SymmDomain", nbytes: int):
        L = nat.require()
        self.domain, self.nbytes = domain, nbytes
        p = nat.u64()
        nat.check(L.tb_symm_alloc(nbytes, ctypes.byref(p)), "tb_symm_alloc")
        self.ptr = p.value
        handle = ctypes.create_string_buffer(64)
        nat.check(L.tb_symm_get_handle(self.ptr, handle), "tb_symm_get_handle")
        handles: List[bytes] = [None] * domain.world
        dist.all_gather_object(handles, handle.raw, group=domain.group)
        self.peer_ptrs = (nat.u64 * domain.world)()
        self._opened = []
        for r, h in enumerate(handles):
            if r == domain.rank:
                self.peer_ptrs[r] = self.ptr
            else:
                q = nat.u64()
                hb = ctypes.create_string_buffer(h, 64)
                nat.check(L.tb_symm_open_handle(hb, ctypes.byref(q)), "tb_symm_open_handle")
                self.peer_ptrs[r] = q.value
                self._opened.append(q.value)
        self._holder = _RawCuda(self.ptr, nbytes)
        self.bytes = torch.as_tensor(self._holder, device=domain.device)

    def tensor(self, dtype: torch.dtype, numel: Optional[int] = None, offset_bytes: int = 0) -> torch.Tensor:
        t = self.bytes[offset_bytes:].view(dtype)
        return t if numel is None else t[:numel]

    def contains(self, t: torch.Tensor) -> bool:
        return self.ptr <= t.data_ptr() and t.data_ptr() + t.numel() * t.element_size() <= self.ptr + self.nbytes

    def close(self) -> None:
        """Unmap the peers' allocations and free ours.  Only through ``SymmDomain.close`` (a collective): a peer must not
        still be reading this buffer, and no tensor view of it may be used afterwards."""
        if self.ptr == 0:
            return
        L = nat.require()
        for q in self._opened:
            L.tb_symm_close_handle(q)
        self._opened = []
        self.bytes = None
        self._holder = None
        L.tb_symm_free(self.ptr)
        self.ptr = 0


class SymmDomain:
    _domains: Dict[int, "SymmDomain"] = {}

    def __init__(self, group, device: torch.device):
        self.group, self.device = group, device
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.world > 8:
            raise RuntimeError("symmetric-memory domains cover at most 8 ranks (one NVSwitch domain)")
        self.buffers: List[SymmBuffer] = []
        self.pad = SymmBuffer(self, _PAD_BYTES)
        self.pad_ptrs = self.pad.peer_ptrs
        self.counters = torch.zeros(64, dtype=torch.int32, device=device)
        self.epochs = [0] * 64
        self._blocks = 0
        dist.barrier(group=group, device_ids=[device.index])

    @classmethod
    def get(cls, group, device) -> "SymmDomain":
        key = id(group)
        if key not in cls._domains:
            cls._domains[key] = SymmDomain(group, device)
        return cls._domains[key]

    def close(self) -> None:
        """Collective teardown of the domain: device work drained on every rank, then every mapping is closed and every
        allocation freed.  Engines / collectives built on the domain must not be used afterwards.  Not called
        automatically (the reference's NCCL communicators are not destroyed at exit either); long-lived services that
        rebuild their process groups call it before dropping a group."""
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group, device_ids=[self.device.index])
        for b in self.buffers + [self.pad]:
            b.close()
        self.buffers = []
        for key, d in list(SymmDomain._domains.items()):
            if d is self:
                del SymmDomain._domains[key]

    @classmethod
    def close_all(cls) -> None:
        for d in list(cls._domains.values()):
            d.close()

    def alloc(self, numel: int, dtype: torch.dtype) -> torch.Tensor:
        """Collective: every rank must call with the same size, in the same order."""
        nbytes = (numel * torch.empty(0, dtype=dtype).element_size() + 255) // 256 * 256
        buf = SymmBuffer(self, nbytes)
        self.buffers.append(buf)
        t = buf.tensor(dtype, numel)
        t._tb_symm = buf
        return t

    def find(self, t: torch.Tensor) -> Optional[SymmBuffer]:
        b = getattr(t, "_tb_symm", None)
        if b is not None and b.contains(t):
            return b
        for b in self.buffers:
            if b.contains(t):
                return b
        return None

    def channel_block(self) -> int:
        """Base channel of a fresh block of 4 (collective: every rank creates its instances in the same order)."""
        k = self._blocks
        self._blocks += 1
        if k == 0:
            return 0
        # blocks are recycled round-robin past the 12th extra instance (long test sessions re-create engines; only
        # instances that are active at the same time on different streams must not share a block)
        return _FIRST_EXTRA_BLOCK + 4 * ((k - 1) % _MAX_BLOCKS)

    def next_epoch(self, ch: int) -> int:
        self.epochs[ch] += 1
        return self.epochs[ch]

    def counter_ptr(self, ch: int) -> int:
        return self.counters.data_ptr() + 4 * ch


def symm_available(group) -> bool:
    L = nat.lib()
    if L is None or not hasattr(L, "tb_symm_all_gather") or not torch.cuda.is_available():
        return False
    world = dist.get_world_size(group)
    if world > 8 or world > torch.cuda.device_count():
        return False  # spans nodes
    import os
    return os.environ.get("TORCHACC_B200_SYMM", "1") != "0"


class SymmCollectives(Collectives):
    name = "symm"

    def __init__(self, group, world, rank, device):
        super().__init__(group, world, rank)
        self.device = device
        self.domain = SymmDomain.get(group, device)
        self.nccl = NcclCollectives(group, world, rank)
        self._staging: Dict[tuple, torch.Tensor] = {}
        self.ch0 = self.domain.channel_block()          # this instance's channels: ch0 + {AG, RS, AR, A2A}

    # buffers the engines hand to all_gather / reduce_scatter should come from here
    def alloc(self, numel: int, dtype: torch.dtype, device=None) -> torch.Tensor:
        return self.domain.alloc(numel, dtype)

    def _stage(self, numel, dtype, tag):
        key = (numel, dtype, tag)
        if key not in self._staging:
            self._staging[key] = self.domain.alloc(numel, dtype)
        return self._staging[key]

    def all_gather(self, shard: torch.Tensor, full: torch.Tensor) -> None:
        nbytes = shard.numel() * shard.element_size()
        if nbytes % 16 != 0 or not shard.is_contiguous() or not full.is_contiguous():
            return self.nccl.all_gather(shard, full)
        d = self.domain
        buf = d.find(shard)
        if buf is None:
            st = self._stage(shard.numel(), shard.dtype, "ag")
            st.copy_(shard)
            shard, buf = st, d.find(st)
        off = shard.data_ptr() - buf.ptr
        L = nat.require()
        nat.check(
            L.tb_symm_all_gather(buf.peer_ptrs, d.pad_ptrs, off, full.data_ptr(), nbytes, d.rank, d.world,
                                 self.ch0 + CH_ALL_GATHER, d.next_epoch(self.ch0 + CH_ALL_GATHER), d.counter_ptr(self.ch0 + CH_ALL_GATHER),
                                 nat.num_sms(), nat.stream()), "tb_symm_all_gather")
        nat.count_launch()

    def reduce_scatter(self, full: torch.Tensor, out: torch.Tensor, scale: float = 1.0) -> None:
        n = out.numel()
        ok = (full.dtype in (torch.bfloat16, torch.float32) and out.dtype in (torch.bfloat16, torch.float32)
              and n % 8 == 0 and full.numel() == n * self.world and full.is_contiguous() and out.is_contiguous())
        if not ok:
            return self.nccl.reduce_scatter(full, out, scale)
        d = self.domain
        buf = d.find(full)
        if buf is None:
            st = self._stage(full.numel(), full.dtype, "rs")
            st.copy_(full)
            full, buf = st, d.find(st)
        off = full.data_ptr() - buf.ptr
        L = nat.require()
        nat.check(
            L.tb_symm_reduce_scatter(buf.peer_ptrs, d.pad_ptrs, off, out.data_ptr(), n,
                                     int(full.dtype == torch.bfloat16), int(out.dtype == torch.float32), scale, d.rank,
                                     d.world, self.ch0 + CH_REDUCE_SCATTER, d.next_epoch(self.ch0 + CH_REDUCE_SCATTER),
                                     d.counter_ptr(self.ch0 + CH_REDUCE_SCATTER), nat.num_sms(), nat.stream()),
            "tb_symm_reduce_scatter")
        nat.count_launch()

    def all_reduce(self, t: torch.Tensor, scale: float = 1.0) -> None:
        """Small tensors: one-shot (gather everything, reduce locally).  Large: reduce-scatter + all-gather."""
        n = t.numel()
        es = t.element_size()
        if t.dtype not in (torch.float32, torch.bfloat16) or not t.is_contiguous():
            return self.nccl.all_reduce(t, scale)
        d = self.domain
        if n * es <= (1 << 20):
            pad = (-(n * es)) % 16 // es if es in (2, 4) else 0
            m = n + pad
            st = self._stage(m, t.dtype, "ar_in")
            st[:n].copy_(t)
            if pad:
                st[n:].zero_()
            gathered = torch.empty(m * self.world, dtype=t.dtype, device=t.device)
            buf = d.find(st)
            L = nat.require()
            nat.check(
                L.tb_symm_all_gather(buf.peer_ptrs, d.pad_ptrs, st.data_ptr() - buf.ptr, gathered.data_ptr(), m * es,
                                     d.rank, d.world, self.ch0 + CH_ALL_REDUCE, d.next_epoch(self.ch0 + CH_ALL_REDUCE),
                                     d.counter_ptr(self.ch0 + CH_ALL_REDUCE), nat.num_sms(), nat.stream()),
                "tb_symm_all_gather")
            nat.count_launch()
            red = gathered.view(self.world, m)[:, :n].float().sum(0)
            if scale != 1.0:
                red.mul_(scale)
            t.copy_(red.to(t.dtype))
            return
        if n % (8 * self.world) != 0:
            return self.nccl.all_reduce(t, scale)
        per = n // self.world
        st = self._stage(n, t.dtype, "ar_big")
        st.copy_(t)
        # reduced slice goes to a second symmetric buffer at the SAME offset on every rank (the all-gather kernel
        # applies one source offset to all peers)
        red = self._stage(per, t.dtype, "ar_big_out")
        self.reduce_scatter(st, red, scale)
        self.all_gather(red, t)

    def all_to_all(self, inp: torch.Tensor, out: torch.Tensor) -> None:
        """``out[r*c:(r+1)*c] = inp_of_rank_r[rank*c:(rank+1)*c]`` for equal contiguous chunks."""
        n = inp.numel()
        es = inp.element_size()
        if n % self.world != 0 or (n // self.world * es) % 16 != 0 or not inp.is_contiguous() or not out.is_contiguous():
            return dist.all_to_all_single(out, inp, group=self.group)
        d = self.domain
        buf = d.find(inp)
        if buf is None:
            st = self._stage(n, inp.dtype, "a2a")
            st.copy_(inp.reshape(-1))
            inp, buf = st, d.find(st)
        L = nat.require()
        nat.check(
            L.tb_symm_all_to_all(buf.peer_ptrs, d.pad_ptrs, inp.data_ptr() - buf.ptr, out.data_ptr(),
                                 n // self.world * es, d.rank, d.world, self.ch0 + CH_ALL_TO_ALL,
                                 d.next_epoch(self.ch0 + CH_ALL_TO_ALL), d.counter_ptr(self.ch0 + CH_ALL_TO_ALL),
                                 nat.num_sms(), nat.stream()), "tb_symm_all_to_all")
        nat.count_launch()
