"""Fused tensor-parallel GEMMs over NVLink peer memory (csrc/gemm/gemm_bf16.cu, kFuse = 1 / 2).

* ``ag_gemm(x_shard, w)``  : all-gather -> GEMM in ONE kernel.  A few leading CTA clusters pull the other ranks' row
  blocks of the activation from peer memory while the remaining clusters already multiply the local block; TMA
  producers wait on per-source ready counters, so the transfer of shard r+1 hides behind the tensor-core work of
  shard r.  The gathered activation is a by-product (returned for the wgrad GEMM).
* ``gemm_rs(x, w)``        : GEMM -> reduce-scatter.  The GEMM epilogue stores each bf16 partial tile directly into the
  staging slot of the rank that owns those rows (peer stores) and bumps an arrival counter; a reduce kernel sums the
  ``world`` slots in fp32 as soon as every source has delivered (optionally fusing the residual add).

These are the "compute step followed by a collective" hot ops of tensor parallelism (SURVEY 2.2 "TP", 6 roofline
table: comm-bound unless fused).  Falls back to the unfused path when the shape rules are not met
(rows per rank % 256, N % 32, K % 8, <= 8 ranks on one NVSwitch domain).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Tuple

import torch

from .. import _native as nat
from .symm_mem import SymmDomain

u64p = ctypes.POINTER(nat.u64)
nat.register_signatures({
    "tb_ag_gemm_bf16": ([u64p, u64p, nat.u64, nat.u64, nat.u64, nat.u64, nat.i32, nat.i32, nat.i32, nat.i64, nat.i64,
                         nat.i32, nat.i32, nat.i32, nat.u64, ctypes.c_uint32, nat.u64, nat.i32, ctypes.c_uint32, nat.i32,
                         nat.i32, nat.u64], nat.i32),
    "tb_gemm_rs_bf16": ([nat.u64, nat.u64, u64p, u64p, u64p, nat.i32, nat.i32, nat.i32, nat.i64, nat.i64, nat.i32,
                         nat.i32, nat.i32, nat.i32, nat.i32, ctypes.c_uint32, nat.i32, nat.u64], nat.i32),
    "tb_rs_reduce_bf16": ([nat.u64, nat.u64, ctypes.c_uint32, nat.u64, nat.u64, nat.i32, nat.i32, nat.i32, nat.i64,
                           nat.i32, nat.u64], nat.i32),
})

CH_AG_GEMM, CH_GEMM_RS = 8, 9
TILE_M = 256


class FusedTP:
    """Per-process-group state of the fused kernels: symmetric gather / staging buffers, counters, epochs."""

    def __init__(self, group, device: torch.device, comm_clusters: Optional[int] = None):
        if comm_clusters is None:
            import os
            comm_clusters = int(os.environ.get("TORCHACC_B200_AG_CLUSTERS", "0"))   # 0 = per-shape heuristic
        self.domain = SymmDomain.get(group, device)
        self.device = device
        self.world, self.rank = self.domain.world, self.domain.rank
        self.comm_clusters = comm_clusters
        self._gather: Dict[Tuple[int, int], torch.Tensor] = {}
        self._stage: Dict[Tuple[int, int], torch.Tensor] = {}
        self.flags = torch.zeros(8, dtype=torch.int32, device=device)          # local per-source ready counters
        self.flag_calls = 0
        self.counters = self.domain.alloc(64, torch.int32)                      # peers bump these (symmetric)
        self.counter_expected = 0
        self.block_counter = torch.zeros(1, dtype=torch.int32, device=device)

    # ---- shape rules ----------------------------------------------------------------------------------------
    def ok_ag(self, rows: int, N: int, K: int, dtype) -> bool:
        return dtype == torch.bfloat16 and rows % TILE_M == 0 and N % 8 == 0 and K % 64 == 0 and self.world <= 8

    def ok_rs(self, rows: int, N: int, K: int, dtype) -> bool:
        return dtype == torch.bfloat16 and rows % TILE_M == 0 and N % 32 == 0 and K % 8 == 0 and self.world <= 8

    def gather_buffer(self, rows: int, K: int) -> torch.Tensor:
        key = (rows, K)
        if key not in self._gather:
            self._gather[key] = self.domain.alloc(self.world * rows * K, torch.bfloat16).view(self.world * rows, K)
        return self._gather[key]

    # ---- all-gather -> GEMM ------------------------------------------------------------------------------------
    def ag_gemm(self, x_shard: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
                b_mn_major: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
        """x_shard [rows, K] (this rank's tokens), w [N, K] (or [K, N] when ``b_mn_major``).
        Returns (y [world*rows, N], x_full [world*rows, K])."""
        rows, K = x_shard.shape
        N = w.shape[1] if b_mn_major else w.shape[0]
        full = self.gather_buffer(rows, K)
        full[self.rank * rows:(self.rank + 1) * rows].copy_(x_shard)
        y = torch.empty((self.world * rows, N), dtype=x_shard.dtype, device=x_shard.device)
        d = self.domain
        buf = d.find(full)
        # copy clusters: a short GEMM (small N) has little math to hide the transfer behind -> more copy CTAs;
        # a long one prefers the SMs for tensor work
        cc = self.comm_clusters if self.comm_clusters > 0 else (8 if N <= 4096 else 4)
        self.flag_total = getattr(self, "flag_total", 0) + cc * 2
        self.flag_calls += 1
        L = nat.require()
        nat.check(
            L.tb_ag_gemm_bf16(buf.peer_ptrs, d.pad_ptrs, full.data_ptr(), w.data_ptr(), y.data_ptr(), nat.ptr(bias), rows,
                              N, K, w.stride(0), y.stride(0), int(b_mn_major), self.rank, self.world,
                              self.flags.data_ptr(), self.flag_total,
                              self.block_counter.data_ptr(), CH_AG_GEMM, d.next_epoch(CH_AG_GEMM), cc,
                              nat.num_sms(), nat.stream()), "tb_ag_gemm_bf16")
        nat.count_launch()
        return y, full

    # ---- GEMM -> reduce-scatter --------------------------------------------------------------------------------
    def gemm_rs(self, x: torch.Tensor, w: torch.Tensor, a_mn_major: bool = False, b_mn_major: bool = False,
                residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x [world*rows, K] (or [K, world*rows] if ``a_mn_major``), w [N, K] (or [K, N]).
        Returns this rank's reduced row block [rows, N] (+ residual)."""
        M = x.shape[1] if a_mn_major else x.shape[0]
        K = x.shape[0] if a_mn_major else x.shape[1]
        N = w.shape[1] if b_mn_major else w.shape[0]
        rows = M // self.world
        key = (rows, N)
        slot = rows * ((N + 255) // 256 * 256)       # row-major slots, N padded to the 256-column tile
        if key not in self._stage:
            self._stage[key] = self.domain.alloc(self.world * slot, torch.bfloat16)
        stage = self._stage[key]
        d = self.domain
        sbuf, cbuf = d.find(stage), d.find(self.counters)
        tiles = (rows // 128) * ((N + 255) // 256)
        self.counter_expected += tiles * 8          # 2 MMA warpgroups x 4 warps per 128-row tile
        L = nat.require()
        nat.check(
            L.tb_gemm_rs_bf16(x.data_ptr(), w.data_ptr(), sbuf.peer_ptrs, cbuf.peer_ptrs, d.pad_ptrs, rows, N, K,
                              x.stride(0), w.stride(0), int(a_mn_major), int(b_mn_major), self.rank, self.world,
                              CH_GEMM_RS, d.next_epoch(CH_GEMM_RS), nat.num_sms(), nat.stream()), "tb_gemm_rs_bf16")
        out = torch.empty((rows, N), dtype=torch.bfloat16, device=x.device)
        nat.check(
            L.tb_rs_reduce_bf16(stage.data_ptr(), self.counters.data_ptr(), self.counter_expected, nat.ptr(residual),
                                out.data_ptr(), rows, N, self.world, slot, nat.num_sms(), nat.stream()),
            "tb_rs_reduce_bf16")
        nat.count_launch(2)
        return out


def make_fused_tp(group, device) -> Optional[FusedTP]:
    """FusedTP for ``group`` if the kernels and a symmetric-memory domain are available, else None."""
    import os
    from .symm_mem import symm_available
    if os.environ.get("TORCHACC_B200_FUSED_TP", "1") == "0" or device.type != "cuda":
        return None
    L = nat.lib()
    if L is None or not hasattr(L, "tb_ag_gemm_bf16") or group is None or not symm_available(group):
        return None
    return FusedTP(group, device)
