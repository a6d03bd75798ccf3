"""Glue between the native models and the context-parallel attention variants."""
from __future__ import annotations

import torch

from ..rope import qk_norm_rope_qkv, rope_qkv_
from .comm import _rank, _world
from .ring import ring_attention, zigzag_positions, zigzag_split
from .two_d import context_parallel_2d
from .ulysses import ulysses


def _layout(pctx):
    mesh = pctx.cp_mesh
    mode = pctx.cp_mode or "ulysses"
    zig = mode in ("ring", "2d") and getattr(mesh, "zigzag", True)
    return mesh, mode, zig


def cp_shard_sequence(x: torch.Tensor, seq_dim: int, pctx) -> torch.Tensor:
    """Local shard of a full-sequence tensor (ids / labels) for this rank's place in the sp group."""
    mesh, mode, zig = _layout(pctx)
    g = mesh.get_sp_proc_group()
    if mode == "ring" and zig:
        return zigzag_split(x, seq_dim, g)
    cp, r = _world(g), _rank(g)
    return x.chunk(cp, dim=seq_dim)[r].contiguous() if cp > 1 else x


def cp_local_positions(batch: int, seq_local: int, pctx, device) -> torch.Tensor:
    """Global position of every local token ([batch * seq_local] int32) for RoPE."""
    mesh, mode, zig = _layout(pctx)
    g = mesh.get_sp_proc_group()
    if mode == "ring" and zig:
        pos = zigzag_positions(seq_local, g, device)
    else:
        pos = _rank(g) * seq_local + torch.arange(seq_local, device=device)
    return pos.repeat(batch).to(torch.int32)


def cp_attention_qkvpacked(qkv, hq, hk, d, batch, seq_local, rope, position_ids, pctx, causal=True,
                           window_size=(-1, -1), qk_norm=None):
    """qkv: [batch*seq_local, (hq+2hk)*d] token-major local shard -> [batch*seq_local, hq*d].  ``qk_norm``:
    ``(q_weight, k_weight, eps)`` of a per-head q / k RMSNorm applied before RoPE (per token and head, so it commutes
    with the all-to-all)."""
    mesh, mode, zig = _layout(pctx)
    cos, sin = rope
    T = qkv.shape[0]

    def rope_(x, hq_, hk_, pos, seq):
        if qk_norm is not None:
            return qk_norm_rope_qkv(x, hq_, hk_, d, *qk_norm, cos, sin, pos, seq)
        return rope_qkv_(x, hq_, hk_, d, cos, sin, pos, seq)

    if mode == "ulysses":
        cp = mesh.get_sp_num()
        S = seq_local * cp
        q = qkv[:, :hq * d].reshape(batch, seq_local, hq, d)
        k = qkv[:, hq * d:(hq + hk) * d].reshape(batch, seq_local, hk, d)
        v = qkv[:, (hq + hk) * d:].reshape(batch, seq_local, hk, d)

        def rope_full(q_, k_, v_):
            # full sequences, a slice of the heads: plain positions 0..S-1
            B_, S_, hq_, _ = q_.shape
            hk_ = k_.shape[2]
            packed = torch.cat([q_.reshape(B_ * S_, hq_ * d), k_.reshape(B_ * S_, hk_ * d),
                                v_.reshape(B_ * S_, hk_ * d)], 1).contiguous()
            packed = rope_(packed, hq_, hk_, None, S_)
            q2 = packed[:, :hq_ * d].reshape(B_, S_, hq_, d)
            k2 = packed[:, hq_ * d:(hq_ + hk_) * d].reshape(B_, S_, hk_, d)
            v2 = packed[:, (hq_ + hk_) * d:].reshape(B_, S_, hk_, d)
            return q2, k2, v2

        out = ulysses(q, k, v, causal=causal, window_size=window_size, process_group=mesh.get_sp_proc_group(),
                      rope_func=rope_full)
        return out.reshape(T, hq * d)
    # ring / 2d: RoPE on the local tokens with their global positions, then blockwise attention
    pos = position_ids if position_ids is not None else cp_local_positions(batch, seq_local, pctx, qkv.device)
    qkv = rope_(qkv, hq, hk, pos, seq_local)
    q = qkv[:, :hq * d].reshape(batch, seq_local, hq, d)
    k = qkv[:, hq * d:(hq + hk) * d].reshape(batch, seq_local, hk, d)
    v = qkv[:, (hq + hk) * d:].reshape(batch, seq_local, hk, d)
    if mode == "ring":
        out = ring_attention(q, k, v, causal=causal, window_size=window_size, process_group=mesh.get_sp_proc_group(),
                             zigzag=zig)
    else:
        out = context_parallel_2d(q, k, v, causal=causal, window_size=window_size,
                                  inter_process_group=mesh.get_ring_proc_group(),
                                  intra_process_group=mesh.get_ulysses_proc_group(), zigzag=False)
    return out.reshape(T, hq * d)
