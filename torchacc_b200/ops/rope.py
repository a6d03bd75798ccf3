"""Rotary position embedding (rotate-half / HF Llama convention), applied IN PLACE and strided so it runs
directly on the q and k slices of the fused-QKV GEMM output.  Replaces liger's Triton RoPE
(reference torchacc/ops/liger.py:69-70,121-122)."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import _native as nat


def rope_tables(max_pos: int, dim: int, theta: float = 10000.0, device=None,
                scaling: Optional[dict] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 cos/sin tables of shape [max_pos, dim/2].  ``scaling`` supports Llama-3 style frequency scaling
    (``{"factor", "low_freq_factor", "high_freq_factor", "original_max_position_embeddings"}``)."""
    inv = 1.0 / (theta ** (torch.arange(0, dim, 2, dtype=torch.float64, device=device) / dim))
    if scaling:
        import math
        factor = scaling.get("factor", 8.0)
        lo, hi = scaling.get("low_freq_factor", 1.0), scaling.get("high_freq_factor", 4.0)
        old = scaling.get("original_max_position_embeddings", 8192)
        wavelen = 2 * math.pi / inv
        smooth = ((old / wavelen) - lo) / (hi - lo)
        scaled = torch.where(wavelen > old / lo, inv / factor,
                             torch.where(wavelen < old / hi, inv, (1 - smooth) * inv / factor + smooth * inv))
        inv = scaled
    t = torch.arange(max_pos, dtype=torch.float64, device=device)
    f = torch.outer(t, inv)
    return f.cos().float().contiguous(), f.sin().float().contiguous()


def _rope_ref(x, cos, sin, positions, sign):
    # x: [T, nheads, D]
    T, nh, D = x.shape
    half = D // 2
    pos = positions.long() if positions is not None else torch.arange(T, device=x.device) % cos.shape[0]
    c = cos[pos].unsqueeze(1)
    s = sin[pos].unsqueeze(1) * sign
    xf = x.float()
    x1, x2 = xf[..., :half], xf[..., half:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).to(x.dtype)


def _apply_inplace(x3: torch.Tensor, cos, sin, positions, seq_len: int, backward: bool):
    """x3: [T, nheads, D] view with stride (ts, D, 1)."""
    T, nh, D = x3.shape
    if nat.use_native(x3) and nat.is_half(x3) and D % 16 == 0 and x3.stride(2) == 1 \
            and x3.stride(1) == D and x3.stride(0) % 8 == 0:
        L = nat.require()
        nat.check(
            L.tb_rope_inplace(x3.data_ptr(), cos.data_ptr(), sin.data_ptr(), nat.ptr(positions), T, nh, D,
                              x3.stride(0), seq_len, int(backward), nat.num_sms(), nat.stream(),
                              nat.bf16_flag(x3)), "tb_rope_inplace")
        nat.count_launch()
    else:
        pos = positions
        if pos is None:
            pos = torch.arange(T, device=x3.device) % seq_len
        x3.copy_(_rope_ref(x3, cos, sin, pos, -1.0 if backward else 1.0))


class _RopeFn(torch.autograd.Function):
    """In-place RoPE on q and k (both views may alias one fused QKV buffer)."""

    @staticmethod
    def forward(ctx, q, k, cos, sin, positions, seq_len):
        _apply_inplace(q, cos, sin, positions, seq_len, False)
        _apply_inplace(k, cos, sin, positions, seq_len, False)
        ctx.mark_dirty(q, k)
        ctx.save_for_backward(cos, sin, positions) if positions is not None else ctx.save_for_backward(cos, sin)
        ctx.has_pos = positions is not None
        ctx.seq_len = seq_len
        return q, k

    @staticmethod
    def backward(ctx, dq, dk):
        if ctx.has_pos:
            cos, sin, positions = ctx.saved_tensors
        else:
            (cos, sin), positions = ctx.saved_tensors, None
        dq = dq.clone(memory_format=torch.contiguous_format)
        dk = dk.clone(memory_format=torch.contiguous_format)
        _apply_inplace(dq, cos, sin, positions, ctx.seq_len, True)
        _apply_inplace(dk, cos, sin, positions, ctx.seq_len, True)
        return dq, dk, None, None, None, None


class _RopeOneFn(torch.autograd.Function):
    """In-place RoPE on ONE tensor that may be a view of another tensor (autograd allows an in-place custom Function on
    a view only when it returns a single tensor -- the HF attention modules hand over views of their projections)."""

    @staticmethod
    def forward(ctx, x, cos, sin, positions, seq_len):
        _apply_inplace(x, cos, sin, positions, seq_len, False)
        ctx.mark_dirty(x)
        ctx.save_for_backward(cos, sin, positions) if positions is not None else ctx.save_for_backward(cos, sin)
        ctx.has_pos = positions is not None
        ctx.seq_len = seq_len
        return x

    @staticmethod
    def backward(ctx, dx):
        if ctx.has_pos:
            cos, sin, positions = ctx.saved_tensors
        else:
            (cos, sin), positions = ctx.saved_tensors, None
        dx = dx.clone(memory_format=torch.contiguous_format)
        _apply_inplace(dx, cos, sin, positions, ctx.seq_len, True)
        return dx, None, None, None, None


def apply_rope(q: torch.Tensor, k: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor,
               positions: Optional[torch.Tensor] = None, seq_len: Optional[int] = None):
    """q: [T, Hq, D], k: [T, Hk, D] (token-major, may be strided views).  Returns rotated (q, k); the inputs are
    modified in place.  ``positions`` is an int32 [T] tensor, or None for ``t % seq_len``."""
    if seq_len is None:
        seq_len = cos.shape[0]
    if positions is not None and positions.dtype != torch.int32:
        positions = positions.to(torch.int32)
    return _RopeFn.apply(q, k, cos, sin, positions, seq_len)


class _RopeQKVFn(torch.autograd.Function):
    """RoPE applied in place to the q and k column blocks of a fused ``[T, (Hq + 2*Hk) * D]`` QKV tensor.
    One autograd node over the whole buffer (no view bookkeeping); backward rotates the incoming gradient in
    place with ``-sin``."""

    @staticmethod
    def forward(ctx, qkv, hq, hk, d, cos, sin, positions, seq_len):
        T = qkv.shape[0]
        q = qkv.as_strided((T, hq, d), (qkv.stride(0), d, 1), qkv.storage_offset())
        k = qkv.as_strided((T, hk, d), (qkv.stride(0), d, 1), qkv.storage_offset() + hq * d)
        _apply_inplace(q, cos, sin, positions, seq_len, False)
        _apply_inplace(k, cos, sin, positions, seq_len, False)
        ctx.mark_dirty(qkv)
        ctx.cfg = (hq, hk, d, seq_len)
        ctx.has_pos = positions is not None
        if positions is not None:
            ctx.save_for_backward(cos, sin, positions)
        else:
            ctx.save_for_backward(cos, sin)
        return qkv

    @staticmethod
    def backward(ctx, dqkv):
        hq, hk, d, seq_len = ctx.cfg
        if ctx.has_pos:
            cos, sin, positions = ctx.saved_tensors
        else:
            (cos, sin), positions = ctx.saved_tensors, None
        # the incoming gradient belongs to autograd (it may be shared / inspected by the caller): rotate a copy
        dqkv = dqkv.clone(memory_format=torch.contiguous_format)
        T = dqkv.shape[0]
        dq = dqkv.as_strided((T, hq, d), (dqkv.stride(0), d, 1), dqkv.storage_offset())
        dk = dqkv.as_strided((T, hk, d), (dqkv.stride(0), d, 1), dqkv.storage_offset() + hq * d)
        _apply_inplace(dq, cos, sin, positions, seq_len, True)
        _apply_inplace(dk, cos, sin, positions, seq_len, True)
        return dqkv, None, None, None, None, None, None, None


def rope_qkv_(qkv: torch.Tensor, num_q_heads: int, num_kv_heads: int, head_dim: int, cos: torch.Tensor,
              sin: torch.Tensor, positions: Optional[torch.Tensor] = None, seq_len: Optional[int] = None):
    """In-place RoPE on a fused QKV activation ``[T, (Hq + 2 Hk) D]`` (layout q | k | v along the last dim)."""
    if seq_len is None:
        seq_len = cos.shape[0]
    if positions is not None and positions.dtype != torch.int32:
        positions = positions.to(torch.int32)
    return _RopeQKVFn.apply(qkv, num_q_heads, num_kv_heads, head_dim, cos, sin, positions, seq_len)


class _QKNormRopeQKVFn(torch.autograd.Function):
    """Per-head RMSNorm (own weight for q and for k) then RoPE on a fused QKV buffer, out of place, one kernel each way.
    The pre-norm input and the per-row rstd are saved; the weight gradients come from fp32 per-CTA partials summed
    here (no atomics)."""

    @staticmethod
    def forward(ctx, qkv, q_weight, k_weight, hq, hk, d, eps, cos, sin, positions, seq_len):
        T = qkv.shape[0]
        out = torch.empty_like(qkv)
        rstd = torch.empty((T, hq + hk), dtype=torch.float32, device=qkv.device)
        L = nat.require()
        nat.check(
            L.tb_qk_norm_rope_fwd(qkv.data_ptr(), out.data_ptr(), q_weight.data_ptr(), k_weight.data_ptr(),
                                  rstd.data_ptr(), cos.data_ptr(), sin.data_ptr(), nat.ptr(positions), T, hq, hk, d,
                                  qkv.stride(0), seq_len, eps, nat.num_sms(), nat.stream(), nat.bf16_flag(qkv)),
            "tb_qk_norm_rope_fwd")
        nat.count_launch()
        ctx.cfg = (hq, hk, d, seq_len)
        ctx.save_for_backward(qkv, q_weight, k_weight, rstd, cos, sin, positions)
        return out

    @staticmethod
    def backward(ctx, g):
        hq, hk, d, seq_len = ctx.cfg
        qkv, q_weight, k_weight, rstd, cos, sin, positions = ctx.saved_tensors
        T = qkv.shape[0]
        g = g.contiguous()
        dqkv = torch.empty_like(qkv)
        # one fp32 [2, d] partial per CTA (q, k); two resident CTAs per SM, fewer when there are fewer rows of heads
        rows_per_cta = 256 // _qk_group(d)
        parts = max(1, min(nat.num_sms() * 2, -(-T * (hq + 2 * hk) // rows_per_cta)))
        dw_part = torch.empty((parts, 2, d), dtype=torch.float32, device=qkv.device)
        L = nat.require()
        nat.check(
            L.tb_qk_norm_rope_bwd(g.data_ptr(), qkv.data_ptr(), dqkv.data_ptr(), q_weight.data_ptr(),
                                  k_weight.data_ptr(), rstd.data_ptr(), dw_part.data_ptr(), parts, cos.data_ptr(),
                                  sin.data_ptr(), nat.ptr(positions), T, hq, hk, d, qkv.stride(0), seq_len,
                                  nat.num_sms(), nat.stream(), nat.bf16_flag(qkv)),
            "tb_qk_norm_rope_bwd")
        nat.count_launch()
        dw = dw_part.sum(0)
        return (dqkv, dw[0].to(q_weight.dtype), dw[1].to(k_weight.dtype), None, None, None, None, None, None, None,
                None)


def _qk_group(d: int) -> int:
    """Lanes per head row in the fused kernel: d / 16 rounded up to a power of two."""
    g = 1
    while g < d // 16:
        g *= 2
    return g


def _qk_norm_rope_ref(qkv, hq, hk, d, q_weight, k_weight, eps, cos, sin, positions, seq_len):
    from .rmsnorm import rmsnorm_ref
    T = qkv.shape[0]
    pos = positions if positions is not None else torch.arange(T, device=qkv.device) % seq_len
    q = rmsnorm_ref(qkv[:, :hq * d].reshape(T, hq, d), q_weight, eps)[0]
    k = rmsnorm_ref(qkv[:, hq * d:(hq + hk) * d].reshape(T, hk, d), k_weight, eps)[0]
    q, k = _rope_ref(q, cos, sin, pos, 1.0), _rope_ref(k, cos, sin, pos, 1.0)
    return torch.cat([q.reshape(T, hq * d), k.reshape(T, hk * d), qkv[:, (hq + hk) * d:]], 1)


def qk_norm_rope_qkv(qkv: torch.Tensor, num_q_heads: int, num_kv_heads: int, head_dim: int, q_weight: torch.Tensor,
                     k_weight: torch.Tensor, eps: float, cos: torch.Tensor, sin: torch.Tensor,
                     positions: Optional[torch.Tensor] = None, seq_len: Optional[int] = None) -> torch.Tensor:
    """Qwen3's per-head q / k RMSNorm followed by RoPE on a fused QKV activation ``[T, (Hq + 2 Hk) D]`` (q | k | v along
    the last dim).  Returns a new tensor: q and k rows are normalised with ``q_weight`` / ``k_weight`` ([D] each) and
    rotated, V is copied.  The norm and the rotation run in fp32 with one rounding at the end."""
    if seq_len is None:
        seq_len = cos.shape[0]
    if positions is not None and positions.dtype != torch.int32:
        positions = positions.to(torch.int32)
    if nat.use_native(qkv, q_weight, k_weight) and nat.is_half(qkv, q_weight, k_weight) and head_dim % 16 == 0 \
            and head_dim <= 256 and qkv.dim() == 2 and qkv.shape[1] == (num_q_heads + 2 * num_kv_heads) * head_dim:
        qkv = qkv.contiguous()
        return _QKNormRopeQKVFn.apply(qkv, q_weight.contiguous(), k_weight.contiguous(), num_q_heads, num_kv_heads,
                                      head_dim, eps, cos, sin, positions, seq_len)
    return _qk_norm_rope_ref(qkv, num_q_heads, num_kv_heads, head_dim, q_weight, k_weight, eps, cos, sin, positions,
                             seq_len)
