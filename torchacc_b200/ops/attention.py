"""FlashAttention API on the hand-written wgmma kernels (csrc/attn/).

Public functions keep the reference signatures (reference torchacc/ops/flash_attn.py:313-601): layout
``[B, S, H, D]``, ``softmax_scale``, ``causal`` (bottom-right aligned), ``window_size=(left, right)``,
``alibi_slopes``, ``deterministic``, ``return_attn_probs`` (returns the log-sum-exp).  The ``*_xla`` names are
aliases.  Variants: fixed length, padded batch + ``attention_mask`` (varlen), packed sequences delimited by
``position_ids == 0``, and QKV-packed.

Backends (``set_attention_backend``):
  * ``"native"``  -- sm_90a kernels: S=QK^T and O+=PV on wgmma with register accumulators, TMA-fed K/V ring,
                     online softmax in registers; backward with five wgmma GEMMs per tile.
  * ``"sdpa"``    -- ``torch.nn.functional.scaled_dot_product_attention`` (library; bring-up / unsupported shapes)
  * ``"reference"`` -- explicit fp32 math (test oracle; the only backend on CPU).
Deterministic mode (``deterministic=True``, ``set_deterministic(True)`` -- what ``Config.compute.deterministic`` does --
or ``torch.use_deterministic_algorithms(True)``): the native backward computes dQ in a query-stationary kernel without
atomics, so repeated backward passes give bitwise-equal gradients (cost: DESIGN.md section 7).
Features the native kernels do not cover (dropout > 0, ALiBi, head_dim not in {64, 128}) route to ``sdpa`` /
``reference`` with a one-time warning rather than failing.
"""
from __future__ import annotations

import math
import os

import torch
import torch.nn.functional as F

from .. import _native as nat
from ..utils.logger import logger

_BACKEND = os.environ.get("TORCHACC_B200_ATTN", "auto")
_warned = set()
_DETERMINISTIC = False
# backward passes that ran the deterministic dQ kernel (tests check that the flag reached the kernels)
DETERMINISTIC_BWD_CALLS = 0


def set_attention_backend(name: str) -> None:
    global _BACKEND
    assert name in ("auto", "native", "sdpa", "reference")
    _BACKEND = name


def get_attention_backend() -> str:
    return _BACKEND


def set_deterministic(flag: bool) -> None:
    """Process-wide switch: every native attention backward takes the deterministic (atomic-free) dQ path."""
    global _DETERMINISTIC
    _DETERMINISTIC = bool(flag)


def deterministic_enabled(flag: bool = False) -> bool:
    """Effective flag: the per-call ``deterministic`` argument, the process switch or PyTorch's global switch."""
    return bool(flag) or _DETERMINISTIC or torch.are_deterministic_algorithms_enabled()


def _warn_once(key, msg):
    if key not in _warned:
        _warned.add(key)
        logger.warning(msg)


nat.register_signatures({
    "tb_flash_attn_fwd": ([nat.u64] * 7 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32] + [nat.i32] * 3 +
                          [nat.i64, nat.i64, nat.i32, nat.i32, nat.u64, nat.i32, nat.u64, nat.i32], nat.i32),
    "tb_flash_attn_bwd": ([nat.u64] * 13 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32] + [nat.i32] * 3 +
                          [nat.i64] * 5 + [nat.i32, nat.u64, nat.i32, nat.u64, nat.i32], nat.i32),
    "tb_flash_attn_fwd_dropout": ([nat.u64] * 7 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32] + [nat.i32] * 3 +
                                  [nat.i64, nat.i64, nat.i32, nat.u64, nat.i32, nat.u64, nat.i32, nat.f32, nat.u64],
                                  nat.i32),
    "tb_flash_attn_bwd_dropout": ([nat.u64] * 13 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32] + [nat.i32] * 3 +
                                  [nat.i64] * 5 + [nat.i32, nat.u64, nat.i32, nat.u64, nat.i32, nat.f32, nat.u64],
                                  nat.i32),
    "tb_flash_attn_bwd_deterministic": ([nat.u64] * 13 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32] + [nat.i32] * 3 +
                                        [nat.i64] * 5 + [nat.i32, nat.u64, nat.i32, nat.u64, nat.i32, nat.f32, nat.u64],
                                        nat.i32),
})


def native_supported(q, k, v, dropout_p, alibi_slopes, pad_ok: bool = False) -> bool:
    L = nat.lib()
    if L is None or not hasattr(L, "tb_flash_attn_fwd"):
        return False
    D = q.shape[-1]
    # head dims other than 64 / 128 are zero-padded up to the next supported size by the callers (_pad_head_dim);
    # ALiBi, fp16 and dropout (counter-based mask, csrc/attn/dropout.cuh) are native
    d_ok = D in (64, 128) or (pad_ok and D <= 128 and D % 8 == 0)
    drop_ok = dropout_p == 0.0 or (0.0 < dropout_p < 1.0 and hasattr(L, "tb_flash_attn_fwd_dropout"))
    return (q.is_cuda and q.dtype in (torch.bfloat16, torch.float16) and d_ok and drop_ok
            and q.stride(-1) == 1 and k.stride(-1) == 1 and v.stride(-1) == 1)


# ------------------------------------------------------------------------------------------------------
# Reference math (fp32).  Token-major [T, H, D] per sequence; used as test oracle and CPU path.
# ------------------------------------------------------------------------------------------------------
def _mask_for(sq, sk, causal, window, device):
    """True = masked out.  Bottom-right aligned causal / sliding window (FA2 semantics)."""
    if not causal and window[0] < 0 and window[1] < 0:
        return None
    qi = torch.arange(sq, device=device).unsqueeze(1) + (sk - sq)
    ki = torch.arange(sk, device=device).unsqueeze(0)
    left, right = window
    if causal:
        right = 0 if right < 0 else min(right, 0)
    m = torch.zeros(sq, sk, dtype=torch.bool, device=device)
    if right >= 0:
        m |= ki > qi + right
    if left >= 0:
        m |= ki < qi - left
    return m


def attention_reference(q, k, v, softmax_scale=None, causal=False, window_size=(-1, -1), alibi_slopes=None,
                        dropout_p=0.0, keep_mask=None):
    """q: [B, Sq, Hq, D], k/v: [B, Sk, Hk, D] -> (out [B,Sq,Hq,D] in q.dtype, lse [B,Hq,Sq] fp32)."""
    B, Sq, Hq, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    g = Hq // Hk
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().permute(0, 2, 1, 3).repeat_interleave(g, dim=1)
    vf = v.float().permute(0, 2, 1, 3).repeat_interleave(g, dim=1)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if alibi_slopes is not None:
        sl = alibi_slopes.float().view(-1, Hq, 1, 1) if alibi_slopes.dim() == 2 else alibi_slopes.float().view(1, Hq, 1, 1)
        qi = torch.arange(Sq, device=q.device).view(1, 1, Sq, 1) + (Sk - Sq)
        ki = torch.arange(Sk, device=q.device).view(1, 1, 1, Sk)
        s = s - sl * (qi - ki).abs()
    m = _mask_for(Sq, Sk, causal, window_size, q.device)
    if m is not None:
        s = s.masked_fill(m, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse.unsqueeze(-1))
    p = torch.nan_to_num(p, nan=0.0)  # fully-masked rows -> zeros (FA2 semantics)
    if keep_mask is not None:       # explicit mask [B, Hq, Sq, Sk] (the kernels' counter-based mask: dropout_keep_mask)
        p = p * keep_mask.to(p.dtype) / (1.0 - dropout_p)
    elif dropout_p > 0:
        p = F.dropout(p, dropout_p)
    o = torch.matmul(p, vf).permute(0, 2, 1, 3)
    return o.to(q.dtype), lse


# ------------------------------------------------------------------------------------------------------
# Native launcher (tokens flattened; see csrc/attn/attn.h)
# ------------------------------------------------------------------------------------------------------
def _alibi_args(alibi, Hq):
    """(pointer, batch stride) of fp32 ALiBi slopes given as [Hq] or [B, Hq] (reference flash_attn.py:313-601)."""
    if alibi is None:
        return 0, 0
    assert alibi.dtype == torch.float32 and alibi.is_contiguous() and alibi.shape[-1] == Hq
    return alibi.data_ptr(), (Hq if alibi.dim() == 2 else 0)


def new_dropout_seed() -> int:
    """64-bit seed for one attention call, drawn from torch's CPU generator (``torch.manual_seed`` makes it
    reproducible, activation checkpointing restores the generator state so the recomputed forward draws the same
    value) -- no device sync."""
    return int(torch.empty((), dtype=torch.int64).random_().item()) & 0x7FFFFFFFFFFFFFFF


def _mix32(x):
    x = x & 0xFFFFFFFF
    x = x ^ (x >> 16)
    x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x = x ^ (x >> 15)
    x = (x * 0x846CA68B) & 0xFFFFFFFF
    return x ^ (x >> 16)


def dropout_keep_mask(seed: int, p_drop: float, B: int, Hq: int, Sq: int, Sk: int, device="cpu") -> torch.Tensor:
    """Bit-exact PyTorch mirror of csrc/attn/dropout.cuh: bool [B, Hq, Sq, Sk], True = kept.  Test oracle (and the
    S_dmask a caller may ask for); the kernels never materialise it."""
    M = 0xFFFFFFFF
    lo, hi = seed & M, (seed >> 32) & M
    bh = torch.arange(B * Hq, dtype=torch.int64, device=device).view(B, Hq, 1, 1)
    qi = torch.arange(Sq, dtype=torch.int64, device=device).view(1, 1, Sq, 1)
    ki = torch.arange(Sk, dtype=torch.int64, device=device).view(1, 1, 1, Sk)
    head = lo ^ ((bh * 0x9E3779B1) & M)
    row = ((head ^ ((qi * 0x85EBCA77) & M)) * 0xC2B2AE3D) & M
    key = (hi + ki * 0x27D4EB2F) & M
    x = _mix32(row ^ key)
    p32 = torch.tensor(p_drop, dtype=torch.float32).item()          # the kernels receive p as a C float
    return (x >> 8) >= int(p32 * 16777216.0 + 0.5)


def _native_fwd(q3, k3, v3, cu_q, cu_k, B, Sq, Sk, scale, causal, window, alibi=None, dropout=None):
    """q3: [Tq, Hq, D] strided view (token stride arbitrary, head stride D); returns (o [Tq,Hq,D], lse [Hq,Tq]).
    ``dropout`` = (p, seed) or None."""
    Tq, Hq, D = q3.shape
    ap, abs_ = _alibi_args(alibi, Hq)
    Tk, Hk = k3.shape[0], k3.shape[1]
    o = torch.empty((Tq, Hq, D), dtype=q3.dtype, device=q3.device)
    lse = torch.empty((Hq, Tq), dtype=torch.float32, device=q3.device)
    L = nat.require()
    if dropout is not None:
        nat.check(
            L.tb_flash_attn_fwd_dropout(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o.data_ptr(), lse.data_ptr(),
                                        nat.ptr(cu_q), nat.ptr(cu_k), B, Sq, Sk, Hq, Hk, D, q3.stride(0), k3.stride(0),
                                        v3.stride(0), o.stride(0), scale, int(causal), window[0], window[1], Tq, Tk, 0,
                                        nat.stream(), int(q3.dtype == torch.bfloat16), ap, abs_, float(dropout[0]),
                                        int(dropout[1])), "tb_flash_attn_fwd_dropout")
        nat.count_launch()
        return o, lse
    nat.check(
        L.tb_flash_attn_fwd(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o.data_ptr(), lse.data_ptr(), nat.ptr(cu_q),
                            nat.ptr(cu_k), B, Sq, Sk, Hq, Hk, D, q3.stride(0), k3.stride(0), v3.stride(0), o.stride(0),
                            scale, int(causal), window[0], window[1], Tq, Tk, 0, nat.num_sms(), nat.stream(),
                            int(q3.dtype == torch.bfloat16), ap, abs_),
        "tb_flash_attn_fwd")
    nat.count_launch()
    return o, lse


def _native_bwd(do3, q3, k3, v3, o3, lse, cu_q, cu_k, B, Sq, Sk, scale, causal, window, dq3, dk3, dv3,
                deterministic=False, alibi=None, dropout=None):
    Tq, Hq, D = q3.shape
    ap, abs_ = _alibi_args(alibi, Hq)
    Tk, Hk = k3.shape[0], k3.shape[1]
    delta = torch.empty((Hq, Tq), dtype=torch.float32, device=q3.device)
    L = nat.require()
    if deterministic:
        # delta, dK/dV without the dQ step, then the query-stationary dQ kernel: no fp32 accumulator, no atomics
        global DETERMINISTIC_BWD_CALLS
        p, seed = dropout if dropout is not None else (0.0, 0)
        nat.check(
            L.tb_flash_attn_bwd_deterministic(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o3.data_ptr(),
                                              do3.data_ptr(), lse.data_ptr(), dq3.data_ptr(), dk3.data_ptr(),
                                              dv3.data_ptr(), 0, delta.data_ptr(), nat.ptr(cu_q), nat.ptr(cu_k), B,
                                              Sq, Sk, Hq, Hk, D, q3.stride(0), k3.stride(0), v3.stride(0),
                                              do3.stride(0), scale, int(causal), window[0], window[1], Tq, Tk,
                                              dq3.stride(0), dk3.stride(0), dv3.stride(0), nat.num_sms(), nat.stream(),
                                              int(q3.dtype == torch.bfloat16), ap, abs_, float(p), int(seed)),
            "tb_flash_attn_bwd_deterministic")
        nat.count_launch(3)
        DETERMINISTIC_BWD_CALLS += 1
        return
    dq_acc = torch.empty((Tq, Hq, D), dtype=torch.float32, device=q3.device)
    if dropout is not None:
        nat.check(
            L.tb_flash_attn_bwd_dropout(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o3.data_ptr(), do3.data_ptr(),
                                        lse.data_ptr(), dq3.data_ptr(), dk3.data_ptr(), dv3.data_ptr(),
                                        dq_acc.data_ptr(), delta.data_ptr(), nat.ptr(cu_q), nat.ptr(cu_k), B, Sq, Sk,
                                        Hq, Hk, D, q3.stride(0), k3.stride(0), v3.stride(0), do3.stride(0), scale,
                                        int(causal), window[0], window[1], Tq, Tk, dq3.stride(0), dk3.stride(0),
                                        dv3.stride(0), nat.num_sms(), nat.stream(), int(q3.dtype == torch.bfloat16),
                                        ap, abs_, float(dropout[0]), int(dropout[1])), "tb_flash_attn_bwd_dropout")
        nat.count_launch(3)
        return
    nat.check(
        L.tb_flash_attn_bwd(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o3.data_ptr(), do3.data_ptr(),
                            lse.data_ptr(), dq3.data_ptr(), dk3.data_ptr(), dv3.data_ptr(), dq_acc.data_ptr(),
                            delta.data_ptr(), nat.ptr(cu_q), nat.ptr(cu_k), B, Sq, Sk, Hq, Hk, D, q3.stride(0),
                            k3.stride(0), v3.stride(0), do3.stride(0), scale, int(causal), window[0], window[1], Tq,
                            Tk, dq3.stride(0), dk3.stride(0), dv3.stride(0), nat.num_sms(), nat.stream(),
                            int(q3.dtype == torch.bfloat16), ap, abs_),
        "tb_flash_attn_bwd")
    nat.count_launch(3)


class _FlashAttnFn(torch.autograd.Function):
    """Token-flattened attention.  q: [Tq,Hq,D], k/v: [Tk,Hk,D] (strided views allowed)."""

    @staticmethod
    def forward(ctx, q3, k3, v3, cu_q, cu_k, B, Sq, Sk, scale, causal, window, deterministic, alibi=None,
                dropout=None):
        o, lse = _native_fwd(q3, k3, v3, cu_q, cu_k, B, Sq, Sk, scale, causal, window, alibi, dropout)
        ctx.save_for_backward(q3, k3, v3, o, lse, cu_q, cu_k)
        ctx.alibi = alibi
        ctx.dropout = dropout                     # (p, seed): the backward regenerates the mask from it
        ctx.cfg = (B, Sq, Sk, scale, causal, window, deterministic)
        ctx.mark_non_differentiable(lse)
        return o, lse

    @staticmethod
    def backward(ctx, do, _dlse):
        q3, k3, v3, o, lse, cu_q, cu_k = ctx.saved_tensors
        B, Sq, Sk, scale, causal, window, det = ctx.cfg
        do = do if (do.stride(-1) == 1 and do.stride(1) == do.shape[2]) else do.contiguous()
        dq = torch.empty(q3.shape, dtype=q3.dtype, device=q3.device)
        dk = torch.empty(k3.shape, dtype=k3.dtype, device=k3.device)
        dv = torch.empty(v3.shape, dtype=v3.dtype, device=v3.device)
        _native_bwd(do, q3, k3, v3, o, lse, cu_q, cu_k, B, Sq, Sk, scale, causal, window, dq, dk, dv,
                    deterministic_enabled(det), ctx.alibi, ctx.dropout)
        return dq, dk, dv, None, None, None, None, None, None, None, None, None, None, None


class _FlashAttnQKVPackedFn(torch.autograd.Function):
    """Packed variant: qkv [T, (Hq + 2 Hk) * D] -> out [T, Hq*D]; the gradient is written straight into one
    dqkv buffer (no per-view gradient scatter)."""

    @staticmethod
    def forward(ctx, qkv, hq, hk, d, cu, B, S, scale, causal, window):
        T = qkv.shape[0]
        ts, off = qkv.stride(0), qkv.storage_offset()
        q3 = qkv.as_strided((T, hq, d), (ts, d, 1), off)
        k3 = qkv.as_strided((T, hk, d), (ts, d, 1), off + hq * d)
        v3 = qkv.as_strided((T, hk, d), (ts, d, 1), off + (hq + hk) * d)
        o, lse = _native_fwd(q3, k3, v3, cu, cu, B, S, S, scale, causal, window)
        ctx.save_for_backward(qkv, o, lse, cu)
        ctx.cfg = (hq, hk, d, B, S, scale, causal, window)
        return o.view(T, hq * d)

    @staticmethod
    def backward(ctx, do):
        qkv, o, lse, cu = ctx.saved_tensors
        hq, hk, d, B, S, scale, causal, window = ctx.cfg
        T = qkv.shape[0]
        ts, off = qkv.stride(0), qkv.storage_offset()
        q3 = qkv.as_strided((T, hq, d), (ts, d, 1), off)
        k3 = qkv.as_strided((T, hk, d), (ts, d, 1), off + hq * d)
        v3 = qkv.as_strided((T, hk, d), (ts, d, 1), off + (hq + hk) * d)
        dqkv = torch.empty((T, (hq + 2 * hk) * d), dtype=qkv.dtype, device=qkv.device)
        W = dqkv.stride(0)
        dq3 = dqkv.as_strided((T, hq, d), (W, d, 1), 0)
        dk3 = dqkv.as_strided((T, hk, d), (W, d, 1), hq * d)
        dv3 = dqkv.as_strided((T, hk, d), (W, d, 1), (hq + hk) * d)
        do3 = do.contiguous().view(T, hq, d)
        _native_bwd(do3, q3, k3, v3, o, lse, cu, cu, B, S, S, scale, causal, window, dq3, dk3, dv3,
                    deterministic_enabled())
        return dqkv, None, None, None, None, None, None, None, None, None


# ------------------------------------------------------------------------------------------------------
# Dispatch helpers
# ------------------------------------------------------------------------------------------------------
def _pad_head_dim(*ts):
    """Zero-pad the head dim to the next native size (64 / 128): zero columns change neither q k^T nor the first D
    columns of P v, so the caller slices the output back (softmax scale stays 1/sqrt(original D))."""
    D = ts[0].shape[-1]
    Dp = 64 if D <= 64 else 128
    if D == Dp:
        return ts, D
    return tuple(F.pad(t, (0, Dp - D)) for t in ts), D


def _pick_backend(q, k, v, dropout_p, alibi_slopes, pad_ok: bool = False):
    b = _BACKEND
    if b == "reference" or not q.is_cuda:
        return "reference"
    if b in ("auto", "native"):
        if native_supported(q, k, v, dropout_p, alibi_slopes, pad_ok):
            return "native"
        if b == "native":
            _warn_once(("native-unsupported", q.shape[-1], dropout_p, alibi_slopes is None),
                       "native attention does not cover this configuration (head_dim/dropout/alibi); using SDPA")
        if nat.lib() is None and not nat.allow_fallback():
            nat.require()
    return "sdpa"


def _sdpa(q, k, v, scale, causal, window, alibi_slopes, dropout_p):
    """Library fallback on [B,S,H,D] tensors.  Returns (out, lse or None)."""
    B, Sq, Hq, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    simple = window == (-1, -1) and alibi_slopes is None and (not causal or Sq == Sk)
    if not simple:
        return attention_reference(q, k, v, scale, causal, window, alibi_slopes, dropout_p)
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    o = F.scaled_dot_product_attention(qt, kt, vt, dropout_p=dropout_p, is_causal=causal, scale=scale,
                                       enable_gqa=(Hq != Hk))
    return o.transpose(1, 2), None


def _lse_or_compute(q, k, scale, causal, window, lse):
    if lse is not None:
        return lse
    with torch.no_grad():
        _, lse = attention_reference(q, k, torch.zeros_like(k), scale, causal, window)
    return lse


# ------------------------------------------------------------------------------------------------------
# Public API
# ------------------------------------------------------------------------------------------------------
def flash_attn_func(q, k, v, dropout_p=0.0, softmax_scale=None, causal=False, window_size=(-1, -1),
                    alibi_slopes=None, deterministic=False, return_attn_probs=False):
    """Fixed-length attention.  q: [B,Sq,Hq,D]; k,v: [B,Sk,Hk,D] (reference flash_attn.py:531-601)."""
    assert q.dtype in (torch.bfloat16, torch.float16, torch.float32)
    B, Sq, Hq, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    window = tuple(window_size)
    backend = _pick_backend(q, k, v, dropout_p, alibi_slopes, pad_ok=True)
    if backend == "native":
        (qp, kp, vp), D0 = _pad_head_dim(q, k, v)
        Dp = qp.shape[-1]
        q3 = qp.reshape(B * Sq, Hq, Dp) if qp.is_contiguous() else qp.contiguous().view(B * Sq, Hq, Dp)
        k3 = kp.reshape(B * Sk, Hk, Dp) if kp.is_contiguous() else kp.contiguous().view(B * Sk, Hk, Dp)
        v3 = vp.reshape(B * Sk, Hk, Dp) if vp.is_contiguous() else vp.contiguous().view(B * Sk, Hk, Dp)
        alibi = alibi_slopes.float().contiguous() if alibi_slopes is not None else None
        dropout = (float(dropout_p), new_dropout_seed()) if dropout_p > 0.0 else None
        o, lse = _FlashAttnFn.apply(q3, k3, v3, None, None, B, Sq, Sk, scale, causal, window, deterministic, alibi,
                                    dropout)
        out = o.view(B, Sq, Hq, Dp)[..., :D0]
        if return_attn_probs:
            # like flash-attn, the third value is only meaningful for testing: the keep mask [B, Hq, Sq, Sk]
            dmask = dropout_keep_mask(dropout[1], dropout[0], B, Hq, Sq, Sk, q.device) if dropout else None
            return out, lse.view(Hq, B, Sq).transpose(0, 1).contiguous(), dmask
        return out
    if backend == "sdpa":
        out, lse = _sdpa(q, k, v, scale, causal, window, alibi_slopes, dropout_p)
    else:
        out, lse = attention_reference(q, k, v, scale, causal, window, alibi_slopes, dropout_p)
    if return_attn_probs:
        return out, _lse_or_compute(q, k, scale, causal, window, lse), None
    return out


def flash_attn_qkvpacked_tokens(qkv, num_q_heads, num_kv_heads, head_dim, batch, seq_len, softmax_scale=None,
                                causal=True, window_size=(-1, -1), cu_seqlens=None):
    """Native-model fast path.  qkv: [T, (Hq+2Hk)*D] (q|k|v along the last dim, T = batch*seq_len or packed with
    ``cu_seqlens``).  Returns [T, Hq*D].  The backward is deterministic when ``set_deterministic(True)`` or
    ``torch.use_deterministic_algorithms(True)`` is in effect."""
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(head_dim)
    T = qkv.shape[0]
    hq, hk, d = num_q_heads, num_kv_heads, head_dim
    ts, off = qkv.stride(0), qkv.storage_offset()
    q3 = qkv.as_strided((T, hq, d), (ts, d, 1), off)
    k3 = qkv.as_strided((T, hk, d), (ts, d, 1), off + hq * d)
    v3 = qkv.as_strided((T, hk, d), (ts, d, 1), off + (hq + hk) * d)
    backend = _pick_backend(q3, k3, v3, 0.0, None)
    if backend == "native":
        return _FlashAttnQKVPackedFn.apply(qkv, hq, hk, d, cu_seqlens, batch, seq_len, scale, causal,
                                           tuple(window_size))
    if cu_seqlens is not None:
        out = flash_attn_varlen_cu(q3, k3, v3, cu_seqlens, cu_seqlens, scale, causal, tuple(window_size))
        return out.reshape(T, hq * d)
    q4 = q3.reshape(batch, seq_len, hq, d)
    k4 = k3.reshape(batch, seq_len, hk, d)
    v4 = v3.reshape(batch, seq_len, hk, d)
    out = flash_attn_func(q4, k4, v4, softmax_scale=scale, causal=causal, window_size=window_size)
    return out.reshape(T, hq * d)


def flash_attn_varlen_cu(q3, k3, v3, cu_q, cu_k, scale, causal, window, return_lse=False, dropout_p=0.0,
                         alibi_slopes=None, deterministic=False):
    """Packed sequences: q3 [Tq,Hq,D], k3/v3 [Tk,Hk,D], cu_* int32 [B+1]."""
    backend = _pick_backend(q3, k3, v3, dropout_p, alibi_slopes, pad_ok=True)
    Bn = cu_q.numel() - 1
    if backend == "native":
        (qp, kp, vp), D0 = _pad_head_dim(q3, k3, v3)
        alibi = alibi_slopes.float().contiguous() if alibi_slopes is not None else None
        dropout = (float(dropout_p), new_dropout_seed()) if dropout_p > 0.0 else None
        o, lse = _FlashAttnFn.apply(qp, kp, vp, cu_q.int(), cu_k.int(), Bn, 0, 0, scale, causal, window, deterministic,
                                    alibi, dropout)
        o = o[..., :D0]
        return (o, lse) if return_lse else o
    assert dropout_p == 0.0 and alibi_slopes is None, "the per-sequence fallback handles plain attention only"
    outs, lses = [], []
    cq, ck = cu_q.tolist(), cu_k.tolist()
    for b in range(Bn):
        qs, ks, vs = q3[cq[b]:cq[b + 1]], k3[ck[b]:ck[b + 1]], v3[ck[b]:ck[b + 1]]
        if qs.shape[0] == 0:
            continue
        o, l = attention_reference(qs.unsqueeze(0), ks.unsqueeze(0), vs.unsqueeze(0), scale, causal, window)
        outs.append(o[0])
        lses.append(l[0])
    o = torch.cat(outs, 0)
    if return_lse:
        return o, torch.cat(lses, 1)
    return o


def _lens_to_cu(lens: torch.Tensor) -> torch.Tensor:
    return F.pad(lens.cumsum(0, dtype=torch.int32), (1, 0))


def flash_attn_varlen_func(q, k, v, attention_mask, dropout_p=0.0, softmax_scale=None, causal=False,
                           window_size=(-1, -1), alibi_slopes=None, deterministic=False, return_attn_probs=False):
    """Padded batch + ``attention_mask`` [B, S] (1 = token).  Padding is assumed right-aligned, as in HF batches
    (reference flash_attn.py:373-449).  Output rows of padded positions are zero."""
    B, Sq, Hq, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    mask = attention_mask.to(torch.bool)
    assert Sq == Sk, "flash_attn_varlen_func expects self-attention shaped inputs (Sq == Sk)"
    idx = mask.reshape(-1).nonzero(as_tuple=False).squeeze(1)
    lens = mask.sum(1).to(torch.int32)
    cu = _lens_to_cu(lens)
    q3 = q.reshape(B * Sq, Hq, D).index_select(0, idx)
    k3 = k.reshape(B * Sk, Hk, D).index_select(0, idx)
    v3 = v.reshape(B * Sk, Hk, D).index_select(0, idx)
    if (dropout_p > 0 or alibi_slopes is not None) and _pick_backend(q3, k3, v3, dropout_p, alibi_slopes,
                                                                      pad_ok=True) != "native":
        _warn_once("varlen-extra", "varlen attention with dropout/ALiBi runs on the reference path")
        o4, lse4 = attention_reference_masked(q, k, v, mask, scale, causal, window_size, alibi_slopes, dropout_p)
        return (o4, lse4, None) if return_attn_probs else o4
    res = flash_attn_varlen_cu(q3, k3, v3, cu, cu, scale, causal, tuple(window_size), return_lse=return_attn_probs,
                               dropout_p=dropout_p, alibi_slopes=alibi_slopes, deterministic=deterministic)
    o3 = res[0] if return_attn_probs else res
    out = torch.zeros((B * Sq, Hq, D), dtype=q.dtype, device=q.device).index_copy(0, idx, o3).view(B, Sq, Hq, D)
    if return_attn_probs:
        lse = torch.full((Hq, B * Sq), float("inf"), dtype=torch.float32, device=q.device)
        lse = lse.index_copy(1, idx, res[1]).view(Hq, B, Sq).transpose(0, 1).contiguous()
        return out, lse, None
    return out


def attention_reference_masked(q, k, v, mask, scale, causal, window, alibi_slopes=None, dropout_p=0.0):
    """Oracle for padded batches: per-sample slicing."""
    B = q.shape[0]
    out = torch.zeros_like(q)
    lse = torch.full((B, q.shape[2], q.shape[1]), float("inf"), dtype=torch.float32, device=q.device)
    for b in range(B):
        n = int(mask[b].sum())
        if n == 0:
            continue
        o, l = attention_reference(q[b:b + 1, :n], k[b:b + 1, :n], v[b:b + 1, :n], scale, causal, tuple(window),
                                   alibi_slopes[b:b + 1] if (alibi_slopes is not None and alibi_slopes.dim() == 2)
                                   else alibi_slopes, dropout_p)
        out[b, :n] = o[0]
        lse[b, :, :n] = l[0]
    return out, lse


def flash_attn_varlen_qkvpacked_func(qkv, attention_mask, dropout_p=0.0, softmax_scale=None, causal=False,
                                     window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                                     return_attn_probs=False):
    """qkv: [B, S, 3, H, D] (reference flash_attn.py:313-336)."""
    q, k, v = qkv.unbind(2)
    return flash_attn_varlen_func(q, k, v, attention_mask, dropout_p, softmax_scale, causal, window_size,
                                  alibi_slopes, deterministic, return_attn_probs)


def position_ids_to_cu_seqlens(position_ids: torch.Tensor) -> torch.Tensor:
    """Sequence starts are where ``position_ids == 0`` (packed batch of size 1; reference flash_attn.py:173-216)."""
    pid = position_ids.reshape(-1)
    starts = (pid == 0).nonzero(as_tuple=False).squeeze(1).to(torch.int32)
    total = torch.tensor([pid.numel()], dtype=torch.int32, device=pid.device)
    if starts.numel() == 0 or int(starts[0]) != 0:
        starts = torch.cat([torch.zeros(1, dtype=torch.int32, device=pid.device), starts])
    return torch.cat([starts, total])


def flash_attn_varlen_position_ids_func(q, k, v, position_ids, dropout_p=0.0, softmax_scale=None, causal=False,
                                        window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                                        return_attn_probs=False):
    """Packed sequences in a batch of 1, boundaries from ``position_ids`` (reference flash_attn.py:452-528)."""
    B, S, Hq, D = q.shape
    assert B == 1, "position_ids packing expects batch size 1"
    Hk = k.shape[2]
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    cu = position_ids_to_cu_seqlens(position_ids)
    res = flash_attn_varlen_cu(q.reshape(S, Hq, D), k.reshape(S, Hk, D), v.reshape(S, Hk, D), cu, cu, scale, causal,
                               tuple(window_size), return_lse=return_attn_probs, deterministic=deterministic)
    if return_attn_probs:
        return res[0].view(1, S, Hq, D), res[1].view(Hq, 1, S).transpose(0, 1).contiguous(), None
    return res.view(1, S, Hq, D)


def spmd_flash_attn_varlen_func(q, k, v, attention_mask, dropout_p=0.0, softmax_scale=None, causal=False,
                                window_size=(-1, -1), alibi_slopes=None, deterministic=False,
                                return_attn_probs=False, mesh=None, partition_spec=None):
    """Kept for API compatibility (reference flash_attn.py:339-370): there is no SPMD partitioner here; each rank
    already holds its shard of batch/heads, so this is the plain varlen call."""
    return flash_attn_varlen_func(q, k, v, attention_mask, dropout_p, softmax_scale, causal, window_size,
                                  alibi_slopes, deterministic, return_attn_probs)


# reference-compatible aliases
flash_attn_xla = flash_attn_func
flash_attn_varlen_xla = flash_attn_varlen_func
flash_attn_varlen_qkvpacked_xla = flash_attn_varlen_qkvpacked_func
flash_attn_varlen_position_ids_xla = flash_attn_varlen_position_ids_func
spmd_flash_attn_varlen_xla = spmd_flash_attn_varlen_func
