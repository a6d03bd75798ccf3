"""Linear layers on the hand-written wgmma GEMM (csrc/gemm/gemm_bf16.cu).

``linear(x, w, bias)`` computes ``x @ w.T + bias`` with three launches of the same kernel:
forward (K-major/K-major), dgrad (K-major/MN-major) and wgrad (MN-major/MN-major) -- no transposed copies.
When the weight carries a ``_tb_grad_view`` (installed by the FSDP/DP engines) the weight gradient is written
or accumulated directly into that flat-buffer slice by the GEMM epilogue and autograd sees ``None``
(gradient-accumulation fusion), so no extra ``grad += `` pass over the weights happens.

The reference reaches cuBLAS through ``nn.Linear`` here (SURVEY 2.4a "Dense GEMMs").
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .. import _native as nat

_CLUSTER = 1   # CTA-pair tiles do not exist on sm_90a; the C ABI keeps the argument


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_mn_major: bool = False, b_mn_major: bool = False,
         out: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None, accumulate: bool = False,
         out_dtype: Optional[torch.dtype] = None, addend: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``D[M,N] (+)= A_op[M,K] @ B_op[N,K]^T (+ bias) (+ addend)`` on 2-D bf16 tensors (last dim contiguous).

    ``a`` is ``[M,K]`` (or ``[K,M]`` when ``a_mn_major``); ``b`` is ``[N,K]`` (or ``[K,N]`` when ``b_mn_major``).
    ``addend`` ([M,N], D's dtype) is added in the GEMM epilogue (fused residual add); ``accumulate`` is the special
    case addend == out.
    """
    assert a.dim() == 2 and b.dim() == 2
    if a_mn_major:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn_major:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert K == Kb, f"reduction dims differ: {K} vs {Kb}"
    if out is None:
        assert not accumulate
        out = torch.empty((M, N), dtype=out_dtype or (a.dtype if a.dtype != torch.float32 else torch.bfloat16),
                          device=a.device)
    assert not (accumulate and addend is not None)
    if not nat.use_native(a, b):
        A = a.t() if a_mn_major else a
        B = b if b_mn_major else b.t()
        r = A.float() @ B.float()
        if bias is not None:
            r = r + bias.float()
        if addend is not None:
            r = r + addend.float()
        if accumulate:
            out.add_(r.to(out.dtype))
        else:
            out.copy_(r.to(out.dtype))
        return out
    assert a.dtype == b.dtype and a.dtype in (torch.bfloat16, torch.float16), "native GEMM: bf16 x bf16 or fp16 x fp16"
    f16 = int(a.dtype == torch.float16)
    assert out.dtype in (a.dtype, torch.float32)
    assert a.stride(1) == 1 and b.stride(1) == 1 and out.stride(1) == 1
    assert a.stride(0) % 8 == 0 and b.stride(0) % 8 == 0, "row pitch must be a multiple of 16 bytes (TMA)"
    if bias is not None:
        assert bias.dtype == a.dtype and bias.is_contiguous()
    L = nat.require()
    if addend is not None:
        assert addend.dtype == out.dtype and addend.shape == out.shape and addend.stride(1) == 1 \
            and addend.stride(0) % 8 == 0
        nat.check(
            L.tb_gemm_bf16_ex(a.data_ptr(), b.data_ptr(), out.data_ptr(), nat.ptr(bias), addend.data_ptr(), M, N, K,
                              a.stride(0), b.stride(0), out.stride(0), addend.stride(0), int(a_mn_major),
                              int(b_mn_major), int(out.dtype == torch.float32), _CLUSTER, nat.num_sms(), nat.stream(),
                              f16),
            "tb_gemm_bf16_ex")
    else:
        nat.check(
            L.tb_gemm_bf16(a.data_ptr(), b.data_ptr(), out.data_ptr(), nat.ptr(bias), M, N, K, a.stride(0), b.stride(0),
                           out.stride(0), int(a_mn_major), int(b_mn_major), int(out.dtype == torch.float32),
                           int(accumulate), _CLUSTER, nat.num_sms(), nat.stream(), f16), "tb_gemm_bf16")
    nat.count_launch()
    return out


class _LinearFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, w, bias, residual=None):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if x2.stride(-1) != 1 or x2.stride(0) % 8 != 0:
            x2 = x2.contiguous()
        # allocate with the final shape: returning a view made inside a custom Function would forbid later
        # in-place ops on the result (RoPE rotates the QKV activation in place)
        y = torch.empty((*shp[:-1], w.shape[0]), dtype=x.dtype, device=x.device)
        r2 = None
        if residual is not None:
            r2 = residual.reshape(-1, w.shape[0])
            if r2.stride(-1) != 1 or r2.stride(0) % 8 != 0:
                r2 = r2.contiguous()
        gemm(x2, w, bias=bias, out=y.view(-1, w.shape[0]), addend=r2)   # y = x W^T (+ b) (+ residual), one kernel
        ctx.has_res = residual is not None
        ctx.save_for_backward(x2, w)
        # the engine's hand-off attributes (_tb_grad_view / _tb_grad_ready) live on the parameter OBJECT; under
        # non-reentrant activation checkpointing ctx.saved_tensors returns detached aliases without them
        ctx.w_obj = w
        ctx.has_bias = bias is not None
        ctx.x_shape = shp
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.stride(-1) != 1 or dy2.stride(0) % 8 != 0:
            dy2 = dy2.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(ctx.x_shape, dtype=dy2.dtype, device=dy2.device)
            gemm(dy2, w, b_mn_major=True, out=dx.view(-1, ctx.x_shape[-1]))
        if ctx.needs_input_grad[1]:
            wo = ctx.w_obj
            view = getattr(wo, "_tb_grad_view", None)
            if view is not None:
                acc = bool(getattr(wo, "_tb_grad_ready", False))
                gemm(dy2, x2, a_mn_major=True, b_mn_major=True, out=view, accumulate=acc)
                wo._tb_grad_ready = True
            else:
                dw = gemm(dy2, x2, a_mn_major=True, b_mn_major=True)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(0).to(dy2.dtype)
        return dx, dw, db, (dy if ctx.has_res else None)


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
           residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Drop-in for ``F.linear`` (bf16 CUDA tensors go through the wgmma GEMM).  ``residual`` (same shape as the
    result) is added inside the GEMM epilogue: ``x @ w.T + bias + residual`` without a separate elementwise pass."""
    if x.is_cuda and nat.is_half(x, w) and nat.use_native(x, w):
        from . import fp8
        if fp8.enabled() and fp8.eligible(x.reshape(-1, x.shape[-1]), w):
            return fp8.fp8_linear(x, w, bias, residual)          # compute.fp8: block-scaled e4m3 GEMMs (ops/fp8.py)
        return _LinearFn.apply(x, w, bias, residual)
    y = F.linear(x, w, bias)
    return y if residual is None else y + residual


class Linear(torch.nn.Linear):
    """``nn.Linear`` whose forward/backward run on the wgmma GEMM."""

    def forward(self, x):
        return linear(x, self.weight, self.bias)
