"""RMSNorm (+ fused residual add) on the sm_90a kernels in csrc/ops/norm_rope_act.cu.

Replaces liger's Triton RMSNorm that the reference patches into HF Llama/Qwen2
(reference torchacc/ops/liger.py:10-18).  Semantics follow HF ``LlamaRMSNorm``: statistics in fp32,
output cast to the input dtype after multiplying by the weight.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import _native as nat


def rmsnorm_ref(x, w, eps, residual=None):
    h = x if residual is None else x + residual
    hf = h.float()
    y = hf * torch.rsqrt(hf.pow(2).mean(-1, keepdim=True) + eps)
    return (y * w.float()).to(x.dtype), h


class _RMSNormFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, w, residual, eps, passthrough=False):
        H = x.shape[-1]
        x2 = x.contiguous().view(-1, H)
        r2 = residual.contiguous().view(-1, H) if residual is not None else None
        rows = x2.shape[0]
        y = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        h = torch.empty(x.shape, dtype=x.dtype, device=x.device) if r2 is not None else x2
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        L = nat.require()
        nat.check(
            L.tb_rmsnorm_fwd(x2.data_ptr(), nat.ptr(r2), w.data_ptr(), y.data_ptr(),
                             h.data_ptr() if r2 is not None else 0, rstd.data_ptr(), rows, H, eps, nat.num_sms(),
                             nat.stream(), nat.bf16_flag(x)), "tb_rmsnorm_fwd")
        nat.count_launch()
        ctx.save_for_backward(h.view(-1, H) if r2 is not None else h, w, rstd)
        ctx.has_res = r2 is not None
        ctx.passthrough = bool(passthrough) and r2 is None
        ctx.shape = x.shape
        if r2 is not None:
            return y, h
        if ctx.passthrough:
            return y, x.view_as(x)      # identity branch: its gradient is added inside the backward kernel
        return y, None

    @staticmethod
    def backward(ctx, dy, dh):
        h, w, rstd = ctx.saved_tensors
        H = h.shape[-1]
        rows = h.shape[0]
        dy2 = dy.contiguous().view(-1, H)
        dres = dh.contiguous().view(-1, H) if (dh is not None and (ctx.has_res or ctx.passthrough)) else None
        dx = torch.empty(ctx.shape, dtype=h.dtype, device=h.device)
        # one CTA per partial row: each writes its fp32 column sums (no atomics), summed below
        parts = max(1, min(rows, nat.num_sms() * 2))   # = resident CTAs (2 x 512 threads per SM): persistent rows loop
        dw_part = torch.empty((parts, H), dtype=torch.float32, device=h.device)
        L = nat.require()
        nat.check(
            L.tb_rmsnorm_bwd(dy2.data_ptr(), h.data_ptr(), w.data_ptr(), rstd.data_ptr(), nat.ptr(dres),
                             dx.data_ptr(), dw_part.data_ptr(), parts, rows, H, nat.num_sms(), nat.stream(),
                             nat.bf16_flag(h)),
            "tb_rmsnorm_bwd")
        nat.count_launch()
        return dx, dw_part.sum(0).to(w.dtype), (dx if ctx.has_res else None), None, None


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6, residual: Optional[torch.Tensor] = None,
            passthrough: bool = False) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Returns ``(y, h)``: ``h = x + residual`` (the updated residual stream, ``None`` without residual) and
    ``y = rmsnorm(h) * weight``.  With ``passthrough`` (and no residual) ``h`` is ``x`` itself routed through the
    op, so a consumer of the skip branch sends its gradient into the fused backward kernel instead of a separate
    autograd accumulation pass."""
    if nat.is_half(x, weight) and (residual is None or residual.dtype == x.dtype) and nat.use_native(x, weight) \
            and x.shape[-1] % 8 == 0 and x.shape[-1] <= 16384:
        return _RMSNormFn.apply(x, weight, residual, eps, passthrough)
    y, h = rmsnorm_ref(x, weight, eps, residual)
    return y, (h if residual is not None else (x if passthrough else None))


class RMSNorm(torch.nn.Module):

    def __init__(self, hidden_size: int, eps: float = 1e-6, device=None, dtype=None):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.ones(hidden_size, device=device, dtype=dtype))
        self.eps = eps

    def forward(self, x, residual=None):
        y, h = rmsnorm(x, self.weight, self.eps, residual)
        return y if residual is None else (y, h)
