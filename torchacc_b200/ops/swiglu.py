"""SwiGLU: ``h = silu(g) * u`` on the kernels in csrc/ops/norm_rope_act.cu.

``swiglu(gu)`` takes the fused gate|up projection output ``[..., 2F]``; ``swiglu_separate(g, u)`` takes the two
halves as separate (row-strided) tensors, which is what the HF module patches use.
Replaces liger's Triton SiLU-mul (reference torchacc/ops/liger.py:21-28)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .. import _native as nat


def _rows(t):
    t2 = t.reshape(-1, t.shape[-1])
    if t2.stride(-1) != 1 or t2.stride(0) % 8 != 0:
        t2 = t2.contiguous()
    return t2


class _SwiGLUFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, g, u):
        Fdim = g.shape[-1]
        g2, u2 = _rows(g), _rows(u)
        T = g2.shape[0]
        h = torch.empty((*g.shape[:-1], Fdim), dtype=g.dtype, device=g.device)
        L = nat.require()
        nat.check(L.tb_swiglu_fwd(g2.data_ptr(), u2.data_ptr(), h.data_ptr(), T, Fdim, g2.stride(0), u2.stride(0),
                                  nat.num_sms(), nat.stream(), nat.bf16_flag(g2)), "tb_swiglu_fwd")
        nat.count_launch()
        ctx.save_for_backward(g2, u2)
        ctx.shape = g.shape
        return h

    @staticmethod
    def backward(ctx, dh):
        g2, u2 = ctx.saved_tensors
        T, Fdim = g2.shape
        dh2 = dh.contiguous().view(T, Fdim)
        dgu = torch.empty((T, 2 * Fdim), dtype=g2.dtype, device=g2.device)
        dg, du = dgu[:, :Fdim], dgu[:, Fdim:]
        L = nat.require()
        nat.check(
            L.tb_swiglu_bwd(dh2.data_ptr(), g2.data_ptr(), u2.data_ptr(), dg.data_ptr(), du.data_ptr(), T, Fdim,
                            g2.stride(0), u2.stride(0), dgu.stride(0), dgu.stride(0), nat.num_sms(), nat.stream(),
                            nat.bf16_flag(g2)),
            "tb_swiglu_bwd")
        nat.count_launch()
        return dg.view(ctx.shape), du.view(ctx.shape)


def swiglu_separate(g: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    if nat.is_half(g, u) and nat.use_native(g, u) and g.shape[-1] % 8 == 0:
        return _SwiGLUFn.apply(g, u)
    return (F.silu(g.float()) * u.float()).to(g.dtype)


class _SwiGLUFusedFn(torch.autograd.Function):
    """Fused gate|up input: the gradient is produced as ONE [T, 2F] tensor (no slice-gradient scatter)."""

    @staticmethod
    def forward(ctx, gu):
        Fdim = gu.shape[-1] // 2
        gu2 = _rows(gu)
        T = gu2.shape[0]
        h = torch.empty((*gu.shape[:-1], Fdim), dtype=gu.dtype, device=gu.device)
        L = nat.require()
        nat.check(L.tb_swiglu_fwd(gu2.data_ptr(), gu2.data_ptr() + 2 * Fdim, h.data_ptr(), T, Fdim, gu2.stride(0),
                                  gu2.stride(0), nat.num_sms(), nat.stream(), nat.bf16_flag(gu2)), "tb_swiglu_fwd")
        nat.count_launch()
        ctx.save_for_backward(gu2)
        ctx.shape = gu.shape
        return h

    @staticmethod
    def backward(ctx, dh):
        (gu2,) = ctx.saved_tensors
        T, Fdim = gu2.shape[0], gu2.shape[1] // 2
        dh2 = dh.contiguous().view(T, Fdim)
        dgu = torch.empty(ctx.shape, dtype=gu2.dtype, device=gu2.device)
        ld = 2 * Fdim
        L = nat.require()
        nat.check(
            L.tb_swiglu_bwd(dh2.data_ptr(), gu2.data_ptr(), gu2.data_ptr() + 2 * Fdim, dgu.data_ptr(),
                            dgu.data_ptr() + 2 * Fdim, T, Fdim, gu2.stride(0), gu2.stride(0), ld, ld, nat.num_sms(),
                            nat.stream(), nat.bf16_flag(gu2)), "tb_swiglu_bwd")
        nat.count_launch()
        return dgu


# ---- gate|up projection with the activation in the GEMM epilogue -----------------------------------------------------
# While a module runs its FIRST forward under activation checkpointing nothing it saves survives (the backward
# recomputes the module), so the fused op writes only h = silu(g) * u and never materialises the [T, 2F] pre-activation.
# The sharding engine / gradient_checkpoint wrappers flip this flag around their checkpointed call.
_RECOMPUTED_LATER = [False]


class activations_recomputed_later:
    def __enter__(self):
        self.prev = _RECOMPUTED_LATER[0]
        _RECOMPUTED_LATER[0] = True

    def __exit__(self, *exc):
        _RECOMPUTED_LATER[0] = self.prev
        return False


nat.register_signatures({
    "tb_gemm_swiglu": ([nat.u64, nat.u64, nat.u64, nat.u64, nat.i32, nat.i32, nat.i32, nat.i64, nat.i64, nat.i64, nat.i64,
                        nat.i32, nat.u64, nat.i32], nat.i32),
})


class _GateUpSwiGLUFn(torch.autograd.Function):
    """h = silu(x Wg^T) * (x Wu^T) in ONE wgmma GEMM (csrc/gemm/gemm_bf16.cu, SwiGLU epilogue: every stage holds the
    matching gate / up weight rows, so both halves of an output column sit in the same accumulator tile)."""

    @staticmethod
    def forward(ctx, x, w_gu):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if x2.stride(-1) != 1 or x2.stride(0) % 8 != 0:
            x2 = x2.contiguous()
        T, K = x2.shape
        Fdim = w_gu.shape[0] // 2
        need = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        h = torch.empty((*shp[:-1], Fdim), dtype=x.dtype, device=x.device)
        # Under non-reentrant checkpointing the backward runs on THIS node with the tensors the recomputation saves in
        # the same slots (same shapes): the slot always exists, but in the pass whose saved tensors are thrown away the
        # kernel does not write it (the allocation is returned to the pool when the pack hook drops it).
        gu = torch.empty((T, 2 * Fdim), dtype=x.dtype, device=x.device) if need else None
        write_gu = gu is not None and not _RECOMPUTED_LATER[0]
        L = nat.require()
        nat.check(L.tb_gemm_swiglu(x2.data_ptr(), w_gu.data_ptr(), h.data_ptr(), gu.data_ptr() if write_gu else 0, T,
                                   Fdim, K, x2.stride(0), w_gu.stride(0), Fdim, 2 * Fdim, nat.num_sms(), nat.stream(),
                                   int(x.dtype == torch.float16)), "tb_gemm_swiglu")
        nat.count_launch()
        if need:
            ctx.save_for_backward(x2, w_gu, gu)
        ctx.w_obj = w_gu
        ctx.x_shape = shp
        return h

    @staticmethod
    def backward(ctx, dh):
        from .linear import gemm
        x2, w, gu = ctx.saved_tensors
        T, Fdim = gu.shape[0], gu.shape[1] // 2
        dh2 = dh.contiguous().view(T, Fdim)
        dgu = torch.empty_like(gu)
        L = nat.require()
        nat.check(
            L.tb_swiglu_bwd(dh2.data_ptr(), gu.data_ptr(), gu.data_ptr() + 2 * Fdim, dgu.data_ptr(),
                            dgu.data_ptr() + 2 * Fdim, T, Fdim, gu.stride(0), gu.stride(0), 2 * Fdim, 2 * Fdim,
                            nat.num_sms(), nat.stream(), nat.bf16_flag(gu)), "tb_swiglu_bwd")
        nat.count_launch()
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(ctx.x_shape, dtype=dgu.dtype, device=dgu.device)
            gemm(dgu, w, b_mn_major=True, out=dx.view(-1, ctx.x_shape[-1]))
        if ctx.needs_input_grad[1]:
            wo = ctx.w_obj
            view = getattr(wo, "_tb_grad_view", None)
            if view is not None:
                acc = bool(getattr(wo, "_tb_grad_ready", False))
                gemm(dgu, x2, a_mn_major=True, b_mn_major=True, out=view, accumulate=acc)
                wo._tb_grad_ready = True
            else:
                dw = gemm(dgu, x2, a_mn_major=True, b_mn_major=True)
        return dx, dw


def gate_up_swiglu(x: torch.Tensor, w_gu: torch.Tensor) -> torch.Tensor:
    """``swiglu(x @ w_gu.T)`` for ``w_gu = [W_gate; W_up]`` ([2F, K]); one fused kernel when eligible."""
    Fdim = w_gu.shape[0] // 2
    from . import fp8
    if (x.is_cuda and nat.is_half(x, w_gu) and nat.use_native(x, w_gu) and Fdim % 128 == 0 and w_gu.stride(1) == 1
            and w_gu.stride(0) % 8 == 0 and not fp8.enabled() and _FUSE_GATE_UP):
        return _GateUpSwiGLUFn.apply(x, w_gu)
    from .linear import linear
    return swiglu(linear(x, w_gu))


import os as _os  # noqa: E402
_FUSE_GATE_UP = _os.environ.get("TORCHACC_B200_FUSE_SWIGLU", "1") != "0"


def swiglu(gu: torch.Tensor) -> torch.Tensor:
    """gu: [..., 2F] with gate in the first half and up in the second half."""
    Fdim = gu.shape[-1] // 2
    if nat.is_half(gu) and nat.use_native(gu) and Fdim % 8 == 0:
        return _SwiGLUFusedFn.apply(gu)
    return (F.silu(gu[..., :Fdim].float()) * gu[..., Fdim:].float()).to(gu.dtype)
