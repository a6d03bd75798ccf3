"""Block-scaled FP8 (MX: e4m3 + one UE8M0 scale per 32 elements) linear layers on wgmma
(csrc/gemm/gemm_mxfp8.cu, csrc/ops/quant_mxfp8.cu).  Enabled by ``Config.compute.fp8``.

All three GEMMs of a linear layer run in fp8 with fp32 accumulation in registers:

    forward  y  = x  W^T : x  quantised along features,   W   along in-features
    dgrad    dx = dy W   : dy quantised along out-features, W^T along out-features   (transposed quantisation of W)
    wgrad    dW = dy^T x : dy^T and x^T quantised along TOKENS                       (transposed quantisation of both)

so every tensor is quantised in one pass that emits both orientations.  The activation saved for backward is the fp8
copy (half the bytes of bf16).  The weight gradient goes straight into the FSDP engine's flat gradient slice
(``_tb_grad_view``) like the bf16 path.  Master weights, optimizer, norms, attention, loss stay as in bf16 training.

The reference has no fp8 mode (torchacc/config.py:27-54); BASELINE.json lists block-scaled fp8 on the GEMM paths.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import _native as nat

nat.register_signatures({
    "tb_quant_mxfp8": ([nat.u64, nat.i64, nat.i32, nat.i32, nat.u64, nat.i64, nat.u64, nat.u64, nat.i64, nat.u64,
                        nat.u64], nat.i32),
    "tb_gemm_mxfp8": ([nat.u64, nat.u64, nat.u64, nat.u64, nat.u64, nat.u64, nat.i32, nat.i32, nat.i32, nat.i64, nat.i64,
                       nat.i64, nat.i64, nat.i32, nat.i32, nat.u64], nat.i32),
})

_ENABLED = False
BLOCK = 32          # elements per scale
ATOM_ROWS, ATOM_K = 128, 128


def enable(flag: bool = True) -> None:
    global _ENABLED
    _ENABLED = bool(flag)


def enabled() -> bool:
    return _ENABLED


def available() -> bool:
    L = nat.lib()
    return L is not None and hasattr(L, "tb_gemm_mxfp8")


class MXTensor:
    """e4m3 payload ``q`` [rows, K] (uint8) + atom-tiled UE8M0 scales ``sf`` for a K-major GEMM operand."""
    __slots__ = ("q", "sf", "rows", "k")

    def __init__(self, q, sf, rows, k):
        self.q, self.sf, self.rows, self.k = q, sf, rows, k


def _sf_buffer(rows: int, k: int, device) -> torch.Tensor:
    atoms_r = (rows + ATOM_ROWS - 1) // ATOM_ROWS
    atoms_k = (k + ATOM_K - 1) // ATOM_K
    return torch.zeros(atoms_r * atoms_k * 512, dtype=torch.uint8, device=device)


def quantize_mxfp8(x: torch.Tensor, rowwise: bool = True, colwise: bool = False) -> Tuple[Optional[MXTensor],
                                                                                           Optional[MXTensor]]:
    """x: bf16 [R, C] (last dim contiguous).  Returns ``(row, col)``: ``row`` = x with scales along C,
    ``col`` = x^T ([C, R]) with scales along R."""
    assert x.dim() == 2 and x.dtype == torch.bfloat16 and x.stride(1) == 1 and x.stride(0) % 8 == 0
    R, C = x.shape
    dev = x.device
    if x.data_ptr() % 16 != 0:   # the kernel loads 16 bytes at a time: copy a view such as x[:, 1:] to an aligned base
        pitch = -(-max(x.stride(0), C) // 8) * 8
        x = torch.empty((R, pitch), dtype=x.dtype, device=dev)[:, :C].copy_(x)
    row = col = None
    q = sf = qt = sft = None
    if rowwise:
        q = torch.empty((R, C), dtype=torch.uint8, device=dev)
        sf = _sf_buffer(R, C, dev)
        row = MXTensor(q, sf, R, C)
    if colwise:
        qt = torch.empty((C, R), dtype=torch.uint8, device=dev)
        sft = _sf_buffer(C, R, dev)
        col = MXTensor(qt, sft, C, R)
    L = nat.require()
    nat.check(L.tb_quant_mxfp8(x.data_ptr(), x.stride(0), R, C, nat.ptr(q), C, nat.ptr(sf), nat.ptr(qt), R,
                               nat.ptr(sft), nat.stream()), "tb_quant_mxfp8")
    nat.count_launch()
    return row, col


def gemm_mxfp8(a: MXTensor, b: MXTensor, out: Optional[torch.Tensor] = None, out_dtype=torch.bfloat16,
               addend: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """``D[M, N] = a[M, K] @ b[N, K]^T (+ addend)``; ``accumulate`` adds into ``out``."""
    assert a.k == b.k and a.k % ATOM_K == 0, "K must be a multiple of 128"
    M, N, K = a.rows, b.rows, a.k
    if out is None:
        assert not accumulate
        out = torch.empty((M, N), dtype=out_dtype, device=a.q.device)
    assert out.stride(1) == 1
    c = out if accumulate else addend
    if c is not None:
        assert c.dtype == out.dtype and c.shape == out.shape and c.stride(1) == 1
    L = nat.require()
    nat.check(L.tb_gemm_mxfp8(a.q.data_ptr(), a.sf.data_ptr(), b.q.data_ptr(), b.sf.data_ptr(), out.data_ptr(),
                              nat.ptr(c), M, N, K, a.q.stride(0), b.q.stride(0), out.stride(0),
                              c.stride(0) if c is not None else 0, int(out.dtype == torch.float32), nat.num_sms(),
                              nat.stream()), "tb_gemm_mxfp8")
    nat.count_launch()
    return out


# ---- reference (de)quantisation: test oracles and the CPU tier ---------------------------------------------------
def sf_to_matrix(sf: torch.Tensor, rows: int, k: int) -> torch.Tensor:
    """Atom-tiled UE8M0 bytes -> float32 scale matrix [rows, k / 32]."""
    atoms_k = (k + ATOM_K - 1) // ATOM_K
    atoms_r = sf.numel() // (512 * atoms_k)
    t = sf.view(atoms_r, atoms_k, 32, 4, 4)            # [row atom, k atom, r % 32, (r % 128) // 32, kblock % 4]
    t = t.permute(0, 3, 2, 1, 4).reshape(atoms_r * 128, atoms_k * 4)
    return torch.pow(2.0, t[:rows, :k // BLOCK].float() - 127.0)


def dequantize_mxfp8(t: MXTensor) -> torch.Tensor:
    vals = t.q.view(torch.float8_e4m3fn).float()
    scale = sf_to_matrix(t.sf, t.rows, t.k).repeat_interleave(BLOCK, dim=1)
    return vals * scale


def quantize_mxfp8_ref(x: torch.Tensor) -> torch.Tensor:
    """fp32 value of x after MX-FP8 quantisation along the last dim (pure PyTorch, any device), as the kernel computes
    it, non-finite input included:
      - a NaN element does not enter its block's amax (the kernel takes it with fmaxf): the block keeps the scale of its
        finite elements and only the NaN element quantises to NaN;
      - an infinite element clamps the scale to 2^127, whose inverse the kernel multiplies by is 0 in fp32: the
        infinity quantises to NaN and every finite element of its block to +-0."""
    R, C = x.shape
    xb = x.float().reshape(R, C // BLOCK, BLOCK)
    a = xb.abs()
    amax = torch.where(torch.isnan(a), torch.zeros_like(a), a).amax(-1, keepdim=True)
    e = torch.ceil(torch.log2(amax / 448.0)).clamp(min=-126, max=127)
    scale = torch.where(amax > 0, torch.pow(2.0, e), torch.ones_like(amax))
    inv = torch.where(torch.isinf(amax), torch.zeros_like(amax), 1.0 / scale)
    q = (xb * inv).to(torch.float8_e4m3fn).float()
    return (q * scale).reshape(R, C)


# ---- autograd ------------------------------------------------------------------------------------------------------
def eligible(x2: torch.Tensor, w: torch.Tensor) -> bool:
    """All three GEMMs need their contraction dim to be a multiple of 128."""
    T, K = x2.shape
    N = w.shape[0]
    return (K % 128 == 0 and N % 128 == 0 and T % 128 == 0 and x2.dtype == torch.bfloat16
            and w.dtype == torch.bfloat16 and nat.use_native(x2, w))


class _Fp8LinearFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, w, bias, residual=None):
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if x2.stride(-1) != 1 or x2.stride(0) % 8 != 0:
            x2 = x2.contiguous()
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        xr, xc = quantize_mxfp8(x2, True, need_dw)                 # x (fwd) and x^T (wgrad) in one pass
        wr, wc = quantize_mxfp8(w, True, need_dx)                  # W (fwd) and W^T (dgrad)
        y = torch.empty((*shp[:-1], w.shape[0]), dtype=x.dtype, device=x.device)
        r2 = None
        if residual is not None:
            r2 = residual.reshape(-1, w.shape[0])
            if r2.stride(-1) != 1:
                r2 = r2.contiguous()
        gemm_mxfp8(xr, wr, out=y.view(-1, w.shape[0]), addend=r2)
        if bias is not None:
            y += bias
        ctx.xc, ctx.wc = xc, wc
        ctx.w_obj = w
        ctx.has_res, ctx.has_bias = residual is not None, bias is not None
        ctx.x_shape = shp
        return y

    @staticmethod
    def backward(ctx, dy):
        dy2 = dy.reshape(-1, dy.shape[-1])
        if dy2.stride(-1) != 1 or dy2.stride(0) % 8 != 0:
            dy2 = dy2.contiguous()
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dyr, dyc = quantize_mxfp8(dy2, need_dx, need_dw)
        dx = dw = db = None
        if need_dx:
            dx = torch.empty(ctx.x_shape, dtype=dy2.dtype, device=dy2.device)
            gemm_mxfp8(dyr, ctx.wc, out=dx.view(-1, ctx.x_shape[-1]))              # dy [T, N] . (W^T [K, N])^T
        if need_dw:
            wo = ctx.w_obj
            view = getattr(wo, "_tb_grad_view", None)
            if view is not None:
                acc = bool(getattr(wo, "_tb_grad_ready", False))
                gemm_mxfp8(dyc, ctx.xc, out=view, accumulate=acc)                  # dy^T [N, T] . (x^T [K, T])^T
                wo._tb_grad_ready = True
            else:
                dw = gemm_mxfp8(dyc, ctx.xc)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(0).to(dy2.dtype)
        ctx.xc = ctx.wc = None
        return dx, dw, db, (dy if ctx.has_res else None)


def fp8_linear(x, w, bias=None, residual=None):
    return _Fp8LinearFn.apply(x, w, bias, residual)
