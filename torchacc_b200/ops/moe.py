"""Mixture-of-experts layers on the grouped wgmma GEMM (csrc/gemm/gemm_bf16.cu, GroupArgs) and the routing kernels of
csrc/ops/moe.cu.

``moe_experts(x, expert_ids, weights, w_gate_up, w_down)`` runs the experts of one MoE layer with HF's 3-D weight
layout (``gate_up_proj [E, 2F, H]``, ``down_proj [E, H, F]``):

    index build -> permute (tokens sorted by expert, each expert padded to 128 rows) -> grouped gate|up GEMM with the
    SwiGLU epilogue -> grouped down GEMM -> weighted combine (+ residual)

The token counts never leave the device: buffers are sized by the upper bound ``T*k + E*127`` rows and the GEMMs read
the real tile count from device memory, so neither the forward nor the backward synchronises with the host.  Every
kernel is deterministic (no float atomics), so repeated steps are bitwise equal.

With ``Config.compute.fp8`` on, bf16 experts whose hidden and intermediate sizes are multiples of 128 run their six
GEMMs in MX-FP8 instead (``_MoEExpertsMXFP8Fn``: the grouped modes of csrc/gemm/gemm_mxfp8.cu, operands quantised by
ops/quant_mxfp8.cu); ``moe_experts_mxfp8_reference`` is its PyTorch emulation.

``moe_router(logits, k, norm_topk_prob)`` is the softmax -> top-k -> renormalise router, and ``MoEMLP`` the module the
native decoder layer uses (parameter names as HF Mixtral: ``gate.weight``, ``experts.gate_up_proj``,
``experts.down_proj``).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _native as nat
from ..utils.logger import logger
from . import fp8
from .swiglu import _RECOMPUTED_LATER

TILE = 128                 # rows per grouped-GEMM tile: every expert's segment is padded to a multiple of it
MAX_EXPERTS, MAX_TOP_K = 256, 8

_u64, _i32, _i64 = nat.u64, nat.i32, nat.i64
nat.register_signatures({
    "tb_gemm_grouped": ([_u64, _u64, _u64, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _i32, _u64, _u64, _i32, _u64,
                         _i32], _i32),
    "tb_gemm_grouped_swiglu": ([_u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _i64, _u64, _u64,
                                _i32, _u64, _i32], _i32),
    "tb_gemm_grouped_wgrad": ([_u64, _u64, _u64, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _u64, _i32, _i32, _i32,
                               _u64, _i32], _i32),
    "tb_gemm_grouped_mxfp8": ([_u64, _u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _i32, _u64,
                               _u64, _i32, _u64], _i32),
    "tb_gemm_grouped_wgrad_mxfp8": ([_u64, _u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _i64, _i64, _i64, _u64,
                                     _i32, _i32, _i32, _u64], _i32),
    "tb_moe_router_fwd": ([_u64, _u64, _u64, _i32, _i32, _i32, _i32, _i32, _u64], _i32),
    "tb_moe_router_bwd": ([_u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _i32, _u64], _i32),
    "tb_moe_index": ([_u64, _i32, _i32, _i32, _i32, _u64, _u64, _u64, _u64, _u64, _u64, _u64], _i32),
    "tb_moe_permute": ([_u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _i32, _u64], _i32),
    "tb_moe_unpermute_sum": ([_u64, _u64, _u64, _i32, _i32, _i32, _i32, _u64, _i32], _i32),
    "tb_moe_combine_fwd": ([_u64, _u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _u64, _i32], _i32),
    "tb_moe_combine_bwd": ([_u64, _u64, _u64, _u64, _u64, _u64, _u64, _i32, _i32, _i32, _i32, _i32, _u64, _i32],
                           _i32),
})

_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
FP8_EXPERT_CALLS = 0       # forwards that took the MX-FP8 expert path


def capacity(T: int, k: int, E: int) -> int:
    """Rows of the expert-sorted buffer: every expert adds at most TILE - 1 padding rows."""
    rows = T * k + E * (TILE - 1)
    return (rows + TILE - 1) // TILE * TILE


# ---- pure-PyTorch reference (CPU path and test oracle) ---------------------------------------------------------------

def moe_router_reference(logits: torch.Tensor, k: int, norm_topk_prob: bool = True):
    p = torch.softmax(logits.float(), dim=-1)
    w, ids = torch.topk(p, k, dim=-1)
    if norm_topk_prob:
        w = w / w.sum(dim=-1, keepdim=True)
    return w, ids


def moe_experts_reference(x, expert_ids, weights, w_gate_up, w_down, residual=None):
    """Loop over experts in fp32: ``out[t] = sum_j w[t,j] * down_e(silu(gate_e(x_t)) * up_e(x_t))``."""
    shp = x.shape
    x2 = x.reshape(-1, shp[-1]).float()
    ids = expert_ids.reshape(x2.shape[0], -1)
    w = weights.reshape(ids.shape).float()
    Fdim = w_gate_up.shape[1] // 2
    out = torch.zeros_like(x2)
    for e in range(w_gate_up.shape[0]):
        tok, slot = torch.where(ids == e)
        if tok.numel() == 0:
            continue
        gu = x2[tok] @ w_gate_up[e].float().t()
        h = F.silu(gu[:, :Fdim]) * gu[:, Fdim:]
        y = (h @ w_down[e].float().t()) * w[tok, slot, None]
        out = out.index_add(0, tok, y)
    if residual is not None:
        out = out + residual.reshape(out.shape).float()
    return out.to(x.dtype).reshape(shp)


def _sorted_layout(ids, E):
    """The expert-sorted, 128-row padded layout of the native index build: ``(pos, offsets)``, where ``pos[i]`` is the
    row of flattened (token, slot) entry i (-1 for an id outside [0, E)), ascending entry order inside an expert."""
    flat = ids.reshape(-1)
    ok = (flat >= 0) & (flat < E)
    counts = torch.bincount(flat[ok], minlength=E).tolist()
    offsets = [0]
    for c in counts:
        offsets.append(offsets[-1] + (c + TILE - 1) // TILE * TILE)
    pos = torch.full_like(flat, -1)
    entries = ok.nonzero().flatten()
    src = entries[torch.argsort(flat[entries], stable=True)]
    start = 0
    for e, c in enumerate(counts):
        pos[src[start:start + c]] = offsets[e] + torch.arange(c, device=flat.device)
        start += c
    return pos, offsets


def moe_experts_mxfp8_reference(x, expert_ids, weights, w_gate_up, w_down, residual=None, dout=None):
    """PyTorch emulation of the MX-FP8 expert path (test oracle): every GEMM operand quantised by
    ``fp8.quantize_mxfp8_ref`` in the orientation the kernel reads it, products summed in fp64, and bf16 rounding where
    the native path rounds (pre-activation, h, y_perm, dy_perm, dh, dgu, dx_perm and the outputs).  Returns ``out``;
    with ``dout``, ``(out, dx, dweights, dW_gate_up, dW_down)`` (weight gradients in fp64)."""
    q = fp8.quantize_mxfp8_ref
    f64, bf16 = torch.float64, torch.bfloat16

    def rnd(t):
        return t.to(bf16).to(f64)

    shp = x.shape
    H = shp[-1]
    x2 = x.reshape(-1, H)
    T = x2.shape[0]
    ids = expert_ids.reshape(T, -1)
    k = ids.shape[1]
    w = weights.reshape(T, k).float().to(f64)
    E, F2, _ = w_gate_up.shape
    Fd = F2 // 2
    pos, off = _sorted_layout(ids, E)
    rows = max(off[-1], TILE)
    ent = (pos >= 0).nonzero().flatten()
    rws, tok = pos[ent], ent // k
    xp = torch.zeros(rows, H, dtype=f64, device=x.device)
    xp[rws] = x2[tok].to(f64)

    def grouped(a, b, n, transposed):
        """a [rows, K] times B_e^T per expert segment; b = [E*n, K], or (transposed) [n, E*K]."""
        out = torch.zeros(rows, n, dtype=f64, device=a.device)
        K = a.shape[1]
        for e in range(E):
            r = slice(off[e], off[e + 1])
            if r.stop > r.start:
                be = b[:, e * K:(e + 1) * K] if transposed else b[e * n:(e + 1) * n]
                out[r] = a[r] @ be.t()
        return out

    def wgrad(a_t, b_t, m, n):
        """[E, m, n]: a_t [m, rows] times b_t [n, rows]^T over every expert's padded rows."""
        out = torch.zeros(E, m, n, dtype=f64, device=a_t.device)
        for e in range(E):
            r = slice(off[e], off[e + 1])
            out[e] = a_t[:, r] @ b_t[:, r].t()
        return out

    wgu2 = w_gate_up.reshape(E * F2, H)
    wd2 = w_down.reshape(E * H, Fd)
    gu = rnd(grouped(q(xp).to(f64), q(wgu2).to(f64), F2, False))
    g, u = gu[:, :Fd], gu[:, Fd:]
    sg = torch.sigmoid(g)
    h = rnd(g * sg * u)
    y = rnd(grouped(q(h).to(f64), q(wd2).to(f64), H, False))
    per = torch.zeros(T * k, H, dtype=f64, device=x.device)
    per[ent] = y[rws] * w.reshape(-1)[ent, None]
    out = per.view(T, k, H).sum(1)
    if residual is not None:
        out = out + residual.reshape(T, H).to(f64)
    out = out.to(x.dtype).reshape(shp)
    if dout is None:
        return out
    d2 = dout.reshape(T, H).to(f64)
    dyp = torch.zeros(rows, H, dtype=f64, device=x.device)
    dyp[rws] = rnd(d2[tok] * w.reshape(-1)[ent, None])
    dw = torch.zeros(T * k, dtype=f64, device=x.device)
    dw[ent] = (y[rws] * d2[tok]).sum(1)
    dh = rnd(grouped(q(dyp).to(f64), q(wd2.t()).to(f64), Fd, True))
    dg = rnd(dh * u * (sg + g * sg * (1 - sg)))
    du = rnd(dh * g * sg)
    dgu = torch.cat([dg, du], 1)
    dxp = rnd(grouped(q(dgu).to(f64), q(wgu2.t()).to(f64), H, True))
    per = torch.zeros(T * k, H, dtype=f64, device=x.device)
    per[ent] = dxp[rws]
    dx = per.view(T, k, H).sum(1).to(x.dtype).reshape(shp)
    d_down = wgrad(q(dyp.t()).to(f64), q(h.t()).to(f64), H, Fd)
    d_gu = wgrad(q(dgu.t()).to(f64), q(xp.t()).to(f64), F2, H)
    return out, dx, dw.view(weights.shape).to(weights.dtype), d_gu, d_down


# ---- native path -----------------------------------------------------------------------------------------------------

class MoEIndex:
    """Device-resident routing schedule of one call (see csrc/ops/moe.cu, moe_index_kernel)."""

    def __init__(self, expert_ids: torch.Tensor, num_experts: int):
        ids = expert_ids.reshape(-1, expert_ids.shape[-1])   # [T, k]; -1 in the last place is ambiguous at T = 0
        if ids.dtype != torch.int64:
            ids = ids.long()
        ids = ids.contiguous()
        T, k = ids.shape
        E = num_experts
        dev = ids.device
        self.T, self.k, self.E = T, k, E
        self.rows = capacity(T, k, E)
        i32 = torch.int32
        self.counts = torch.empty(E, dtype=i32, device=dev)
        self.offsets = torch.empty(E + 1, dtype=i32, device=dev)
        self.tile_expert = torch.empty(self.rows // TILE, dtype=i32, device=dev)
        self.num_m_tiles = torch.empty(1, dtype=i32, device=dev)
        self.pos = torch.empty((T, k), dtype=i32, device=dev)
        self.row_src = torch.empty(self.rows, dtype=i32, device=dev)
        L = nat.require()
        nat.check(L.tb_moe_index(ids.data_ptr(), T, k, E, self.rows, self.counts.data_ptr(), self.offsets.data_ptr(),
                                 self.tile_expert.data_ptr(), self.num_m_tiles.data_ptr(), self.pos.data_ptr(),
                                 self.row_src.data_ptr(), nat.stream()), "tb_moe_index")
        nat.count_launch()

    def tensors(self):
        return self.counts, self.offsets, self.tile_expert, self.num_m_tiles, self.pos, self.row_src


def _f16(t):
    return int(t.dtype == torch.float16)


def _rows16(t, H):
    """``t`` as contiguous ``[rows, H]`` rows on a 16-byte aligned base (the row movers load 16 bytes per thread)."""
    t2 = t.reshape(-1, H).contiguous()
    if t2.data_ptr() % 16 != 0:
        t2 = t2.clone()
    return t2


def grouped_gemm(a, w, idx: MoEIndex, *, b_mn_major: bool = False, out=None):
    """``out[r] = a[r] @ B_e^T`` for every sorted row r of expert e; ``w`` is ``[E, N, K]`` (``b_mn_major``: ``[E, K, N]``,
    read transposed)."""
    E = w.shape[0]
    K = a.shape[1]
    N = w.shape[2] if b_mn_major else w.shape[1]
    assert w.shape[1 if b_mn_major else 2] == K
    w2 = w.reshape(E * w.shape[1], w.shape[2])
    if out is None:
        out = torch.empty((a.shape[0], N), dtype=a.dtype, device=a.device)
    L = nat.require()
    nat.check(L.tb_gemm_grouped(a.data_ptr(), w2.data_ptr(), out.data_ptr(), a.shape[0], N, K, E, a.stride(0),
                                w2.stride(0), out.stride(0), int(b_mn_major), idx.tile_expert.data_ptr(),
                                idx.num_m_tiles.data_ptr(), nat.num_sms(), nat.stream(), _f16(a)), "tb_gemm_grouped")
    nat.count_launch()
    return out


def grouped_swiglu(a, w_gate_up, idx: MoEIndex, gu_out=None):
    """``h[r] = silu(a[r] Wg_e^T) * (a[r] Wu_e^T)`` with ``w_gate_up [E, 2F, K]``; ``gu_out`` ([rows, 2F]) receives the
    pre-activation when given."""
    E, F2, K = w_gate_up.shape
    Fdim = F2 // 2
    h = torch.empty((a.shape[0], Fdim), dtype=a.dtype, device=a.device)
    w2 = w_gate_up.reshape(E * F2, K)
    L = nat.require()
    nat.check(L.tb_gemm_grouped_swiglu(a.data_ptr(), w2.data_ptr(), h.data_ptr(), nat.ptr(gu_out), a.shape[0], Fdim, K,
                                       E, a.stride(0), w2.stride(0), h.stride(0), 2 * Fdim, idx.tile_expert.data_ptr(),
                                       idx.num_m_tiles.data_ptr(), nat.num_sms(), nat.stream(), _f16(a)),
              "tb_gemm_grouped_swiglu")
    nat.count_launch()
    return h


def grouped_wgrad(dy, x, idx: MoEIndex, out, accumulate: bool = False):
    """``out[e] (+)= dy_e^T x_e`` over expert e's sorted rows; ``out`` is ``[E, M, N]`` (fp32 or dy's dtype)."""
    E, M, N = out.shape
    o2 = out.view(E * M, N)
    assert o2.stride(1) == 1 and dy.shape[1] == M and x.shape[1] == N
    L = nat.require()
    nat.check(L.tb_gemm_grouped_wgrad(dy.data_ptr(), x.data_ptr(), o2.data_ptr(), M, N, E, dy.shape[0], dy.stride(0),
                                      x.stride(0), o2.stride(0), idx.offsets.data_ptr(),
                                      int(out.dtype == torch.float32), int(accumulate), nat.num_sms(), nat.stream(),
                                      _f16(dy)), "tb_gemm_grouped_wgrad")
    nat.count_launch()
    return out


def _weight_grad(wgrad, w_obj, like):
    """Weight gradient ``wgrad(out, accumulate)`` straight into the engine's flat-buffer view when there is one (see
    ops/linear.py)."""
    view = getattr(w_obj, "_tb_grad_view", None)
    if view is not None:
        wgrad(view, bool(getattr(w_obj, "_tb_grad_ready", False)))
        w_obj._tb_grad_ready = True
        return None
    return wgrad(torch.empty_like(like), False)


class _MoEExpertsFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weights, w_gate_up, w_down, expert_ids, residual, index):
        shp = x.shape
        H = shp[-1]
        x2 = _rows16(x, H)
        T = x2.shape[0]
        E, F2, _ = w_gate_up.shape
        idx = index if index is not None else MoEIndex(expert_ids.reshape(T, -1), E)
        if (idx.T, idx.E) != (T, E):
            raise ValueError(f"MoEIndex built for {idx.T} tokens and {idx.E} experts, called with {T} and {E}")
        k = idx.k
        w32 = weights.reshape(T, k).float().contiguous()
        L = nat.require()
        bf = nat.bf16_flag(x2)
        x_perm = torch.empty((idx.rows, H), dtype=x.dtype, device=x.device)
        nat.check(L.tb_moe_permute(x2.data_ptr(), idx.row_src.data_ptr(), idx.offsets.data_ptr(), x_perm.data_ptr(),
                                   idx.rows, k, E, H, nat.num_sms(), nat.stream()), "tb_moe_permute")
        nat.count_launch()
        need = any(ctx.needs_input_grad[:4])
        # as _GateUpSwiGLUFn: the pre-activation slot always exists when a backward may run, but it is not written in
        # the forward whose saved tensors the checkpointing recomputation replaces
        gu = torch.empty((idx.rows, F2), dtype=x.dtype, device=x.device) if need else None
        write_gu = gu is not None and not _RECOMPUTED_LATER[0]
        h = grouped_swiglu(x_perm, w_gate_up, idx, gu if write_gu else None)
        y_perm = grouped_gemm(h, w_down, idx)
        out = torch.empty(shp, dtype=x.dtype, device=x.device)
        res = None
        if residual is not None:
            res = _rows16(residual, H)
        nat.check(L.tb_moe_combine_fwd(y_perm.data_ptr(), idx.pos.data_ptr(), w32.data_ptr(), nat.ptr(res),
                                       out.data_ptr(), T, k, H, nat.num_sms(), nat.stream(), bf), "tb_moe_combine_fwd")
        nat.count_launch()
        ctx.need = need
        if need:
            ctx.save_for_backward(x_perm, gu, h, y_perm, w32, w_gate_up, w_down, *idx.tensors())
        ctx.idx_meta = (T, k, E, idx.rows)
        ctx.w_objs = (w_gate_up, w_down)
        ctx.shape, ctx.w_dtype = shp, weights.dtype
        ctx.has_res = residual is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        if not ctx.need:   # only the residual asked for a gradient
            return None, None, None, None, None, dout, None
        x_perm, gu, h, y_perm, w32, w_gate_up, w_down, *it = ctx.saved_tensors
        T, k, E, rows = ctx.idx_meta
        idx = MoEIndex.__new__(MoEIndex)
        idx.T, idx.k, idx.E, idx.rows = T, k, E, rows
        idx.counts, idx.offsets, idx.tile_expert, idx.num_m_tiles, idx.pos, idx.row_src = it
        H = x_perm.shape[1]
        F2 = gu.shape[1]
        Fdim = F2 // 2
        dout2 = _rows16(dout, H)
        L = nat.require()
        bf = nat.bf16_flag(dout2)
        dy_perm = torch.empty((rows, H), dtype=dout2.dtype, device=dout2.device)
        # zeros: an entry with an expert id outside [0, E) owns no sorted row, so the combine backward never writes it
        dw = torch.zeros((T, k), dtype=torch.float32, device=dout2.device)
        nat.check(L.tb_moe_combine_bwd(dout2.data_ptr(), y_perm.data_ptr(), idx.row_src.data_ptr(),
                                       idx.offsets.data_ptr(), w32.data_ptr(), dy_perm.data_ptr(), dw.data_ptr(), rows,
                                       k, E, H, nat.num_sms(), nat.stream(), bf), "tb_moe_combine_bwd")
        nat.count_launch()
        w_gu_obj, w_down_obj = ctx.w_objs
        d_down = d_gu = None
        dh = grouped_gemm(dy_perm, w_down, idx, b_mn_major=True)                   # dh = dy W_down_e
        if ctx.needs_input_grad[3]:
            d_down = _weight_grad(lambda o, acc: grouped_wgrad(dy_perm, h, idx, o, acc),   # dW_down_e = dy_e^T h_e
                                  w_down_obj, w_down)
        dgu = torch.empty_like(gu)
        nat.check(L.tb_swiglu_bwd(dh.data_ptr(), gu.data_ptr(), gu.data_ptr() + 2 * Fdim, dgu.data_ptr(),
                                  dgu.data_ptr() + 2 * Fdim, rows, Fdim, F2, F2, F2, F2, nat.num_sms(), nat.stream(), bf),
                  "tb_swiglu_bwd")
        nat.count_launch()
        dx = None
        if ctx.needs_input_grad[0]:
            dx_perm = grouped_gemm(dgu, w_gate_up, idx, b_mn_major=True)            # dx_perm = dgu W_gu_e
            dx = torch.empty(ctx.shape, dtype=dout2.dtype, device=dout2.device)
            nat.check(L.tb_moe_unpermute_sum(dx_perm.data_ptr(), idx.pos.data_ptr(), dx.data_ptr(), T, k, H,
                                             nat.num_sms(), nat.stream(), bf), "tb_moe_unpermute_sum")
            nat.count_launch()
        if ctx.needs_input_grad[2]:
            d_gu = _weight_grad(lambda o, acc: grouped_wgrad(dgu, x_perm, idx, o, acc),    # dW_gu_e = dgu_e^T x_e
                                w_gu_obj, w_gate_up)
        dweights = dw.reshape(ctx.shape[:-1] + (k,)) if len(ctx.shape) > 2 else dw
        dweights = dweights.to(ctx.w_dtype) if ctx.needs_input_grad[1] else None
        return dx, dweights, d_gu, d_down, None, (dout if ctx.has_res else None), None


def grouped_gemm_mxfp8(a: fp8.MXTensor, b: fp8.MXTensor, idx: MoEIndex, *, transposed: bool = False):
    """``out[r] = a[r] @ B_e^T`` (bf16) for every sorted row r of expert e.  ``b`` is the quantised ``[E*N, K]`` weight
    (forward) or, ``transposed``, the transposed quantisation ``[N, E*K]`` of an ``[E*K, N]`` weight (dgrad)."""
    E, K = idx.E, a.k
    N = b.rows if transposed else b.rows // E
    assert b.k == (E * K if transposed else K)
    out = torch.empty((a.rows, N), dtype=torch.bfloat16, device=a.q.device)
    L = nat.require()
    nat.check(L.tb_gemm_grouped_mxfp8(a.q.data_ptr(), a.sf.data_ptr(), b.q.data_ptr(), b.sf.data_ptr(), out.data_ptr(),
                                      a.rows, N, K, E, a.q.stride(0), b.q.stride(0), out.stride(0), int(transposed),
                                      idx.tile_expert.data_ptr(), idx.num_m_tiles.data_ptr(), nat.num_sms(),
                                      nat.stream()), "tb_gemm_grouped_mxfp8")
    nat.count_launch()
    return out


def grouped_wgrad_mxfp8(dyt: fp8.MXTensor, xt: fp8.MXTensor, idx: MoEIndex, out, accumulate: bool = False):
    """``out[e] (+)= dy_e^T x_e`` over expert e's sorted rows from the transposed quantisations ``dyt [M, rows]`` and
    ``xt [N, rows]``; ``out`` is ``[E, M, N]`` (fp32 or bf16)."""
    E, M, N = out.shape
    o2 = out.view(E * M, N)
    assert o2.stride(1) == 1 and dyt.rows == M and xt.rows == N and dyt.k == xt.k
    L = nat.require()
    nat.check(L.tb_gemm_grouped_wgrad_mxfp8(dyt.q.data_ptr(), dyt.sf.data_ptr(), xt.q.data_ptr(), xt.sf.data_ptr(),
                                            o2.data_ptr(), M, N, E, dyt.k, dyt.q.stride(0), xt.q.stride(0),
                                            o2.stride(0), idx.offsets.data_ptr(), int(out.dtype == torch.float32),
                                            int(accumulate), nat.num_sms(), nat.stream()),
              "tb_gemm_grouped_wgrad_mxfp8")
    nat.count_launch()
    return out


class _MoEExpertsMXFP8Fn(torch.autograd.Function):
    """The experts with all six GEMMs in MX-FP8.  Activations are quantised once, in both orientations where the
    backward needs the second: the backward keeps the fp8 transposed copies x^T and h^T (through ``save_for_backward``,
    so activation checkpointing drops and recomputes them) instead of the bf16 x_perm and h.  The weights are saved as
    they are, like the bf16 path does, and the backward quantises their transposed orientation (W_gu^T, W_down^T) when
    it needs it, so no fp8 weight copy lives from the forward to the backward.  The quantiser also runs over the capacity rows past the device-side tile count, which no
    kernel writes: their row-wise scales sit in row tiles the GEMMs never load, and their column-wise scales in K
    blocks past offsets[E], which no expert's K range reaches, so whatever they hold cannot reach a result."""

    @staticmethod
    def forward(ctx, x, weights, w_gate_up, w_down, expert_ids, residual, index):
        global FP8_EXPERT_CALLS
        FP8_EXPERT_CALLS += 1
        shp = x.shape
        H = shp[-1]
        x2 = _rows16(x, H)
        T = x2.shape[0]
        E, F2, _ = w_gate_up.shape
        Fdim = F2 // 2
        idx = index if index is not None else MoEIndex(expert_ids.reshape(T, -1), E)
        if (idx.T, idx.E) != (T, E):
            raise ValueError(f"MoEIndex built for {idx.T} tokens and {idx.E} experts, called with {T} and {E}")
        k, rows = idx.k, idx.rows
        w32 = weights.reshape(T, k).float().contiguous()
        L = nat.require()
        x_perm = torch.empty((rows, H), dtype=x.dtype, device=x.device)
        nat.check(L.tb_moe_permute(x2.data_ptr(), idx.row_src.data_ptr(), idx.offsets.data_ptr(), x_perm.data_ptr(),
                                   rows, k, E, H, nat.num_sms(), nat.stream()), "tb_moe_permute")
        nat.count_launch()
        need_dx, need_gu, need_down = ctx.needs_input_grad[0], ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        need_dh = need_dx or need_gu
        xr, xc = fp8.quantize_mxfp8(x_perm, True, need_gu)
        gur, _ = fp8.quantize_mxfp8(w_gate_up.view(E * F2, H))
        gu = grouped_gemm_mxfp8(xr, gur, idx)                                    # [rows, 2F] = x W_gu_e^T
        h = torch.empty((rows, Fdim), dtype=x.dtype, device=x.device)
        nat.check(L.tb_swiglu_fwd(gu.data_ptr(), gu.data_ptr() + 2 * Fdim, h.data_ptr(), rows, Fdim, F2, F2,
                                  nat.num_sms(), nat.stream(), 1), "tb_swiglu_fwd")
        nat.count_launch()
        hr, hc = fp8.quantize_mxfp8(h, True, need_down)
        wdr, _ = fp8.quantize_mxfp8(w_down.view(E * H, Fdim))
        y_perm = grouped_gemm_mxfp8(hr, wdr, idx)                                # [rows, H] = h W_down_e^T
        out = torch.empty(shp, dtype=x.dtype, device=x.device)
        res = _rows16(residual, H) if residual is not None else None
        nat.check(L.tb_moe_combine_fwd(y_perm.data_ptr(), idx.pos.data_ptr(), w32.data_ptr(), nat.ptr(res),
                                       out.data_ptr(), T, k, H, nat.num_sms(), nat.stream(), 1), "tb_moe_combine_fwd")
        nat.count_launch()
        ctx.need = any(ctx.needs_input_grad[:4])
        if ctx.need:
            xq, xs = (xc.q, xc.sf) if xc is not None else (None, None)
            hq, hs = (hc.q, hc.sf) if hc is not None else (None, None)
            ctx.save_for_backward(gu if need_dh else None, y_perm, w32, w_gate_up, w_down, xq, xs, hq, hs,
                                  *idx.tensors())
        ctx.idx_meta = (T, k, E, rows, H, Fdim)
        ctx.w_objs = (w_gate_up, w_down)
        ctx.shape, ctx.w_dtype = shp, weights.dtype
        ctx.has_res = residual is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        if not ctx.need:   # only the residual asked for a gradient
            return None, None, None, None, None, dout, None
        gu, y_perm, w32, w_gate_up, w_down, xc_q, xc_sf, hc_q, hc_sf, *it = ctx.saved_tensors
        T, k, E, rows, H, Fdim = ctx.idx_meta
        F2 = 2 * Fdim
        idx = MoEIndex.__new__(MoEIndex)
        idx.T, idx.k, idx.E, idx.rows = T, k, E, rows
        idx.counts, idx.offsets, idx.tile_expert, idx.num_m_tiles, idx.pos, idx.row_src = it
        need_dx, need_gu, need_down = ctx.needs_input_grad[0], ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        dout2 = _rows16(dout, H)
        L = nat.require()
        dy_perm = torch.empty((rows, H), dtype=dout2.dtype, device=dout2.device)
        dw = torch.zeros((T, k), dtype=torch.float32, device=dout2.device)   # sentinel entries own no row
        nat.check(L.tb_moe_combine_bwd(dout2.data_ptr(), y_perm.data_ptr(), idx.row_src.data_ptr(),
                                       idx.offsets.data_ptr(), w32.data_ptr(), dy_perm.data_ptr(), dw.data_ptr(), rows,
                                       k, E, H, nat.num_sms(), nat.stream(), 1), "tb_moe_combine_bwd")
        nat.count_launch()
        w_gu_obj, w_down_obj = ctx.w_objs
        d_down = d_gu = dx = None
        dyr, dyc = fp8.quantize_mxfp8(dy_perm, need_dx or need_gu, need_down)
        if need_down:
            hc = fp8.MXTensor(hc_q, hc_sf, *hc_q.shape)
            d_down = _weight_grad(lambda o, acc: grouped_wgrad_mxfp8(dyc, hc, idx, o, acc),   # dW_down_e = dy_e^T h_e
                                  w_down_obj, w_down_obj)
        if need_dx or need_gu:
            _, wdc = fp8.quantize_mxfp8(w_down.view(E * H, Fdim), False, True)         # W_down^T [F, E*H]
            dh = grouped_gemm_mxfp8(dyr, wdc, idx, transposed=True)                    # dh = dy W_down_e
            del wdc
            dgu = torch.empty_like(gu)
            nat.check(L.tb_swiglu_bwd(dh.data_ptr(), gu.data_ptr(), gu.data_ptr() + 2 * Fdim, dgu.data_ptr(),
                                      dgu.data_ptr() + 2 * Fdim, rows, Fdim, F2, F2, F2, F2, nat.num_sms(),
                                      nat.stream(), 1), "tb_swiglu_bwd")
            nat.count_launch()
            dgur, dguc = fp8.quantize_mxfp8(dgu, need_dx, need_gu)
            if need_dx:
                _, guc = fp8.quantize_mxfp8(w_gate_up.view(E * F2, H), False, True)   # W_gu^T [H, E*2F]
                dx_perm = grouped_gemm_mxfp8(dgur, guc, idx, transposed=True)          # dx_perm = dgu W_gu_e
                del guc
                dx = torch.empty(ctx.shape, dtype=dout2.dtype, device=dout2.device)
                nat.check(L.tb_moe_unpermute_sum(dx_perm.data_ptr(), idx.pos.data_ptr(), dx.data_ptr(), T, k, H,
                                                 nat.num_sms(), nat.stream(), 1), "tb_moe_unpermute_sum")
                nat.count_launch()
            if need_gu:
                xc = fp8.MXTensor(xc_q, xc_sf, *xc_q.shape)
                d_gu = _weight_grad(lambda o, acc: grouped_wgrad_mxfp8(dguc, xc, idx, o, acc),   # dW_gu_e = dgu_e^T x_e
                                    w_gu_obj, w_gu_obj)
        dweights = dw.reshape(ctx.shape[:-1] + (k,)) if len(ctx.shape) > 2 else dw
        dweights = dweights.to(ctx.w_dtype) if ctx.needs_input_grad[1] else None
        return dx, dweights, d_gu, d_down, None, (dout if ctx.has_res else None), None


_WARNED = set()


def _native_ok(x, w_gate_up, w_down) -> bool:
    if not (x.is_cuda and nat.is_half(x, w_gate_up, w_down) and nat.use_native(x, w_gate_up, w_down)):
        return False
    E, F2, H = w_gate_up.shape
    why = None
    if (F2 // 2) % 128 != 0:
        why = f"intermediate size {F2 // 2} is not a multiple of 128"
    elif H % 8 != 0:
        why = f"hidden size {H} is not a multiple of 8"
    elif E > MAX_EXPERTS:
        why = f"{E} experts (at most {MAX_EXPERTS})"
    elif not (w_gate_up.is_contiguous() and w_down.is_contiguous()):
        why = "expert weights are not contiguous"
    elif w_gate_up.data_ptr() % 16 != 0 or w_down.data_ptr() % 16 != 0:
        why = "expert weights are not 16-byte aligned"
    if why is not None:
        if why not in _WARNED:
            _WARNED.add(why)
            logger.warning(f"moe_experts: {why}; using the PyTorch reference path")
        return False
    return True


def _fp8_ok(x, w_gate_up, w_down) -> bool:
    """The MX-FP8 expert path: ``compute.fp8`` on, bf16 input and weights, hidden and intermediate sizes multiples of
    128 (every GEMM's contraction dimension, and each expert's slice of a quantised weight, whole scale atoms)."""
    if not fp8.enabled() or not (x.dtype == w_gate_up.dtype == w_down.dtype == torch.bfloat16):
        return False
    _, F2, H = w_gate_up.shape
    return H % 128 == 0 and (F2 // 2) % 128 == 0


def moe_experts(x: torch.Tensor, expert_ids: torch.Tensor, weights: torch.Tensor, w_gate_up: torch.Tensor,
                w_down: torch.Tensor, residual: torch.Tensor | None = None,
                index: MoEIndex | None = None) -> torch.Tensor:
    """Experts of one MoE layer: ``out[t] = sum_j weights[t,j] * expert_{ids[t,j]}(x[t]) (+ residual[t])``.

    ``x [..., H]``, ``expert_ids`` / ``weights [..., k]``, ``w_gate_up [E, 2F, H]`` (gate rows first, as HF),
    ``w_down [E, H, F]``.  Differentiable in x, weights, both weights tensors and residual.  An expert id outside
    ``[0, E)`` (HF uses ``E`` as a "no expert" sentinel) contributes nothing and gets a zero weight gradient.
    ``index`` is a ``MoEIndex`` already built for these ids (native path only; built here when omitted).  Under
    ``Config.compute.fp8`` eligible bf16 experts run their GEMMs in MX-FP8 (see ``_fp8_ok``)."""
    if _native_ok(x, w_gate_up, w_down):
        if _fp8_ok(x, w_gate_up, w_down):
            return _MoEExpertsMXFP8Fn.apply(x, weights, w_gate_up, w_down, expert_ids, residual, index)
        return _MoEExpertsFn.apply(x, weights, w_gate_up, w_down, expert_ids, residual, index)
    return moe_experts_reference(x, expert_ids, weights, w_gate_up, w_down, residual)


class _MoERouterFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, logits, k, norm):
        E = logits.shape[-1]
        l2 = logits.reshape(-1, E).contiguous()
        T = l2.shape[0]
        w = torch.empty((T, k), dtype=torch.float32, device=logits.device)
        ids = torch.empty((T, k), dtype=torch.int64, device=logits.device)
        L = nat.require()
        nat.check(L.tb_moe_router_fwd(l2.data_ptr(), w.data_ptr(), ids.data_ptr(), T, E, k, int(norm),
                                      _DTYPE_CODE[l2.dtype], nat.stream()), "tb_moe_router_fwd")
        nat.count_launch()
        ctx.save_for_backward(l2, ids)
        ctx.k, ctx.norm, ctx.shape = k, norm, logits.shape
        ctx.mark_non_differentiable(ids)
        lead = logits.shape[:-1]
        return w.view(*lead, k), ids.view(*lead, k)

    @staticmethod
    def backward(ctx, dw, _dids):
        l2, ids = ctx.saved_tensors
        T, E = l2.shape
        dw2 = dw.reshape(T, ctx.k).float().contiguous()
        dl = torch.empty_like(l2)
        L = nat.require()
        nat.check(L.tb_moe_router_bwd(l2.data_ptr(), ids.data_ptr(), dw2.data_ptr(), dl.data_ptr(), T, E, ctx.k,
                                      int(ctx.norm), _DTYPE_CODE[l2.dtype], nat.stream()), "tb_moe_router_bwd")
        nat.count_launch()
        return dl.view(ctx.shape), None, None


def moe_router(logits: torch.Tensor, k: int, norm_topk_prob: bool = True):
    """softmax(logits) -> top-k -> (renormalised) weights.  Returns ``(weights fp32 [..., k], expert_ids int64 [..., k])``;
    the weights are differentiable in the logits."""
    E = logits.shape[-1]
    if E > MAX_EXPERTS or k > MAX_TOP_K or k > E:
        raise ValueError(f"moe_router supports at most {MAX_EXPERTS} experts and top-{MAX_TOP_K} (got E={E}, k={k})")
    if logits.is_cuda and logits.dtype in _DTYPE_CODE and nat.use_native(logits):
        return _MoERouterFn.apply(logits, k, norm_topk_prob)
    return moe_router_reference(logits, k, norm_topk_prob)


class MoEExperts(nn.Module):
    """3-D expert weights in HF's layout (``gate_up_proj [E, 2F, H]``, ``down_proj [E, H, F]``)."""

    def __init__(self, num_experts: int, hidden_size: int, intermediate_size: int, **kw):
        super().__init__()
        self.gate_up_proj = nn.Parameter(torch.empty(num_experts, 2 * intermediate_size, hidden_size, **kw))
        self.down_proj = nn.Parameter(torch.empty(num_experts, hidden_size, intermediate_size, **kw))
        # the sharding engines hand these weight gradients to the grouped wgrad through _tb_grad_view
        self.gate_up_proj._tb_gemm_weight = True
        self.down_proj._tb_gemm_weight = True

    def forward(self, x, expert_ids, weights, residual=None):
        return moe_experts(x, expert_ids, weights, self.gate_up_proj, self.down_proj, residual)


class MoEMLP(nn.Module):
    """Router (``gate``: ``[E, H]`` linear -> softmax -> top-k) + experts.  ``forward(x, residual=None)`` returns the
    layer output (plus the residual when given); ``last_router_logits`` and ``last_counts`` (device-resident routed
    (token, slot) pairs per expert) of the latest call feed the load-balancing loss."""

    def __init__(self, hidden_size: int, intermediate_size: int, num_experts: int, top_k: int,
                 norm_topk_prob: bool = True, **kw):
        super().__init__()
        if num_experts > MAX_EXPERTS or top_k > MAX_TOP_K or top_k > num_experts:
            raise ValueError(f"MoEMLP supports at most {MAX_EXPERTS} experts and top-{MAX_TOP_K}")
        self.num_experts, self.top_k, self.norm_topk_prob = num_experts, top_k, norm_topk_prob
        self.gate = nn.Linear(hidden_size, num_experts, bias=False, **kw)
        self.experts = MoEExperts(num_experts, hidden_size, intermediate_size, **kw)
        self.last_router_logits = None
        self.last_counts = None

    def forward(self, x, residual=None):
        from .linear import linear
        # the native GEMM needs 16-byte row pitches: a router with E % 8 != 0 (Qwen1.5-MoE's 60) is a tiny [T, E] GEMM
        # left to PyTorch
        w = self.gate.weight
        logits = linear(x, w) if self.num_experts % 8 == 0 else F.linear(x, w)
        weights, ids = moe_router(logits, self.top_k, self.norm_topk_prob)
        ex = self.experts
        index = None
        if _native_ok(x, ex.gate_up_proj, ex.down_proj):
            index = MoEIndex(ids, self.num_experts)     # its counts stay on the device
            counts = index.counts
        else:
            counts = F.one_hot(ids.reshape(-1), self.num_experts).sum(0)
        self.last_router_logits, self.last_counts = logits, counts
        return moe_experts(x, ids, weights, ex.gate_up_proj, ex.down_proj, residual, index=index)


def load_balancing_loss(router_logits, counts, num_experts: int) -> torch.Tensor:
    """Switch-style auxiliary loss over a model's MoE layers, on the scale of HF Mixtral's ``load_balancing_loss_func``
    (so Mixtral's ``router_aux_loss_coef`` means the same here):  ``E * sum_e (C_e / N) * P_e``, where N is the number of
    tokens summed over the layers, C_e the (token, slot) pairs routed to expert e over the layers, and P_e the mean
    router probability of expert e over the same N tokens.

    ``router_logits``: one ``[T, E]`` tensor per layer; ``counts``: one ``[E]`` integer tensor per layer (the
    device-resident counts of the index build, so nothing synchronises with the host)."""
    p = torch.cat([l.reshape(-1, num_experts) for l in router_logits]).float().softmax(-1)
    c = torch.stack([x.reshape(num_experts) for x in counts]).sum(0).float()
    return num_experts * (c / p.shape[0] * p.mean(0)).sum()
