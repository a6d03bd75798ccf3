"""Ring / blockwise context-parallel attention (reference torchacc/ops/context_parallel/ring_attn.py:22-508).

Q stays put, K/V blocks of the other ranks are visited one at a time and merged with the running (out, lse) pair in
fp32.  Differences from the reference:
* **causal load balancing**: with ``zigzag=True`` rank r holds sequence chunks ``r`` and ``2cp-1-r``; every step then
  costs half a block on every rank (the reference skips blocks, so rank r does r+1 of them -- SURVEY 5.7);
* K/V movement: on one NVSwitch domain all K/V blocks are fetched with ONE peer-memory all-gather (GQA K/V are
  small) and the loop runs without per-step communication; ``impl="p2p"`` keeps the classic isend/irecv ring with
  the next transfer always in flight while the current block is attended to (``_LazyRing``);
* backward: per-block flash backward with the GLOBAL out/lse, dQ accumulated locally, the dK/dV contributions are
  returned to their owners with one reduce-scatter (fp32 accumulate) instead of a second ring;
* the causal flag is only applied to the diagonal block (the reference's lazy path passes ``causal`` to every
  block, Appendix B #5) and dq keeps the input dtype (the reference hard-codes bf16);
* on the GPU every ring step is ONE kernel launch: the flash forward kernel merges its block into the running
  (fp32 out, lse) pair in its epilogue (``tb_flash_attn_block_fwd``; the reference runs ~8 elementwise kernels per
  step for the merge, utils.py:302-343), half-blocks of the zigzag layout are addressed in place (``BlockView``: no
  ``.contiguous()`` copies), the backward runs delta / dQ-zero once, one main kernel per step that reduce-adds dQ into
  one fp32 accumulator and writes dK/dV straight into the owner's slot, and one cast at the end;
* variable-length K (``k_lens``) runs on the same kernels through ``cu_seqlens`` (valid keys packed first); nothing
  materialises an [S, S] score matrix.  With ``causal=True`` valid queries never see a padded key (keys at or before a
  valid query are valid), so ``k_lens`` only matters for non-causal attention.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

from ... import _native as nat
from .. import attention as A
from .comm import _all_gather_dim, _coll, _rank, _world


# ---- block primitives -----------------------------------------------------------------------------------------
def _block_fwd(q, k, v, scale, causal, window, k_lens=None):
    """(out [B,Sq,H,D] in q.dtype, lse [B,H,Sq] fp32)."""
    if k_lens is not None:
        mask_k = (torch.arange(k.shape[1], device=q.device)[None] < k_lens[:, None])
        return _masked_block(q, k, v, scale, mask_k)
    out, lse, _ = A.flash_attn_func(q, k, v, softmax_scale=scale, causal=causal, window_size=window,
                                    return_attn_probs=True)
    return out, lse


def _masked_block(q, k, v, scale, mask_k):
    """Non-causal block with per-batch key validity (varlen K, reference ring_attn.py:486-491)."""
    B, Sq, Hq, D = q.shape
    g = Hq // k.shape[2]
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().permute(0, 2, 1, 3).repeat_interleave(g, 1)
    vf = v.float().permute(0, 2, 1, 3).repeat_interleave(g, 1)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    s = s.masked_fill(~mask_k[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.nan_to_num(torch.exp(s - lse.unsqueeze(-1)))
    return torch.matmul(p, vf).permute(0, 2, 1, 3).to(q.dtype), lse


def _block_bwd(do, q, k, v, out, lse, scale, causal, window, mask_k=None):
    """Gradients of one block given the GLOBAL (out, lse).  Returns (dq, dk, dv) in fp32."""
    B, Sq, Hq, D = q.shape
    Sk, Hk = k.shape[1], k.shape[2]
    if mask_k is None and A.native_supported(q, k, v, 0.0, None) and A.get_attention_backend() in ("auto", "native"):
        q3, k3, v3 = q.reshape(B * Sq, Hq, D), k.reshape(B * Sk, Hk, D), v.reshape(B * Sk, Hk, D)
        dq, dk, dv = torch.empty_like(q3), torch.empty_like(k3), torch.empty_like(v3)
        lse_t = lse.permute(1, 0, 2).reshape(Hq, B * Sq).contiguous()
        A._native_bwd(do.reshape(B * Sq, Hq, D).contiguous(), q3, k3, v3, out.reshape(B * Sq, Hq, D).contiguous(), lse_t,
                      None, None, B, Sq, Sk, scale, causal, window, dq, dk, dv)
        return dq.view_as(q).float(), dk.view_as(k).float(), dv.view_as(v).float()
    g = Hq // Hk
    qf, dof, of = (t.float().permute(0, 2, 1, 3) for t in (q, do, out))
    kf = k.float().permute(0, 2, 1, 3).repeat_interleave(g, 1)
    vf = v.float().permute(0, 2, 1, 3).repeat_interleave(g, 1)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    m = A._mask_for(Sq, Sk, causal, window, q.device)
    if m is not None:
        s = s.masked_fill(m, float("-inf"))
    if mask_k is not None:
        s = s.masked_fill(~mask_k[:, None, None, :], float("-inf"))
    p = torch.exp(s - lse.unsqueeze(-1))
    p = torch.nan_to_num(p, nan=0.0, posinf=0.0)
    dv = torch.matmul(p.transpose(-1, -2), dof)
    dp = torch.matmul(dof, vf.transpose(-1, -2))
    delta = (dof * of).sum(-1, keepdim=True)
    ds = p * (dp - delta) * scale
    dq = torch.matmul(ds, kf)
    dk = torch.matmul(ds.transpose(-1, -2), qf)
    dk = dk.view(B, Hk, g, Sk, D).sum(2)
    dv = dv.view(B, Hk, g, Sk, D).sum(2)
    return dq.permute(0, 2, 1, 3), dk.permute(0, 2, 1, 3), dv.permute(0, 2, 1, 3)


def merge_out_lse(out, lse, blk_out, blk_lse):
    """Numerically stable merge of two partial softmax results (reference utils.py:302-343); all fp32.
    out: [B,S,H,D], lse: [B,H,S]."""
    if out is None:
        return blk_out.float(), blk_lse
    new_lse = torch.logaddexp(lse, blk_lse)
    w_old = torch.exp(lse - new_lse).transpose(1, 2).unsqueeze(-1)
    w_new = torch.exp(blk_lse - new_lse).transpose(1, 2).unsqueeze(-1)
    w_old, w_new = torch.nan_to_num(w_old), torch.nan_to_num(w_new)
    return out * w_old + blk_out.float() * w_new, new_lse


# ---- native blockwise kernels (csrc/attn: BlockView addressing, in-kernel merge, phased backward) --------------
nat.register_signatures({
    "tb_flash_attn_block_fwd": ([nat.u64] * 7 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32, nat.i32, nat.i32, nat.i32,
                                nat.i64, nat.i64, nat.u64, nat.i32, nat.i32, nat.i32, nat.i32, nat.i32, nat.u64,
                                nat.i32], nat.i32),
    "tb_flash_attn_block_bwd": ([nat.u64] * 13 + [nat.i32] * 6 + [nat.i64] * 4 + [nat.f32, nat.i32, nat.i32, nat.i32,
                                nat.i64, nat.i64, nat.i64, nat.i64, nat.i64, nat.i32, nat.u64, nat.i32, nat.i32,
                                nat.i32, nat.i32, nat.i32, nat.i32], nat.i32),
})


def native_blockwise_ok(q, k, v) -> bool:
    L = nat.lib()
    return (L is not None and hasattr(L, "tb_flash_attn_block_fwd") and A.native_supported(q, k, v, 0.0, None)
            and A.get_attention_backend() in ("auto", "native") and q.shape[-1] in (64, 128))


def _blk_fwd(q3, k3, v3, o3, lse, acc, first, B, Sq, Sk, scale, causal, window=(-1, -1), view=(0, 0, 0, 0),
             cu_k=None):
    """One ring step: attention of the addressed q rows against the addressed keys, merged into (acc, lse, o3)."""
    Tq, Hq, D = q3.shape
    Tk, Hk = k3.shape[0], k3.shape[1]
    L = nat.require()
    nat.check(
        L.tb_flash_attn_block_fwd(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o3.data_ptr(), lse.data_ptr(), 0,
                                  nat.ptr(cu_k), B, Sq, Sk, Hq, Hk, D, q3.stride(0), k3.stride(0), v3.stride(0),
                                  o3.stride(0), scale, int(causal), window[0], window[1], Tq, Tk, nat.stream(),
                                  int(q3.dtype == torch.bfloat16), view[0], view[1], view[2], view[3], acc.data_ptr(),
                                  int(first)), "tb_flash_attn_block_fwd")
    nat.count_launch()


def _blk_bwd(do3, q3, k3, v3, o3, lse, dq3, dk3, dv3, dq_acc, delta, B, Sq, Sk, scale, causal, window, view, phases,
             cu_k=None):
    Tq, Hq, D = q3.shape
    Tk, Hk = k3.shape[0], k3.shape[1]
    L = nat.require()
    nat.check(
        L.tb_flash_attn_block_bwd(q3.data_ptr(), k3.data_ptr(), v3.data_ptr(), o3.data_ptr(), do3.data_ptr(),
                                  lse.data_ptr(), dq3.data_ptr(), dk3.data_ptr(), dv3.data_ptr(), dq_acc.data_ptr(),
                                  delta.data_ptr(), 0, nat.ptr(cu_k), B, Sq, Sk, Hq, Hk, D, q3.stride(0), k3.stride(0),
                                  v3.stride(0), do3.stride(0), scale, int(causal), window[0], window[1], Tq, Tk,
                                  dq3.stride(0), dk3.stride(0), dv3.stride(0), nat.num_sms(), nat.stream(),
                                  int(q3.dtype == torch.bfloat16), view[0], view[1], view[2], view[3], phases),
        "tb_flash_attn_block_bwd")
    nat.count_launch()


def _pack_valid_keys(kv, lens, S):
    """kv: [2, B*S, Hk, D]; lens: [B] valid keys per sequence (a prefix).  Returns (packed kv with the valid tokens
    first, int32 cu_seqlens [B+1], the permutation) -- no host sync."""
    B = lens.shape[0]
    invalid = (torch.arange(S, device=kv.device)[None] >= lens[:, None]).reshape(-1)
    order = torch.argsort(invalid, stable=True)
    cu = torch.zeros(B + 1, dtype=torch.int32, device=kv.device)
    cu[1:] = torch.cumsum(lens, 0)
    return kv[:, order].contiguous(), cu, order


def ring_forward_native(q, blocks, steps, scale, window=(-1, -1), k_lens=None):
    """q: [B, S, Hq, D]; blocks[j]: [2, B, S, Hk, D] (K and V of owner j); steps: output of ``_plan``.
    Returns (out [B, S, Hq, D] in q.dtype, lse [Hq, B*S] fp32).  One kernel per step."""
    B, S, Hq, D = q.shape
    T, half = B * S, S // 2
    q3 = q.view(T, Hq, D)
    out = torch.empty_like(q)
    o3 = out.view(T, Hq, D)
    acc = torch.empty((T, Hq, D), dtype=torch.float32, device=q.device)
    lse = torch.empty((Hq, T), dtype=torch.float32, device=q.device)
    for i, (j, mode) in enumerate(steps):
        kv = blocks[j].reshape(2, T, -1, D)
        k3, v3 = kv[0], kv[1]
        if mode == "diag":
            _blk_fwd(q3, k3, v3, o3, lse, acc, i == 0, B, S, S, scale, True, window)
        elif mode == "full":
            if k_lens is not None:
                lens = (k_lens.to(q.device) - j * S).clamp(0, S)
                pk, cu, _ = _pack_valid_keys(kv, lens, S)
                _blk_fwd(q3, pk[0], pk[1], o3, lse, acc, i == 0, B, S, S, scale, False, cu_k=cu)
            else:
                _blk_fwd(q3, k3, v3, o3, lse, acc, i == 0, B, S, S, scale, False)
        elif mode == "kv_first_half":
            _blk_fwd(q3, k3, v3, o3, lse, acc, i == 0, B, S, half, scale, False, view=(0, 0, S, 0))
        else:  # q_second_half
            _blk_fwd(q3, k3, v3, o3, lse, acc, i == 0, B, half, S, scale, False, view=(S, half, 0, 0))
    return out, lse


def ring_backward_native(do, q, out, lse, blocks, steps, scale, window=(-1, -1), k_lens=None):
    """Returns (dq [B, S, Hq, D] in q.dtype, dkv [cp, 2, B, S, Hk, D] in q.dtype: this rank's contribution to every
    owner's dK/dV, zero where nothing was visited)."""
    B, S, Hq, D = q.shape
    T, half = B * S, S // 2
    cp = len(blocks)
    Hk = blocks[0].shape[3]
    q3, o3 = q.view(T, Hq, D), out.view(T, Hq, D)
    do3 = do.contiguous().view(T, Hq, D)
    dq = torch.empty_like(q)
    dq3 = dq.view(T, Hq, D)
    dq_acc = torch.empty((T, Hq, D), dtype=torch.float32, device=q.device)
    delta = torch.empty((Hq, T), dtype=torch.float32, device=q.device)
    dkv = torch.zeros((cp, 2, T, Hk, D), dtype=q.dtype, device=q.device)
    kv0 = blocks[0].reshape(2, T, Hk, D)
    none = (0, 0, 0, 0)
    _blk_bwd(do3, q3, kv0[0], kv0[1], o3, lse, dq3, dkv[0, 0], dkv[0, 1], dq_acc, delta, B, S, S, scale, False,
             (-1, -1), none, 1)                                         # delta = rowsum(dO o O), dq_acc = 0
    for j, mode in steps:
        kv = blocks[j].reshape(2, T, Hk, D)
        k3, v3 = kv[0], kv[1]
        if mode == "diag":
            _blk_bwd(do3, q3, k3, v3, o3, lse, dq3, dkv[j, 0], dkv[j, 1], dq_acc, delta, B, S, S, scale, True, window,
                     none, 2)
        elif mode == "full":
            if k_lens is not None:
                lens = (k_lens.to(q.device) - j * S).clamp(0, S)
                pk, cu, order = _pack_valid_keys(kv, lens, S)
                dpk = torch.zeros_like(pk)
                _blk_bwd(do3, q3, pk[0], pk[1], o3, lse, dq3, dpk[0], dpk[1], dq_acc, delta, B, S, S, scale, False,
                         (-1, -1), none, 2, cu_k=cu)
                dkv[j].index_copy_(1, order, dpk)
            else:
                _blk_bwd(do3, q3, k3, v3, o3, lse, dq3, dkv[j, 0], dkv[j, 1], dq_acc, delta, B, S, S, scale, False,
                         (-1, -1), none, 2)
        elif mode == "kv_first_half":
            _blk_bwd(do3, q3, k3, v3, o3, lse, dq3, dkv[j, 0], dkv[j, 1], dq_acc, delta, B, S, half, scale, False,
                     (-1, -1), (0, 0, S, 0), 2)
        else:
            _blk_bwd(do3, q3, k3, v3, o3, lse, dq3, dkv[j, 0], dkv[j, 1], dq_acc, delta, B, half, S, scale, False,
                     (-1, -1), (S, half, 0, 0), 2)
    _blk_bwd(do3, q3, kv0[0], kv0[1], o3, lse, dq3, dkv[0, 0], dkv[0, 1], dq_acc, delta, B, S, S, scale, False,
             (-1, -1), none, 4)                                         # dq = cast(dq_acc)
    return dq, dkv.view(cp, 2, B, S, Hk, D)


# ---- schedule -------------------------------------------------------------------------------------------------
def _plan(rank: int, cp: int, causal: bool, zigzag: bool) -> List[Tuple[int, str]]:
    """Which K/V owner is visited and how: 'diag' (causal on the local block), 'full', 'kv_first_half',
    'q_second_half'."""
    steps = []
    for s in range(cp):
        j = (rank - s) % cp
        if not causal:
            steps.append((j, "full"))
        elif s == 0:
            steps.append((j, "diag"))
        elif zigzag:
            steps.append((j, "kv_first_half" if j < rank else "q_second_half"))
        elif j < rank:
            steps.append((j, "full"))
    return steps


class _RingAttnFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, q, k, v, scale, causal, window, group, zigzag, impl, k_lens):
        cp, rank = _world(group), _rank(group)
        B, S, Hq, D = q.shape
        zig = bool(zigzag and causal and cp > 1)
        if zig and S % 2:
            raise ValueError("zigzag ring attention needs an even local sequence length")
        if window != (-1, -1) and cp > 1:
            raise NotImplementedError("sliding-window masks are not supported across ring blocks")
        # fetch every rank's K/V block: one peer-memory all-gather (impl='allgather') or the classic ring
        if cp > 1:
            kv = torch.stack([k, v], 0).contiguous()                       # [2, B, S, Hk, D]
            if impl == "p2p":
                blocks = _LazyRing(kv, group)
            else:
                allkv = _all_gather_dim(kv.unsqueeze(0), 0, group)         # [cp, 2, B, S, Hk, D]
                blocks = [allkv[j] for j in range(cp)]
        else:
            blocks = [torch.stack([k, v], 0)]
        steps = _plan(rank, cp, causal, zig)
        ctx.native = native_blockwise_ok(q, k, v)
        if ctx.native:
            # valid queries of a causal mask never see padded keys: k_lens only matters for non-causal attention
            lens = None if causal else k_lens
            out_lp, lse_t = ring_forward_native(q, blocks, steps, scale, window, lens)
            if isinstance(blocks, _LazyRing):
                blocks = blocks.all()
            ctx.save_for_backward(q, out_lp, lse_t, *blocks)
            ctx.cfg = (scale, causal, window, group, zig, cp, rank, lens)
            return out_lp
        out, lse = None, None
        half = S // 2
        for j, mode in steps:
            kj, vj = blocks[j][0], blocks[j][1]
            lens_j = None
            if k_lens is not None:
                lens_j = (k_lens - j * S).clamp(0, S)
            if mode == "diag":
                o, l = _block_fwd(q, kj, vj, scale, True, window) if lens_j is None else \
                    _masked_diag(q, kj, vj, scale, lens_j)
                out, lse = merge_out_lse(out, lse, o, l)
            elif mode == "full":
                o, l = _block_fwd(q, kj, vj, scale, False, (-1, -1), lens_j)
                out, lse = merge_out_lse(out, lse, o, l)
            elif mode == "kv_first_half":
                o, l = _block_fwd(q, kj[:, :half].contiguous(), vj[:, :half].contiguous(), scale, False, (-1, -1))
                out, lse = merge_out_lse(out, lse, o, l)
            else:  # q_second_half
                o, l = _block_fwd(q[:, half:].contiguous(), kj, vj, scale, False, (-1, -1))
                o2, l2 = merge_out_lse(out[:, half:], lse[:, :, half:], o, l)
                out = torch.cat([out[:, :half], o2], 1)
                lse = torch.cat([lse[:, :, :half], l2], 2)
        out_lp = out.to(q.dtype)
        if isinstance(blocks, _LazyRing):
            blocks = blocks.all()
        ctx.save_for_backward(q, out_lp, lse, *blocks)
        ctx.cfg = (scale, causal, window, group, zig, cp, rank, k_lens)
        return out_lp

    @staticmethod
    def backward(ctx, do):
        q, out, lse, *blocks = ctx.saved_tensors
        scale, causal, window, group, zig, cp, rank, k_lens = ctx.cfg
        B, S, Hq, D = q.shape
        half = S // 2
        do = do.contiguous()
        if ctx.native:
            dq, dkv = ring_backward_native(do, q, out, lse, blocks, _plan(rank, cp, causal, zig), scale, window, k_lens)
            if cp > 1:
                mine = torch.empty(dkv.shape[1:], dtype=dkv.dtype, device=dkv.device)
                _coll(group, q.device).reduce_scatter(dkv.reshape(-1), mine.reshape(-1))   # fp32 accumulation inside
            else:
                mine = dkv[0]
            return dq, mine[0], mine[1], None, None, None, None, None, None, None
        dq = torch.zeros(q.shape, dtype=torch.float32, device=q.device)
        Hk = blocks[0].shape[3]
        dkv = torch.zeros((cp, 2, B, S, Hk, D), dtype=torch.float32, device=q.device)
        for j, mode in _plan(rank, cp, causal, zig):
            kj, vj = blocks[j][0], blocks[j][1]
            mask_k = None
            if k_lens is not None:
                lens_j = (k_lens - j * S).clamp(0, S)
                mask_k = torch.arange(S, device=q.device)[None] < lens_j[:, None]
            if mode in ("diag", "full"):
                a, bk, bv = _block_bwd(do, q, kj, vj, out, lse, scale, mode == "diag", window if mode == "diag" else (-1, -1), mask_k)
                dq += a
                dkv[j, 0] += bk
                dkv[j, 1] += bv
            elif mode == "kv_first_half":
                a, bk, bv = _block_bwd(do, q, kj[:, :half].contiguous(), vj[:, :half].contiguous(), out, lse, scale,
                                       False, (-1, -1))
                dq += a
                dkv[j, 0, :, :half] += bk
                dkv[j, 1, :, :half] += bv
            else:
                a, bk, bv = _block_bwd(do[:, half:].contiguous(), q[:, half:].contiguous(), kj, vj,
                                       out[:, half:].contiguous(), lse[:, :, half:].contiguous(), scale, False, (-1, -1))
                dq[:, half:] += a
                dkv[j, 0] += bk
                dkv[j, 1] += bv
        if cp > 1:
            mine = torch.empty((2, B, S, Hk, D), dtype=torch.float32, device=q.device)
            _coll(group, q.device).reduce_scatter(dkv.reshape(-1), mine.reshape(-1))
        else:
            mine = dkv[0]
        return dq.to(q.dtype), mine[0].to(q.dtype), mine[1].to(q.dtype), None, None, None, None, None, None, None


def _masked_diag(q, k, v, scale, lens):
    S = q.shape[1]
    causal = torch.ones(S, S, dtype=torch.bool, device=q.device).tril()
    mask_k = torch.arange(S, device=q.device)[None] < lens[:, None]
    B, Sq, Hq, D = q.shape
    g = Hq // k.shape[2]
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().permute(0, 2, 1, 3).repeat_interleave(g, 1)
    vf = v.float().permute(0, 2, 1, 3).repeat_interleave(g, 1)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    s = s.masked_fill(~(causal[None, None] & mask_k[:, None, None, :]), float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.nan_to_num(torch.exp(s - lse.unsqueeze(-1)))
    return torch.matmul(p, vf).permute(0, 2, 1, 3).to(q.dtype), lse


class _LazyRing:
    """Classic ring exchange with the NEXT transfer always in flight: block ``(rank - s) % cp`` arrives in round ``s``, and
    as soon as the consumer asks for it the block is forwarded to the next rank, so that transfer overlaps the consumer's
    attention on the block (the reference overlaps the same way with its RingComm, context_parallel/utils.py:398-415)."""

    def __init__(self, kv: torch.Tensor, group):
        self.group = group
        self.cp, self.rank = _world(group), _rank(group)
        self.blocks: List[Optional[torch.Tensor]] = [None] * self.cp
        self.blocks[self.rank] = kv
        self.send_to = dist.get_global_rank(group, (self.rank + 1) % self.cp)
        self.recv_from = dist.get_global_rank(group, (self.rank - 1) % self.cp)
        self.cur, self.round, self.pending = kv, 0, None
        self._post()

    def _post(self) -> None:
        if self.round + 1 >= self.cp:
            self.pending = None
            return
        nxt = torch.empty_like(self.cur)
        ops = [dist.P2POp(dist.isend, self.cur, self.send_to, self.group),
               dist.P2POp(dist.irecv, nxt, self.recv_from, self.group)]
        if self.rank % 2:
            ops.reverse()
        self.pending = (dist.batch_isend_irecv(ops), nxt)

    def _advance(self) -> None:
        works, nxt = self.pending
        for w in works:
            w.wait()
        self.round += 1
        self.blocks[(self.rank - self.round) % self.cp] = nxt
        self.cur = nxt
        self._post()

    def __getitem__(self, j: int) -> torch.Tensor:
        while self.blocks[j] is None:
            self._advance()
        return self.blocks[j]

    def all(self) -> List[torch.Tensor]:
        """Finish the ring (blocks the plan skipped still have to travel on) and return every block by owner."""
        while self.round + 1 < self.cp:
            self._advance()
        return self.blocks


def zigzag_split(x: torch.Tensor, seq_dim: int, group) -> torch.Tensor:
    """Take this rank's zigzag shard (chunks r and 2cp-1-r) of a full sequence."""
    cp, r = _world(group), _rank(group)
    if cp == 1:
        return x
    chunks = x.chunk(2 * cp, dim=seq_dim)
    return torch.cat([chunks[r], chunks[2 * cp - 1 - r]], dim=seq_dim).contiguous()


def zigzag_positions(seq_len_local: int, group, device) -> torch.Tensor:
    cp, r = _world(group), _rank(group)
    half = seq_len_local // 2
    a = torch.arange(half, device=device)
    return torch.cat([r * half + a, (2 * cp - 1 - r) * half + a])


def ring_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q_lens: Optional[torch.Tensor] = None,
                   k_lens: Optional[torch.Tensor] = None, dropout_p: float = 0.0, softmax_scale: Optional[float] = None,
                   causal: bool = False, window_size: tuple = (-1, -1), alibi_slopes: Optional[tuple] = None,
                   deterministic: bool = False, process_group: Optional[dist.ProcessGroup] = None,
                   zigzag: bool = False, impl: str = "allgather"):
    """q: [B, S/cp, Hq, D]; k, v: [B, S/cp, Hk, D] sequence shards (contiguous chunks, or zigzag shards when
    ``zigzag=True`` -- see ``zigzag_split``).  ``k_lens`` are GLOBAL key lengths per batch entry (varlen K, contiguous
    layout only); Q must be full length (same restrictions as the reference, ring_attn.py:475-491)."""
    if q_lens is not None:
        raise NotImplementedError("ring attention supports variable-length K only (q must be full length)")
    if alibi_slopes is not None:
        raise NotImplementedError("ALiBi is not supported by ring attention (reference ring_attn.py:298)")
    if dropout_p != 0.0:
        raise NotImplementedError("dropout is not supported by ring attention")
    if k_lens is not None and zigzag:
        raise NotImplementedError("variable-length K needs the contiguous (non-zigzag) layout")
    if deterministic:
        A._warn_once("ring-deterministic", "ring attention reduces dQ with atomics across its blocks: "
                     "deterministic=True is not honoured by ring attention (its gradients may differ in the last bits "
                     "from run to run)")
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(q.shape[-1])
    return _RingAttnFn.apply(q.contiguous(), k.contiguous(), v.contiguous(), scale, causal, tuple(window_size),
                             process_group, zigzag, impl, k_lens)
