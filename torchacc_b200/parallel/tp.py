"""Tensor parallelism (Megatron-style) with sequence-parallel residual stream.

The reference has NO tensor-parallel implementation of its own: ``torchacc/dist/tp.py:1-5`` only aliases
``xs.Mesh`` / ``xs.mark_sharding`` and leaves everything to XLA's SPMD partitioner; in its eager backend
``tp.size > 1`` has no effect on the model (SURVEY 2.1 #17, Appendix B #2).  This module is the from-scratch design:

* **column-parallel linear** (QKV, gate|up, lm_head): weight rows split over the tp group.  With sequence
  parallelism the input arrives token-sharded ``[T/tp, K]`` and is all-gathered right before the GEMM
  (all-gather -> GEMM); backward = dgrad GEMM -> reduce-scatter, wgrad on the re-gathered input.
* **row-parallel linear** (o_proj, down_proj): weight columns split; the GEMM produces partial sums for all tokens
  which are reduce-scattered back to token shards (GEMM -> reduce-scatter); backward = all-gather -> GEMMs.
* norms / residual adds / embedding run on token shards; parameters that stay replicated get their gradients
  summed over the group by ``tp_replicated``.
* the loss uses a vocab-parallel cross-entropy (two tiny all-reduces over [T] statistics, no logits gather).

The collectives come from ``parallel.collectives`` (peer-memory kernels on NVSwitch, NCCL or gloo), so the same code
runs in the CPU test tier.  ``mark_sharding`` / ``Mesh`` are kept as API aliases of the reference names.
"""
from __future__ import annotations


import torch
import torch.distributed as dist
import torch.nn as nn

from ..ops.linear import gemm
from .collectives import Collectives, make_collectives
from .mesh import Mesh  # noqa: F401  (reference: tp.Mesh alias)


class TPContext:
    """Everything the TP layers need: group, size, rank, collectives, sequence-parallel flag."""

    def __init__(self, group, device, sequence_parallel: bool = True, prefer_symm: bool = True):
        self.group = group
        self.size = dist.get_world_size(group) if group is not None else 1
        self.rank = dist.get_rank(group) if group is not None else 0
        self.sequence_parallel = sequence_parallel and self.size > 1
        self.coll: Collectives = make_collectives(group, device, prefer_symm)
        # fused all-gather->GEMM / GEMM->reduce-scatter kernels over peer memory (None on CPU / multi-node groups)
        self.fused = None
        if prefer_symm and self.size > 1:
            try:
                from .fused_tp import make_fused_tp
                self.fused = make_fused_tp(group, device)
            except Exception as e:  # pragma: no cover - depends on the box
                from ..utils.logger import logger
                logger.warning("fused TP kernels unavailable (%s); using separate collectives", e)


def _mm(a, b, **kw):
    """GEMM that works on CPU tensors too (gemm() falls back to fp32 matmul there)."""
    return gemm(a, b, **kw)


def _all_gather_rows(x: torch.Tensor, ctx: TPContext) -> torch.Tensor:
    full = torch.empty((x.shape[0] * ctx.size, *x.shape[1:]), dtype=x.dtype, device=x.device)
    ctx.coll.all_gather(x.contiguous().reshape(-1), full.reshape(-1))
    return full


def _reduce_scatter_rows(x: torch.Tensor, ctx: TPContext) -> torch.Tensor:
    assert x.shape[0] % ctx.size == 0, "token count must be divisible by the tp size"
    out = torch.empty((x.shape[0] // ctx.size, *x.shape[1:]), dtype=x.dtype, device=x.device)
    ctx.coll.reduce_scatter(x.contiguous().reshape(-1), out.reshape(-1))
    return out


def _wgrad(dy2, x2, w):
    view = getattr(w, "_tb_grad_view", None)
    if view is not None:
        _mm(dy2, x2, a_mn_major=True, b_mn_major=True, out=view, accumulate=bool(getattr(w, "_tb_grad_ready", False)))
        w._tb_grad_ready = True
        return None
    return _mm(dy2, x2, a_mn_major=True, b_mn_major=True, out_dtype=w.dtype)


class _ColumnParallel(torch.autograd.Function):
    """y_local = gather(x) @ W_local^T (+ b_local)."""

    @staticmethod
    def forward(ctx, x, w, bias, tp: TPContext):
        x2 = x.reshape(-1, x.shape[-1])
        f = tp.fused
        if tp.sequence_parallel and f is not None and x2.is_cuda and f.ok_ag(x2.shape[0], w.shape[0], x2.shape[1], x2.dtype):
            y, _ = f.ag_gemm(x2.contiguous(), w, bias)          # ONE kernel: peer pull of the token shards + wgmma GEMM
        else:
            xf = _all_gather_rows(x2, tp) if tp.sequence_parallel else x2
            y = _mm(xf, w, bias=bias, out_dtype=x.dtype)
        ctx.save_for_backward(x2, w)
        ctx.w_obj = w            # parameter object carrying the engine's _tb_grad_view (see ops/linear.py)
        ctx.tp, ctx.has_bias = tp, bias is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        tp: TPContext = ctx.tp
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        xf = _all_gather_rows(x2, tp) if tp.sequence_parallel else x2       # re-gather instead of saving [T, K]
        f = tp.fused
        if tp.sequence_parallel and f is not None and dy2.is_cuda and \
                f.ok_rs(dy2.shape[0] // tp.size, w.shape[1], w.shape[0], dy2.dtype):
            dx = f.gemm_rs(dy2, w, b_mn_major=True)                          # dgrad GEMM -> reduce-scatter, fused
        else:
            dx = _mm(dy2, w, b_mn_major=True, out_dtype=dy2.dtype)           # partial over the tp group
            if tp.sequence_parallel:
                dx = _reduce_scatter_rows(dx, tp)
            else:
                tp.coll.all_reduce(dx)
        dw = _wgrad(dy2, xf, ctx.w_obj) if ctx.needs_input_grad[1] else None
        db = dy2.float().sum(0).to(dy2.dtype) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return dx, dw, db, None


class _RowParallel(torch.autograd.Function):
    """y = scatter(sum_r x_local @ W_local^T)."""

    @staticmethod
    def forward(ctx, x, w, tp: TPContext):
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        f = tp.fused
        if tp.sequence_parallel and f is not None and x2.is_cuda and \
                f.ok_rs(x2.shape[0] // tp.size, w.shape[0], x2.shape[1], x2.dtype):
            y = f.gemm_rs(x2, w)                                              # GEMM -> reduce-scatter, fused
        else:
            y = _mm(x2, w, out_dtype=x.dtype)
            if tp.sequence_parallel:
                y = _reduce_scatter_rows(y, tp)
            else:
                tp.coll.all_reduce(y)
        ctx.save_for_backward(x2, w)
        ctx.w_obj = w
        ctx.tp = tp
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        tp: TPContext = ctx.tp
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        f = tp.fused
        if tp.sequence_parallel and f is not None and dy2.is_cuda and \
                f.ok_ag(dy2.shape[0], w.shape[1], dy2.shape[1], dy2.dtype):
            dx, dyf = f.ag_gemm(dy2, w, b_mn_major=True)                      # all-gather(dy) -> dgrad GEMM, fused
        else:
            dyf = _all_gather_rows(dy2, tp) if tp.sequence_parallel else dy2
            dx = _mm(dyf, w, b_mn_major=True, out_dtype=dy2.dtype)
        dw = _wgrad(dyf, x2, ctx.w_obj) if ctx.needs_input_grad[1] else None
        return dx, dw, None


class _ReplicatedParam(torch.autograd.Function):
    """Identity forward; backward sums the gradient over the tp group (parameters that every rank holds in full but
    applies to a different token shard)."""

    @staticmethod
    def forward(ctx, p, tp: TPContext):
        ctx.tp = tp
        return p.view_as(p)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        ctx.tp.coll.all_reduce(g)
        return g, None


class _GatherTokens(torch.autograd.Function):
    """all-gather rows forward, reduce-scatter rows backward."""

    @staticmethod
    def forward(ctx, x, tp: TPContext):
        ctx.tp = tp
        return _all_gather_rows(x, tp)

    @staticmethod
    def backward(ctx, g):
        return _reduce_scatter_rows(g.contiguous(), ctx.tp), None


class _GatherTokensReplicatedGrad(torch.autograd.Function):
    """all-gather rows forward; backward keeps this rank's row block of an upstream gradient that is already COMPLETE
    and identical on every tp rank (a pipeline-stage boundary: each tp peer of the next stage returns the full
    gradient), where ``_GatherTokens``' reduce-scatter would count it tp times."""

    @staticmethod
    def forward(ctx, x, tp: TPContext):
        ctx.tp = tp
        return _all_gather_rows(x, tp)

    @staticmethod
    def backward(ctx, g):
        tp = ctx.tp
        n = g.shape[0] // tp.size
        return g[tp.rank * n:(tp.rank + 1) * n].contiguous(), None


class _ScatterTokens(torch.autograd.Function):
    """take this rank's row block forward, all-gather backward."""

    @staticmethod
    def forward(ctx, x, tp: TPContext):
        ctx.tp = tp
        n = x.shape[0] // tp.size
        return x[tp.rank * n:(tp.rank + 1) * n].contiguous()

    @staticmethod
    def backward(ctx, g):
        return _all_gather_rows(g.contiguous(), ctx.tp), None


def column_parallel_linear(x, w, bias, tp: TPContext):
    return _ColumnParallel.apply(x, w, bias, tp)


def row_parallel_linear(x, w, tp: TPContext):
    return _RowParallel.apply(x, w, tp)


def tp_replicated(p, tp: TPContext):
    return _ReplicatedParam.apply(p, tp) if (tp is not None and tp.sequence_parallel) else p


def tp_head_shared(p, tp: TPContext):
    """A parameter applied to every attention head (Qwen3's q / k norm weights): each rank holds it in full but only
    sees its own heads, so its gradient is summed over the group with or without sequence parallelism."""
    return _ReplicatedParam.apply(p, tp) if tp is not None else p


def gather_tokens(x, tp: TPContext):
    return _GatherTokens.apply(x, tp)


def gather_tokens_replicated_grad(x, tp: TPContext):
    return _GatherTokensReplicatedGrad.apply(x, tp)


def scatter_tokens(x, tp: TPContext):
    return _ScatterTokens.apply(x, tp)


# ------------------------------------------------------------------------------------------------------------
# vocab-parallel cross entropy
# ------------------------------------------------------------------------------------------------------------
class _VocabParallelCE(torch.autograd.Function):
    """Mean CE of ``hidden @ W_local^T`` where each rank owns ``V/tp`` rows of the lm_head.  Logits are computed in
    token chunks; per chunk two all-reduces move [chunk] fp32 statistics (max, then sum-exp and label logit)."""

    @staticmethod
    def forward(ctx, hidden, w_local, labels, tp: TPContext, ignore_index, chunk, n_valid_total=None):
        T, V_local = hidden.shape[0], w_local.shape[0]
        v0 = tp.rank * V_local
        lab = labels.reshape(-1)
        valid = lab != ignore_index
        n_valid = valid.sum().clamp(min=1).float() if n_valid_total is None else \
            torch.as_tensor(n_valid_total, dtype=torch.float32, device=hidden.device).reshape(())
        dh = torch.zeros_like(hidden)
        want_w = ctx.needs_input_grad[1]
        view = getattr(w_local, "_tb_grad_view", None)
        # The weight gradient is produced here for d(loss) = 1 and rescaled in backward (same contract as
        # ops.cross_entropy._FusedLinearCEFn): write straight into the engine's flat gradient slice only when that
        # slice holds nothing yet, otherwise keep a private buffer that backward adds with the incoming scale.
        direct = want_w and view is not None and not bool(getattr(w_local, "_tb_grad_ready", False))
        dw = (view if direct else torch.zeros_like(w_local)) if want_w else None
        first = True
        total = torch.zeros((), dtype=torch.float32, device=hidden.device)
        for s in range(0, T, chunk):
            e = min(T, s + chunk)
            logits = _mm(hidden[s:e], w_local, out_dtype=torch.float32) if not hidden.is_cuda else \
                _mm(hidden[s:e], w_local).float()
            m = logits.max(dim=-1).values
            dist.all_reduce(m, op=dist.ReduceOp.MAX, group=tp.group)
            ex = torch.exp(logits - m[:, None])
            stats = torch.stack([ex.sum(-1), torch.zeros_like(m)])
            l = lab[s:e]
            local = (l >= v0) & (l < v0 + V_local)
            idx = (l - v0).clamp(0, V_local - 1)
            stats[1] = torch.where(local, logits.gather(1, idx[:, None])[:, 0], torch.zeros_like(m))
            dist.all_reduce(stats, group=tp.group)
            lse = m + torch.log(stats[0])
            vmask = valid[s:e]
            total += torch.where(vmask, lse - stats[1], torch.zeros_like(lse)).sum()
            # gradient of the mean loss wrt local logits
            g = ex / stats[0][:, None]
            g[torch.arange(e - s, device=g.device)[local], idx[local]] -= 1.0
            g = (g * (vmask.float() / n_valid)[:, None]).to(hidden.dtype)
            dh[s:e] = _mm(g, w_local, b_mn_major=True, out_dtype=hidden.dtype)
            if want_w:
                _mm(g, hidden[s:e], a_mn_major=True, b_mn_major=True, out=dw, accumulate=not first)
                first = False
        if direct:
            w_local._tb_grad_ready = True
        # Each rank holds the part of dh that flows through ITS vocab slice.  With sequence parallelism the caller
        # gathered the tokens (gather_tokens) and that op's backward reduce-scatters these partials; without it the
        # hidden states are replicated and the full gradient is needed on every rank.
        if not tp.sequence_parallel:
            tp.coll.all_reduce(dh)
        ctx.save_for_backward(dh, dw if (want_w and not direct) else None)
        ctx.mode = "direct" if direct else ("view" if (want_w and view is not None) else ("own" if want_w else "none"))
        ctx.view = view if want_w else None
        ctx.weight = w_local if (want_w and view is not None) else None   # the parameter OBJECT (attributes survive)
        return total / n_valid

    @staticmethod
    def backward(ctx, dloss):
        dh, dw = ctx.saved_tensors
        out_dw = None
        if ctx.mode == "direct":
            ctx.view.mul_(dloss.to(ctx.view.dtype))
        elif ctx.mode == "view":
            ctx.view.add_(dw * dloss.to(dw.dtype))
            ctx.weight._tb_grad_ready = True
        elif ctx.mode == "own":
            out_dw = dw * dloss.to(dw.dtype)
        return (dh * dloss.to(dh.dtype), out_dw, None, None, None, None, None)


def vocab_parallel_cross_entropy(hidden, w_local, labels, tp: TPContext, ignore_index: int = -100,
                                 chunk_tokens: int = 2048, n_valid_total=None):
    return _VocabParallelCE.apply(hidden, w_local, labels, tp, ignore_index, chunk_tokens, n_valid_total)


# ------------------------------------------------------------------------------------------------------------
# sharding a native model
# ------------------------------------------------------------------------------------------------------------
def _shard_rows(w: torch.Tensor, rank: int, size: int) -> torch.Tensor:
    n = w.shape[0] // size
    return w[rank * n:(rank + 1) * n].clone()


def _shard_cols(w: torch.Tensor, rank: int, size: int) -> torch.Tensor:
    n = w.shape[1] // size
    return w[:, rank * n:(rank + 1) * n].clone()


@torch.no_grad()
def shard_llama_for_tp(lm, tp: TPContext) -> None:
    """Rewrite a native ``LlamaForCausalLM`` in place so each rank keeps 1/tp of the attention heads, the MLP width
    and the lm_head vocabulary."""
    cfg = lm.config
    if getattr(cfg, "num_experts", 0):
        raise NotImplementedError("tensor parallelism of mixture-of-experts layers is not supported; use FSDP")
    size, rank = tp.size, tp.rank
    hq, hk, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    if hq % size or hk % size:
        raise ValueError(f"tp size {size} must divide both head counts ({hq}, {hk})")
    if cfg.intermediate_size % size or cfg.vocab_size % size:
        raise ValueError("tp size must divide intermediate_size and vocab_size")

    def set_param(mod, name, value):
        old = getattr(mod, name)
        new = nn.Parameter(value.to(old.device), requires_grad=old.requires_grad)
        setattr(mod, name, new)

    for layer in lm.model.layers:
        att, mlp = layer.self_attn, layer.mlp
        w = att.qkv_proj.weight
        q, k, v = w.split([hq * d, hk * d, hk * d], 0)
        set_param(att.qkv_proj, "weight", torch.cat([_shard_rows(q, rank, size), _shard_rows(k, rank, size),
                                                     _shard_rows(v, rank, size)], 0))
        if att.qkv_proj.bias is not None:
            b = att.qkv_proj.bias
            bq, bk, bv = b.split([hq * d, hk * d, hk * d], 0)
            set_param(att.qkv_proj, "bias", torch.cat([_shard_rows(bq, rank, size), _shard_rows(bk, rank, size),
                                                       _shard_rows(bv, rank, size)], 0))
        set_param(att.o_proj, "weight", _shard_cols(att.o_proj.weight, rank, size))
        g, u = mlp.gate_up_proj.weight.chunk(2, 0)
        set_param(mlp.gate_up_proj, "weight", torch.cat([_shard_rows(g, rank, size), _shard_rows(u, rank, size)], 0))
        set_param(mlp.down_proj, "weight", _shard_cols(mlp.down_proj.weight, rank, size))
    if cfg.tie_word_embeddings:
        raise ValueError("tensor parallelism with tied embeddings is not supported (lm_head is vocab-parallel)")
    set_param(lm.lm_head, "weight", _shard_rows(lm.lm_head.weight, rank, size))
    lm.model.pctx.tp = tp
    lm.model.pctx.tp_group = tp.group
    lm.model.pctx.tp_size = size
    lm.model.pctx.sequence_parallel = tp.sequence_parallel


# ------------------------------------------------------------------------------------------------------------
# HuggingFace decoder models: Megatron-style sharding of the existing nn.Linear modules
# ------------------------------------------------------------------------------------------------------------
class ColumnParallelLinear(nn.Linear):
    """``nn.Linear`` holding the rows ``[rank * out/tp, (rank + 1) * out/tp)`` of the original weight; the input is
    replicated over the tp group, the output is this rank's slice of the features (heads)."""

    @classmethod
    def from_linear(cls, lin: nn.Linear, tp: TPContext) -> "ColumnParallelLinear":
        if lin.out_features % tp.size:
            raise ValueError(f"out_features {lin.out_features} not divisible by the tp size {tp.size}")
        rows = lin.out_features // tp.size
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.out_features = lin.in_features, rows
        new.weight = nn.Parameter(_shard_rows(lin.weight.detach(), tp.rank, tp.size).clone(),
                                  requires_grad=lin.weight.requires_grad)
        new.bias = None if lin.bias is None else nn.Parameter(
            _shard_rows(lin.bias.detach(), tp.rank, tp.size).clone(), requires_grad=lin.bias.requires_grad)
        new.__dict__["tp"] = tp
        return new

    def forward(self, x):
        y = column_parallel_linear(x.reshape(-1, x.shape[-1]), self.weight, self.bias, self.tp)
        return y.view(*x.shape[:-1], self.out_features)


class RowParallelLinear(nn.Linear):
    """``nn.Linear`` holding the columns ``[rank * in/tp, ...)`` of the original weight: consumes the feature slice a
    column-parallel layer produced, the partial products are summed over the tp group (bias added once, after the sum)."""

    @classmethod
    def from_linear(cls, lin: nn.Linear, tp: TPContext) -> "RowParallelLinear":
        if lin.in_features % tp.size:
            raise ValueError(f"in_features {lin.in_features} not divisible by the tp size {tp.size}")
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.out_features = lin.in_features // tp.size, lin.out_features
        new.weight = nn.Parameter(_shard_cols(lin.weight.detach(), tp.rank, tp.size).clone(),
                                  requires_grad=lin.weight.requires_grad)
        new.bias = None if lin.bias is None else nn.Parameter(lin.bias.detach().clone(),
                                                             requires_grad=lin.bias.requires_grad)
        new.__dict__["tp"] = tp
        return new

    def forward(self, x):
        y = row_parallel_linear(x.reshape(-1, x.shape[-1]), self.weight, self.tp).view(*x.shape[:-1], self.out_features)
        return y if self.bias is None else y + self.bias


_HF_COLUMN = ("q_proj", "k_proj", "v_proj", "gate_proj", "up_proj")
_HF_ROW = ("o_proj", "down_proj")


def shard_hf_for_tp(model: nn.Module, tp: TPContext) -> int:
    """Tensor parallelism for HuggingFace decoder families that follow the Llama layout (Llama, Qwen2/3, Mistral, Gemma,
    ...): q/k/v and gate/up projections become column-parallel (whole heads / FFN columns per rank), o_proj and down_proj
    row-parallel; the residual stream, norms, embedding and lm_head stay replicated (their gradients are identical on
    every tp rank because their inputs are).  HF attention modules infer the local head count from the projection
    output (``view(..., -1, head_dim)``), so their forward is untouched.  Returns the number of layers rewritten.
    The reference leaves TP of HF models to XLA's SPMD partitioner (torchacc/dist/tp.py:1-5)."""
    cfg = getattr(model, "config", None)
    hk = getattr(cfg, "num_key_value_heads", None) or getattr(cfg, "num_attention_heads", None)
    hq = getattr(cfg, "num_attention_heads", None)
    for n, name in ((hq, "num_attention_heads"), (hk, "num_key_value_heads")):
        if n is not None and n % tp.size:
            raise ValueError(f"{name} = {n} is not divisible by the tp size {tp.size}")
    count = 0
    for mod in list(model.modules()):
        touched = False
        for name in _HF_COLUMN:
            lin = getattr(mod, name, None)
            if type(lin) is nn.Linear:
                setattr(mod, name, ColumnParallelLinear.from_linear(lin, tp))
                touched = True
        for name in _HF_ROW:
            lin = getattr(mod, name, None)
            if type(lin) is nn.Linear:
                setattr(mod, name, RowParallelLinear.from_linear(lin, tp))
                touched = True
        count += int(touched)
    if count == 0:
        raise NotImplementedError(
            f"{type(model).__name__}: no q_proj/k_proj/v_proj/o_proj or gate_proj/up_proj/down_proj linears found; tensor "
            "parallelism covers the native Llama family and HuggingFace models with the Llama module layout")
    return count


def parallelize_model(model: nn.Module, config, mesh) -> nn.Module:
    """Apply TP and/or context parallelism to a native model (called by DistributedParallel)."""
    from .bootstrap import current_device
    device = current_device()
    core = model
    if config.dist.tp.size > 1:
        if hasattr(model, "config") and hasattr(model, "model") and hasattr(model.model, "pctx"):
            tp = TPContext(mesh.get_tp_proc_group(), device, config.dist.tp.sequence_parallel,
                           config.dist.fsdp.fused_collectives)
            shard_llama_for_tp(model, tp)
        else:
            # HuggingFace layout: replicated residual stream (no sequence parallelism), see shard_hf_for_tp
            tp = TPContext(mesh.get_tp_proc_group(), device, False, config.dist.fsdp.fused_collectives)
            shard_hf_for_tp(model, tp)
    if config.dist.sp.size > 1:
        if hasattr(model, "model") and hasattr(model.model, "pctx"):
            model.model.pctx.cp_mesh = mesh
            model.model.pctx.cp_mode = config.dist.sp.mode
        else:
            from ..ops.context_parallel.hf_hook import HFContextParallel, is_hf_causal_lm
            if not is_hf_causal_lm(model):
                raise NotImplementedError(
                    "context parallelism is wired for the native model families and for HuggingFace causal LMs; call "
                    "torchacc_b200.ops.context_parallel.* directly from custom attention modules")
            core = HFContextParallel(model, mesh, config.dist.sp.mode)
    return core


def mark_sharding(tensor, mesh, partition_spec):
    """Reference API (``xs.mark_sharding``) relied on the XLA SPMD partitioner.  There is no partitioner here: use
    ``parallelize_model`` / the column- and row-parallel layers instead."""
    raise NotImplementedError("mark_sharding needs an SPMD partitioner; use torchacc_b200.parallel.tp.parallelize_model")
