"""Cross-entropy and fused linear + cross-entropy.

``fused_linear_cross_entropy(hidden, lm_head_weight, labels)`` never materialises the ``[T, V]`` logits for the
whole batch: tokens are processed in chunks; for each chunk the lm_head GEMM (wgmma) produces bf16 logits, the
CE kernel (csrc/ops/loss_optim.cu) computes the row losses and overwrites the logits with their gradient, and the
dgrad / wgrad GEMMs consume that gradient immediately (wgrad accumulates across chunks in the GEMM epilogue).
Same idea as liger's fused-linear-CE that the reference enables by default
(reference torchacc/ops/liger.py:32-82 ``fused_linear_cross_entropy=True``), built on our own kernels.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .. import _native as nat
from .linear import gemm


def _ce_native(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int, grad_scale, write_grad: bool):
    """logits [n, V] bf16 (row pitch multiple of 8); returns per-row loss fp32; logits become gradients."""
    n, V = logits.shape
    loss_rows = torch.empty(n, dtype=torch.float32, device=logits.device)
    L = nat.require()
    scale_ptr, scale_val = (grad_scale.data_ptr(), 0.0) if isinstance(grad_scale, torch.Tensor) else (0, float(grad_scale))
    nat.check(
        L.tb_cross_entropy(logits.data_ptr(), labels.data_ptr(), loss_rows.data_ptr(), 0, n, V, logits.stride(0),
                           ignore_index, scale_ptr, scale_val, int(write_grad), nat.stream()), "tb_cross_entropy")
    nat.count_launch()
    return loss_rows


class _CrossEntropyFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, logits, labels, ignore_index, reduction):
        n = labels.numel()
        lg = logits.reshape(n, logits.shape[-1])
        if not lg.is_contiguous():
            lg = lg.contiguous()
        else:
            lg = lg.clone()  # the kernel overwrites its input with the gradient
        lab = labels.reshape(-1).contiguous()
        n_valid = (lab != ignore_index).sum().clamp(min=1).float()
        scale = (1.0 / n_valid) if reduction == "mean" else torch.ones((), device=lg.device)
        scale = scale.reshape(1).contiguous()
        loss_rows = _ce_native(lg, lab, ignore_index, scale, True)
        ctx.save_for_backward(lg)
        ctx.shape = logits.shape
        return loss_rows.sum() * scale[0] if reduction == "mean" else loss_rows.sum()

    @staticmethod
    def backward(ctx, dloss):
        (g,) = ctx.saved_tensors
        return (g * dloss.to(g.dtype)).view(ctx.shape), None, None, None


def cross_entropy(logits: torch.Tensor, labels: torch.Tensor, ignore_index: int = -100,
                  reduction: str = "mean") -> torch.Tensor:
    if logits.dtype == torch.bfloat16 and nat.use_native(logits) and logits.shape[-1] % 8 == 0 \
            and reduction in ("mean", "sum"):
        return _CrossEntropyFn.apply(logits, labels, ignore_index, reduction)
    return F.cross_entropy(logits.float().reshape(-1, logits.shape[-1]), labels.reshape(-1),
                           ignore_index=ignore_index, reduction=reduction)


class _FusedLinearCEFn(torch.autograd.Function):

    @staticmethod
    def forward(ctx, hidden, weight, labels, ignore_index, chunk_tokens, n_valid_total, valid_vocab=None):
        H = hidden.shape[-1]
        h2 = hidden.reshape(-1, H)
        if not h2.is_contiguous():
            h2 = h2.contiguous()
        lab = labels.reshape(-1).contiguous()
        T = h2.shape[0]
        V = weight.shape[0]
        if n_valid_total is None:
            n_valid = (lab != ignore_index).sum().clamp(min=1).float().reshape(1)
        else:
            n_valid = n_valid_total.float().reshape(1)
        scale = (1.0 / n_valid).contiguous()
        want_grad = bool(ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        dh = torch.empty_like(h2) if want_grad else None
        need_w = weight.requires_grad and want_grad
        view = getattr(weight, "_tb_grad_view", None)
        # The weight gradient is produced HERE (forward) for d(loss) = 1; backward rescales it by the incoming
        # gradient.  Writing straight into the engine's flat gradient slice is only possible when that slice holds
        # nothing yet (otherwise our contribution could not be rescaled separately).
        direct = need_w and view is not None and not bool(getattr(weight, "_tb_grad_ready", False))
        if need_w:
            dw = view if direct else torch.zeros_like(weight)
            acc0 = not direct
        else:
            dw, acc0 = None, False
        total = torch.zeros((), dtype=torch.float32, device=h2.device)
        logits = torch.empty((min(chunk_tokens, T), V), dtype=torch.bfloat16, device=h2.device)
        first = True
        for s in range(0, T, chunk_tokens):
            e = min(T, s + chunk_tokens)
            lg = logits[:e - s]
            gemm(h2[s:e], weight, out=lg)                                   # logits chunk
            if valid_vocab is not None and valid_vocab < V:
                lg[:, valid_vocab:] = -1.0e4     # padding rows of the embedding: probability (and gradient) exactly 0
            rows = _ce_native(lg, lab[s:e], ignore_index, scale, want_grad)  # lg <- dlogits (already / n_valid)
            total += rows.sum()
            if not want_grad:
                continue
            gemm(lg, weight, b_mn_major=True, out=dh[s:e])                  # dh = dlogits @ W
            if need_w:
                gemm(lg, h2[s:e], a_mn_major=True, b_mn_major=True, out=dw,
                     accumulate=(acc0 or not first))                        # dW += dlogits^T @ h
            first = False
        if direct:
            weight._tb_grad_ready = True
        ctx.save_for_backward(dh, dw if need_w else None)
        ctx.shape = hidden.shape
        ctx.mode = "direct" if direct else ("view" if (need_w and view is not None) else ("own" if need_w else "none"))
        ctx.view = view if need_w else None
        ctx.weight = weight if (need_w and view is not None) else None
        return total * scale[0]

    @staticmethod
    def backward(ctx, dloss):
        dh, dw = ctx.saved_tensors
        # gradients were computed for d(loss) = 1: apply the incoming scale (1/num_micro_batches, loss scaling ...)
        dh = dh * dloss.to(dh.dtype)
        out_dw = None
        if ctx.mode == "direct":
            ctx.view.mul_(dloss.to(ctx.view.dtype))
        elif ctx.mode == "view":
            ctx.view.add_(dw * dloss.to(dw.dtype))
            ctx.weight._tb_grad_ready = True
        elif ctx.mode == "own":
            out_dw = dw * dloss.to(dw.dtype)
        return dh.view(ctx.shape), out_dw, None, None, None, None, None


def fused_linear_cross_entropy(hidden: torch.Tensor, weight: torch.Tensor, labels: torch.Tensor,
                               ignore_index: int = -100, chunk_tokens: int = 4096,
                               n_valid_total: Optional[torch.Tensor] = None,
                               valid_vocab: Optional[int] = None) -> torch.Tensor:
    """Mean cross-entropy of ``hidden @ weight.T`` against ``labels`` without materialising all logits.
    ``n_valid_total`` overrides the normaliser (e.g. the global valid-token count under data parallelism);
    ``valid_vocab`` < ``weight.shape[0]`` excludes the trailing padding rows of a vocabulary that was padded for
    alignment (GPT-2: 50257 -> 50304) from the softmax."""
    if hidden.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and nat.use_native(hidden, weight) \
            and weight.shape[0] % 8 == 0:
        return _FusedLinearCEFn.apply(hidden, weight, labels, ignore_index, chunk_tokens, n_valid_total, valid_vocab)
    logits = F.linear(hidden, weight).float()
    if valid_vocab is not None and valid_vocab < logits.shape[-1]:
        logits = logits[..., :valid_vocab]
    loss = F.cross_entropy(logits.reshape(-1, logits.shape[-1]), labels.reshape(-1), ignore_index=ignore_index,
                           reduction="sum")
    if n_valid_total is None:
        n_valid_total = (labels != ignore_index).sum().clamp(min=1)
    return loss / n_valid_total.float()
