"""Fused optimizers on flat fp32 shards (csrc/ops/loss_optim.cu).

``FusedAdamW`` is a regular ``torch.optim.Optimizer`` so user code written for the reference
(``torch.optim.AdamW(model.parameters())`` after ``accelerate``; tests/standalone/ta_accelerate.py:66-69) keeps
working -- but it updates every parameter (in practice: one flat fp32 shard per FSDP unit) with one kernel that
also applies the device-resident clip coefficient / inverse loss scale, honours ``found_inf`` without a host
sync, and writes the bf16 compute copy that the next all-gather ships (when the parameter exposes
``_tb_lp_shard``).  Replaces torch's fused/foreach Adam and torch_xla's syncfree optimizers
(reference utils/patch.py:55-58).
"""
from __future__ import annotations

from typing import Iterable, Optional

import torch

from .. import _native as nat

nat.register_signatures({
    "tb_sqnorm_accumulate_ordered": ([nat.u64, nat.i32, nat.i64, nat.u64, nat.f32, nat.u64, nat.u64, nat.i32, nat.u64],
                                     nat.i32),
})

_DETERMINISTIC = False
_ORDERED_WS = {}   # device -> (partials [8 * num_sms] fp32, ticket counter [1] int32)


def set_deterministic(flag: bool) -> None:
    """Process-wide switch: ``grad_sqnorm`` sums in a fixed order (bitwise reproducible gradient norms)."""
    global _DETERMINISTIC
    _DETERMINISTIC = bool(flag)


def deterministic_enabled() -> bool:
    """The process switch or PyTorch's ``torch.use_deterministic_algorithms``."""
    return _DETERMINISTIC or torch.are_deterministic_algorithms_enabled()


def _ordered_workspace(device: torch.device):
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    if key not in _ORDERED_WS:
        _ORDERED_WS[key] = (torch.empty(8 * nat.num_sms(), dtype=torch.float32, device=device),
                            torch.zeros(1, dtype=torch.int32, device=device))
    return _ORDERED_WS[key]


def _sqnorm(t: torch.Tensor, out: torch.Tensor, pre_scale: float = 1.0, ordered: bool = False):
    if nat.use_native(t) and t.dtype in (torch.bfloat16, torch.float32) and t.is_contiguous():
        L = nat.require()
        if ordered:
            partial, counter = _ordered_workspace(t.device)
            nat.check(
                L.tb_sqnorm_accumulate_ordered(t.data_ptr(), int(t.dtype == torch.bfloat16), t.numel(),
                                               out.data_ptr(), pre_scale, partial.data_ptr(), counter.data_ptr(),
                                               nat.num_sms(), nat.stream()), "tb_sqnorm_accumulate_ordered")
        else:
            nat.check(
                L.tb_sqnorm_accumulate(t.data_ptr(), int(t.dtype == torch.bfloat16), t.numel(), out.data_ptr(),
                                       pre_scale, nat.num_sms(), nat.stream()), "tb_sqnorm_accumulate")
        nat.count_launch()
    else:
        x = t.float() * pre_scale
        out[0] += (x * x).sum()
        if not torch.isfinite(x).all():
            out[1] = 1.0


def grad_sqnorm(grads: Iterable[torch.Tensor], device=None) -> torch.Tensor:
    """Returns a 2-element fp32 tensor ``[sum of squares, found_inf]`` accumulated over ``grads`` (no host sync).
    In deterministic mode (``set_deterministic`` / ``torch.use_deterministic_algorithms``) the sums are taken in a
    fixed order, so repeated calls on the same gradients are bitwise equal."""
    grads = [g for g in grads if g is not None]
    dev = device if device is not None else (grads[0].device if grads else torch.device("cpu"))
    out = torch.zeros(2, dtype=torch.float32, device=dev)
    ordered = deterministic_enabled()
    for g in grads:
        _sqnorm(g, out, ordered=ordered)
    return out


def scale_(t: torch.Tensor, scale: torch.Tensor):
    """``t *= scale`` with a device scalar (fp32, shape [1])."""
    if nat.use_native(t) and t.dtype in (torch.bfloat16, torch.float32) and t.is_contiguous():
        L = nat.require()
        nat.check(
            L.tb_scale_inplace(t.data_ptr(), int(t.dtype == torch.bfloat16), t.numel(), scale.data_ptr(),
                               nat.num_sms(), nat.stream()), "tb_scale_inplace")
        nat.count_launch()
    else:
        t.mul_(scale.to(t.dtype))


class FusedAdamW(torch.optim.Optimizer):
    """AdamW with decoupled weight decay; one fused kernel per parameter tensor.

    Extra (optional) state understood per step:
      * ``grad_scale``: fp32 device tensor [1] multiplied into every gradient (clip coefficient, 1/loss_scale);
      * ``found_inf``:  fp32 device tensor [1]; non-zero skips the update on the device.
    Parameters may carry ``_tb_lp_shard`` (bf16 tensor, same numel): the updated value is also written there.
    Gradients may be bf16 or fp32; master params and moments are fp32.
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.grad_scale: Optional[torch.Tensor] = None
        self.found_inf: Optional[torch.Tensor] = None
        # flat shards of a sharding engine: switch the engine to bf16/fp32 `_tb_grad` hand-off (no fp32 .grad copies)
        engines = set()
        for group in self.param_groups:
            for p in group["params"]:
                unit = getattr(p, "_tb_unit", None)
                if unit is not None and id(unit.engine) not in engines:
                    engines.add(id(unit.engine))
                    unit.engine.use_fused_optimizer(self)

    def zero_grad(self, set_to_none: bool = True):
        """Also drops the engine-side gradient hand-off (``_tb_grad``) of flat shards, so the reference's canonical
        ``optimizer.zero_grad()`` loop behaves exactly like ``model.zero_grad()``."""
        super().zero_grad(set_to_none)
        for group in self.param_groups:
            for p in group["params"]:
                if getattr(p, "_tb_grad", None) is not None:
                    p._tb_grad = None

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            b1, b2 = group["betas"]
            for p in group["params"]:
                g = getattr(p, "_tb_grad", None)
                if g is None:
                    g = p.grad
                if g is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, dtype=torch.float32, memory_format=torch.preserve_format)
                st["step"] += 1
                lp = getattr(p, "_tb_lp_shard", None)
                if (p.dtype == torch.float32 and nat.use_native(p, g) and p.is_contiguous() and g.is_contiguous()
                        and g.dtype in (torch.bfloat16, torch.float32)):
                    L = nat.require()
                    lp_native = lp if (lp is not None and lp.dtype == torch.bfloat16) else None   # kernel writes bf16
                    nat.check(
                        L.tb_adamw_flat(p.data_ptr(), g.data_ptr(), int(g.dtype == torch.bfloat16),
                                        st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), nat.ptr(lp_native),
                                        p.numel(),
                                        group["lr"], b1, b2, group["eps"], group["weight_decay"], st["step"],
                                        nat.ptr(self.grad_scale), nat.ptr(self.found_inf), nat.num_sms(),
                                        nat.stream()), "tb_adamw_flat")
                    nat.count_launch()
                    if lp is not None and lp_native is None:
                        lp.copy_(p.data.view_as(lp))           # fp16 compute copy: separate cast
                else:
                    self._reference_update(p, g, st, group, lp)
                unit = getattr(p, "_tb_unit", None)
                if unit is not None:
                    unit.mark_params_updated()       # gathered copies kept across the step are stale now
        return loss

    def _reference_update(self, p, g, st, group, lp):
        b1, b2 = group["betas"]
        if self.found_inf is not None and float(self.found_inf) != 0.0:
            return
        g = g.float()
        if self.grad_scale is not None:
            g = g * self.grad_scale.to(g.device)
        pf = p.data.float()
        pf.mul_(1 - group["lr"] * group["weight_decay"])
        st["exp_avg"].mul_(b1).add_(g.view_as(pf), alpha=1 - b1)
        st["exp_avg_sq"].mul_(b2).addcmul_(g.view_as(pf), g.view_as(pf), value=1 - b2)
        bc1 = 1 - b1 ** st["step"]
        bc2 = 1 - b2 ** st["step"]
        denom = (st["exp_avg_sq"].sqrt() / (bc2 ** 0.5)).add_(group["eps"])
        pf.addcdiv_(st["exp_avg"], denom, value=-group["lr"] / bc1)
        p.data.copy_(pf.to(p.dtype))
        if lp is not None:
            lp.copy_(pf.to(lp.dtype).view_as(lp))


AdamW = FusedAdamW
