"""Kernel patches for HuggingFace models (reference torchacc/ops/liger.py:10-153).

The reference swaps HF module forwards onto liger's Triton kernels.  Same entry points here
(``apply_liger_kernel``, ``apply_liger_kernel_to_llama``, ``apply_liger_kernel_to_qwen2``) but the replacements are
our sm_90a kernels: RMSNorm, SwiGLU, RoPE-free fused loss (linear + cross-entropy), and the wgmma GEMM behind
every ``nn.Linear`` of the model.  Patches are applied to *classes* (like liger) or to one model instance.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from ..utils.logger import logger
from .cross_entropy import fused_linear_cross_entropy
from .linear import linear
from .rmsnorm import rmsnorm
from .swiglu import swiglu_separate


def rms_forward(self, hidden_states):
    eps = getattr(self, "variance_epsilon", getattr(self, "eps", 1e-6))
    y, _ = rmsnorm(hidden_states, self.weight, eps)
    return y


def mlp_forward(self, x):
    if not all(type(m) is nn.Linear for m in (self.gate_proj, self.up_proj, self.down_proj)):
        # tensor-parallel (or otherwise specialised) projections bring their own forward: only the activation is ours
        return self.down_proj(swiglu_separate(self.gate_proj(x), self.up_proj(x)))
    g = linear(x, self.gate_proj.weight, self.gate_proj.bias)
    u = linear(x, self.up_proj.weight, self.up_proj.bias)
    return linear(swiglu_separate(g, u), self.down_proj.weight, self.down_proj.bias)


def hf_apply_rotary_pos_emb(q, k, cos, sin, position_ids=None, unsqueeze_dim=1):
    """Drop-in for HF ``apply_rotary_pos_emb`` (q/k: [B, H, S, D] views of the [B, S, H, D] projections, cos/sin:
    [B, S, D] with duplicated halves): one in-place rotate-half kernel per tensor instead of ~10 elementwise / cat
    launches per layer (reference liger.py:69-70 swaps in liger's Triton RoPE here)."""
    from .rope import _RopeOneFn
    ok = (q.is_cuda and q.dim() == 4 and cos.dim() == 3 and unsqueeze_dim == 1 and q.dtype in (torch.bfloat16, torch.float16)
          and q.shape[-1] % 16 == 0 and q.transpose(1, 2).is_contiguous() and k.transpose(1, 2).is_contiguous())
    if not ok:
        orig = _HF_ROPE_ORIG[0]
        import inspect
        if "position_ids" in inspect.signature(orig).parameters:       # transformers < 4.5x
            return orig(q, k, cos, sin, position_ids, unsqueeze_dim)
        return orig(q, k, cos, sin, unsqueeze_dim=unsqueeze_dim)
    B, H, S, D = q.shape
    half = D // 2
    cos_t = cos[..., :half].float().reshape(-1, half).contiguous()
    sin_t = sin[..., :half].float().reshape(-1, half).contiguous()
    if cos_t.shape[0] != B * S:                                    # broadcast batch dim of the tables
        cos_t = cos_t.reshape(-1, S, half).expand(B, S, half).reshape(B * S, half).contiguous()
        sin_t = sin_t.reshape(-1, S, half).expand(B, S, half).reshape(B * S, half).contiguous()
    q3 = q.transpose(1, 2).reshape(B * S, H, D)
    k3 = k.transpose(1, 2).reshape(B * S, k.shape[1], D)
    q3 = _RopeOneFn.apply(q3, cos_t, sin_t, None, B * S)           # row t of the tables belongs to token t
    k3 = _RopeOneFn.apply(k3, cos_t, sin_t, None, B * S)
    return q3.view(B, S, H, D).transpose(1, 2), k3.view(B, S, k.shape[1], D).transpose(1, 2)


_HF_ROPE_ORIG = []


def linear_forward(self, x):
    return linear(x, self.weight, self.bias)


def _make_lce_forward(orig_forward):
    """Causal-LM forward that computes the loss with fused linear+CE when labels are given."""

    def lce_forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                    inputs_embeds=None, labels=None, use_cache=None, **kwargs):
        if labels is None:
            return orig_forward(self, input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                                past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                                **kwargs)
        shift = kwargs.pop("shift_labels", None)          # HF's own hook for sequence-sharded batches
        outputs = self.model(input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                             past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                             **{k: v for k, v in kwargs.items() if k not in ("num_items_in_batch", "logits_to_keep")})
        hidden = outputs[0]
        if shift is None:
            shift = torch.full_like(labels, -100)
            shift[..., :-1] = labels[..., 1:]
        loss = fused_linear_cross_entropy(hidden.reshape(-1, hidden.shape[-1]), self.lm_head.weight,
                                          shift.reshape(-1))
        from transformers.modeling_outputs import CausalLMOutputWithPast
        return CausalLMOutputWithPast(loss=loss, logits=None, past_key_values=getattr(outputs, "past_key_values", None))

    return lce_forward


def _make_moe_lce_forward(orig_forward, modeling):
    """Causal-LM forward of an HF MoE family with fused linear+CE when labels are given.  The rest is HF's: the router
    logits are requested from the decoder as HF does, and the family's ``load_balancing_loss_func`` is added with
    ``router_aux_loss_coef``; the result is a ``MoeCausalLMOutputWithPast`` with ``aux_loss`` and ``router_logits``."""

    def moe_lce_forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None,
                        inputs_embeds=None, labels=None, use_cache=None, output_router_logits=None, **kwargs):
        if labels is None:
            return orig_forward(self, input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                                past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                                output_router_logits=output_router_logits, **kwargs)
        if output_router_logits is None:
            output_router_logits = self.config.output_router_logits
        shift = kwargs.pop("shift_labels", None)
        outputs = self.model(input_ids=input_ids, attention_mask=attention_mask, position_ids=position_ids,
                             past_key_values=past_key_values, inputs_embeds=inputs_embeds, use_cache=use_cache,
                             output_router_logits=output_router_logits,
                             **{k: v for k, v in kwargs.items() if k not in ("num_items_in_batch", "logits_to_keep")})
        hidden = outputs[0]
        if shift is None:
            shift = torch.full_like(labels, -100)
            shift[..., :-1] = labels[..., 1:]
        loss = fused_linear_cross_entropy(hidden.reshape(-1, hidden.shape[-1]), self.lm_head.weight,
                                          shift.reshape(-1))
        aux_loss = None
        if output_router_logits:
            aux_loss = modeling.load_balancing_loss_func(outputs.router_logits, self.num_experts,
                                                         self.num_experts_per_tok, attention_mask)
            loss = loss + self.router_aux_loss_coef * aux_loss.to(loss.device)
        from transformers.modeling_outputs import MoeCausalLMOutputWithPast
        return MoeCausalLMOutputWithPast(loss=loss, aux_loss=aux_loss, logits=None,
                                         past_key_values=getattr(outputs, "past_key_values", None),
                                         router_logits=getattr(outputs, "router_logits", None))

    return moe_lce_forward


def _patch_family(modeling, prefix: str, rms_norm: bool, swiglu: bool, fused_linear_cross_entropy_: bool,
                  moe: bool = False):
    if rms_norm and hasattr(modeling, f"{prefix}RMSNorm"):
        getattr(modeling, f"{prefix}RMSNorm").forward = rms_forward
    if swiglu and hasattr(modeling, f"{prefix}MLP"):
        getattr(modeling, f"{prefix}MLP").forward = mlp_forward
    if fused_linear_cross_entropy_ and hasattr(modeling, f"{prefix}ForCausalLM"):
        cls = getattr(modeling, f"{prefix}ForCausalLM")
        if not getattr(cls, "_tb_lce_patched", False):
            cls.forward = _make_moe_lce_forward(cls.forward, modeling) if moe else _make_lce_forward(cls.forward)
            cls._tb_lce_patched = True


def apply_liger_kernel_to_llama(rope: bool = True, cross_entropy: bool = False, fused_linear_cross_entropy: bool = True,
                                rms_norm: bool = True, swiglu: bool = True, model: Optional[nn.Module] = None) -> None:
    """Reference liger.py:32-82.  ``rope``: HF applies RoPE inside its attention in a layout our in-place kernel
    does not see; attention itself is redirected by ``utils.patch.patch_fa`` so the flag is accepted and ignored."""
    from transformers.models.llama import modeling_llama
    _patch_family(modeling_llama, "Llama", rms_norm, swiglu, fused_linear_cross_entropy)
    if rope:
        _patch_rope(modeling_llama)


def apply_liger_kernel_to_qwen2(rope: bool = True, cross_entropy: bool = False, fused_linear_cross_entropy: bool = True,
                                rms_norm: bool = True, swiglu: bool = True, model: Optional[nn.Module] = None) -> None:
    """Reference liger.py:86-130."""
    from transformers.models.qwen2 import modeling_qwen2
    _patch_family(modeling_qwen2, "Qwen2", rms_norm, swiglu, fused_linear_cross_entropy)
    if rope:
        _patch_rope(modeling_qwen2)


def apply_liger_kernel_to_qwen3(rope: bool = True, cross_entropy: bool = False, fused_linear_cross_entropy: bool = True,
                                rms_norm: bool = True, swiglu: bool = True, model: Optional[nn.Module] = None) -> None:
    """Dense Qwen3.  Its per-head ``q_norm`` / ``k_norm`` are ``Qwen3RMSNorm`` modules on contiguous [B, S, H, D]
    views, so the RMSNorm class patch puts them on the native kernel too."""
    from transformers.models.qwen3 import modeling_qwen3
    _patch_family(modeling_qwen3, "Qwen3", rms_norm, swiglu, fused_linear_cross_entropy)
    if rope:
        _patch_rope(modeling_qwen3)


def experts_forward(self, hidden_states, top_k_index, top_k_weights):
    """HF 3-D experts module (``gate_up_proj [E, 2F, H]``, ``down_proj [E, H, F]``) on the grouped GEMM + routing
    kernels (ops/moe.py).  HF's router and its auxiliary loss stay HF's."""
    from .moe import moe_experts
    silu = type(getattr(self, "act_fn", None)).__name__ in ("SiLU", "SiLUActivation")
    if not (hidden_states.is_cuda and silu and getattr(self, "gate_up_proj_bias", None) is None):
        return type(self)._tb_orig_forward(self, hidden_states, top_k_index, top_k_weights)
    return moe_experts(hidden_states, top_k_index, top_k_weights, self.gate_up_proj, self.down_proj)


def _patch_experts(modeling, prefix: str) -> None:
    import inspect
    cls = getattr(modeling, f"{prefix}Experts", None)
    if cls is None or getattr(cls, "_tb_orig_forward", None) is not None:
        return
    params = inspect.signature(cls.forward).parameters
    if not all(p in params for p in ("hidden_states", "top_k_index", "top_k_weights")):
        logger.warning(f"{prefix}Experts.forward has an unknown signature; its experts keep HF's implementation")
        return
    cls._tb_orig_forward = cls.forward
    cls.forward = experts_forward


def _moe_family(module_path: str, prefix: str, rms_norm: bool, swiglu: bool, fused_linear_cross_entropy_: bool,
                experts: bool) -> None:
    import importlib
    modeling = importlib.import_module(module_path)
    _patch_family(modeling, prefix, rms_norm, swiglu, fused_linear_cross_entropy_, moe=True)   # swiglu: shared experts
    if experts:
        _patch_experts(modeling, prefix)


def apply_liger_kernel_to_mixtral(fused_linear_cross_entropy: bool = True, rms_norm: bool = True, swiglu: bool = True,
                                  experts: bool = True, **_unused) -> None:
    _moe_family("transformers.models.mixtral.modeling_mixtral", "Mixtral", rms_norm, swiglu,
                fused_linear_cross_entropy, experts)


def apply_liger_kernel_to_qwen2_moe(fused_linear_cross_entropy: bool = True, rms_norm: bool = True, swiglu: bool = True,
                                    experts: bool = True, **_unused) -> None:
    _moe_family("transformers.models.qwen2_moe.modeling_qwen2_moe", "Qwen2Moe", rms_norm, swiglu,
                fused_linear_cross_entropy, experts)


def apply_liger_kernel_to_qwen3_moe(fused_linear_cross_entropy: bool = True, rms_norm: bool = True, swiglu: bool = True,
                                    experts: bool = True, **_unused) -> None:
    _moe_family("transformers.models.qwen3_moe.modeling_qwen3_moe", "Qwen3Moe", rms_norm, swiglu,
                fused_linear_cross_entropy, experts)


def apply_liger_kernel_to_olmoe(fused_linear_cross_entropy: bool = True, rms_norm: bool = True, swiglu: bool = True,
                                experts: bool = True, **_unused) -> None:
    _moe_family("transformers.models.olmoe.modeling_olmoe", "Olmoe", rms_norm, swiglu, fused_linear_cross_entropy,
                experts)


def _patch_rope(modeling) -> None:
    from ..utils.patch import _patch_function
    orig = getattr(modeling, "apply_rotary_pos_emb", None)
    if orig is None or orig is hf_apply_rotary_pos_emb:
        return
    if not _HF_ROPE_ORIG:
        _HF_ROPE_ORIG.append(orig)
    _patch_function(modeling, "apply_rotary_pos_emb", hf_apply_rotary_pos_emb, required_params=("q", "k", "cos", "sin"))


def patch_linears(model: nn.Module) -> int:
    """Route every ``nn.Linear`` of this model instance through the wgmma GEMM."""
    n = 0
    for m in model.modules():
        if type(m) is nn.Linear:
            m.forward = linear_forward.__get__(m, nn.Linear)
            n += 1
    return n


def apply_liger_kernel(model: Optional[nn.Module] = None) -> None:
    """Best-effort patching used by ``accelerate()`` (reference liger.py:133-153).  With a model, only the HF
    families that actually occur in it are patched (class-level patches are process-global; a native model must not
    change how unrelated HF models behave); without one, every supported family is patched like the reference."""
    try:
        import transformers  # noqa: F401
    except Exception:
        transformers = None
    if transformers is not None:
        families = {"transformers.models.llama.": apply_liger_kernel_to_llama,
                    "transformers.models.qwen2.": apply_liger_kernel_to_qwen2,
                    "transformers.models.qwen3.": apply_liger_kernel_to_qwen3,
                    "transformers.models.mixtral.": apply_liger_kernel_to_mixtral,
                    "transformers.models.qwen2_moe.": apply_liger_kernel_to_qwen2_moe,
                    "transformers.models.qwen3_moe.": apply_liger_kernel_to_qwen3_moe,
                    "transformers.models.olmoe.": apply_liger_kernel_to_olmoe}
        if model is None:
            wanted = list(families.values())
        else:
            mods = {type(m).__module__ for m in model.modules()}
            wanted = [fn for prefix, fn in families.items() if any(x.startswith(prefix) for x in mods)]
        for fn in wanted:
            try:
                fn()
            except Exception as e:  # pragma: no cover - depends on the installed transformers
                logger.debug("kernel patch %s skipped: %s", fn.__name__, e)
        if wanted:
            # HF attention call sites (flash_attention_2 / the attention-interface registry) -> our wgmma kernels; the
            # reference does this at import time (torchacc/__init__.py:135), here it happens when a model needs it
            from ..utils.patch import patch_fa
            patch_fa()
    if model is not None and not type(model).__module__.startswith("torchacc_b200"):
        patch_linears(model)
