"""Operator library (reference torchacc/ops/__init__.py:1-6)."""
from .attention import (attention_reference, flash_attn_func, flash_attn_qkvpacked_tokens, flash_attn_varlen_func,
                        flash_attn_varlen_position_ids_func, flash_attn_varlen_position_ids_xla,
                        flash_attn_varlen_qkvpacked_func, flash_attn_varlen_qkvpacked_xla, flash_attn_varlen_xla,
                        flash_attn_xla, get_attention_backend, set_attention_backend, spmd_flash_attn_varlen_xla)
from .cross_entropy import cross_entropy, fused_linear_cross_entropy
from .linear import Linear, gemm, linear
from .liger import (apply_liger_kernel, apply_liger_kernel_to_llama, apply_liger_kernel_to_mixtral,
                    apply_liger_kernel_to_olmoe, apply_liger_kernel_to_qwen2, apply_liger_kernel_to_qwen2_moe,
                    apply_liger_kernel_to_qwen3, apply_liger_kernel_to_qwen3_moe)
from .moe import MoEMLP, moe_experts, moe_router
from .optim import FusedAdamW, grad_sqnorm
from .rmsnorm import RMSNorm, rmsnorm
from .rope import apply_rope, qk_norm_rope_qkv, rope_qkv_, rope_tables
from .sdpa import scaled_dot_product_attention
from .swiglu import swiglu
from . import context_parallel

__all__ = [n for n in dir() if not n.startswith("_")]
