"""Explicit monkey patches for third-party code (reference torchacc/utils/patch.py:16-313).

* ``patch_fa``      : HF ``_flash_attention_forward`` -> our flash-attention ops (fixed / varlen-by-mask /
                      packed-by-position-ids), signature-checked so an incompatible transformers release is refused
                      instead of silently mis-called (the reference logs and continues, patch.py:16-24);
* ``patch_llama`` / ``patch_qwen`` : make HF Llama / Qwen2 use the patched attention + our kernels;
* ``patch_amp``     : ``torch.optim.Adam/AdamW`` -> ``FusedAdamW`` and ``torch.cuda.amp.GradScaler`` -> ours;
* ``patch_autocast``: the reference maps autocast('xla') to 'cuda'; kept as a tolerant alias.
Nothing here runs at import time (the reference patches on import, __init__.py:135-138).
"""
from __future__ import annotations

import inspect
import os
from typing import Callable

import torch

from .logger import logger

_PATCHED = {}


def _patch_function(module, name: str, new: Callable, required_params=()) -> bool:
    """Replace ``module.name`` by ``new`` after checking that the original accepts ``required_params``."""
    orig = getattr(module, name, None)
    if orig is None:
        logger.warning("patch: %s.%s not found", getattr(module, "__name__", module), name)
        return False
    try:
        params = inspect.signature(orig).parameters
    except (TypeError, ValueError):
        params = {}
    missing = [p for p in required_params if p not in params]
    if missing:
        logger.warning("patch: %s.%s has an unexpected signature (missing %s); not patched", module.__name__, name,
                       missing)
        return False
    _PATCHED[(module.__name__, name)] = orig
    setattr(module, name, new)
    return True


def unpatch_all() -> None:
    import importlib
    for (mod, name), orig in list(_PATCHED.items()):
        setattr(importlib.import_module(mod), name, orig)
        del _PATCHED[(mod, name)]


def _hf_flash_attention_forward(query_states, key_states, value_states, attention_mask=None, query_length=None,
                                is_causal=True, dropout=0.0, position_ids=None, softmax_scale=None,
                                sliding_window=None, use_top_left_mask=False, softcap=None, deterministic=None,
                                **kwargs):
    """Drop-in for ``transformers.modeling_flash_attention_utils._flash_attention_forward`` ([B,S,H,D] layout).
    ``deterministic=None`` follows ``FLASH_ATTENTION_DETERMINISTIC=1``, as HF's own function does."""
    from ..ops import attention as A
    window = (sliding_window - 1, 0) if sliding_window else (-1, -1)
    causal = bool(is_causal) and not (use_top_left_mask and query_states.shape[1] == 1)
    if deterministic is None:
        deterministic = os.environ.get("FLASH_ATTENTION_DETERMINISTIC", "0") == "1"
    if attention_mask is not None and attention_mask.dim() == 2 and not bool(attention_mask.all()):
        return A.flash_attn_varlen_func(query_states, key_states, value_states, attention_mask, dropout, softmax_scale,
                                        causal, window, deterministic=deterministic)
    if position_ids is not None and query_states.shape[0] == 1 and position_ids.numel() > 1 \
            and bool((position_ids.reshape(-1)[1:] == 0).any()):
        return A.flash_attn_varlen_position_ids_func(query_states, key_states, value_states, position_ids, dropout,
                                                     softmax_scale, causal, window, deterministic=deterministic)
    return A.flash_attn_func(query_states, key_states, value_states, dropout, softmax_scale, causal, window,
                             deterministic=deterministic)


def patch_fa() -> bool:
    """Route HF flash-attention-2 call sites to our kernels (env ``TORCHACC_PATCH_FA=0`` disables)."""
    if os.environ.get("TORCHACC_PATCH_FA", "1") == "0":
        return False
    try:
        import transformers.modeling_flash_attention_utils as fa_utils
    except Exception as e:
        logger.warning("patch_fa: transformers flash-attention utils unavailable (%s)", e)
        return False
    ok = _patch_function(fa_utils, "_flash_attention_forward", _hf_flash_attention_forward,
                         required_params=("query_states", "key_states", "value_states", "attention_mask"))
    try:  # newer releases dispatch through the attention-interface registry
        from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS

        def _iface(module, query, key, value, attention_mask, dropout=0.0, scaling=None, sliding_window=None,
                   **kwargs):
            q, k, v = query.transpose(1, 2), key.transpose(1, 2), value.transpose(1, 2)
            out = _hf_flash_attention_forward(q, k, v, attention_mask if (attention_mask is not None and
                                                                          attention_mask.dim() == 2) else None,
                                              is_causal=getattr(module, "is_causal", True), dropout=dropout,
                                              softmax_scale=scaling, sliding_window=sliding_window,
                                              position_ids=kwargs.get("position_ids"))
            return out, None

        ALL_ATTENTION_FUNCTIONS["torchacc_b200"] = _iface
        ALL_ATTENTION_FUNCTIONS["flash_attention_2"] = _iface
        ok = True
    except Exception:
        pass
    return ok


def patch_llama(use_flash_attn: bool = True) -> None:
    """HF Llama on our kernels (reference patch.py:224-246)."""
    from ..ops.liger import apply_liger_kernel_to_llama
    apply_liger_kernel_to_llama()
    if use_flash_attn:
        patch_fa()


def patch_qwen(use_flash_attn: bool = True) -> None:
    """HF Qwen2 on our kernels.  (The reference regex-rewrites Qwen remote code for XLA's static shapes,
    patch.py:249-301; unnecessary in eager mode.)"""
    from ..ops.liger import apply_liger_kernel_to_qwen2
    apply_liger_kernel_to_qwen2()
    if use_flash_attn:
        patch_fa()


def patch_amp() -> None:
    """``torch.optim.Adam/AdamW`` -> FusedAdamW, ``torch.cuda.amp.GradScaler`` -> ours (reference patch.py:51-58)."""
    from ..core.amp import GradScaler
    from ..ops.optim import FusedAdamW
    _PATCHED.setdefault(("torch.optim", "AdamW"), torch.optim.AdamW)
    _PATCHED.setdefault(("torch.optim", "Adam"), torch.optim.Adam)
    torch.optim.AdamW = FusedAdamW
    torch.optim.Adam = FusedAdamW
    torch.cuda.amp.GradScaler = GradScaler


def patch_autocast() -> None:
    """Accept ``torch.autocast('xla', ...)`` by mapping it to 'cuda' (reference patch.py:304-313)."""
    if os.environ.get("TORCHACC_PATCH_TORCH_AUTOCAST", "1") == "0" or ("torch", "autocast") in _PATCHED:
        return
    orig = torch.autocast

    class _Autocast(orig):
        def __init__(self, device_type, *args, **kwargs):
            super().__init__("cuda" if device_type == "xla" else device_type, *args, **kwargs)

    _PATCHED[("torch", "autocast")] = orig
    torch.autocast = _Autocast
