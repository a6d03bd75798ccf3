"""``accelerate(model, dataloader=None, config=Config())`` -- the one-call entry point.

Same contract as reference torchacc/accelerate.py:49-149: validate the config, bring up the process groups and the
mesh, wrap the dataloader in an ``AsyncLoader``, apply kernel patches, build the parallel wrappers
(PP / TP / CP / FSDP / DP), apply gradient checkpointing, move to the device and return ``model`` or
``(model, loader)``.  What changed underneath: no XLA flags / lazy device; kernel "patches" swap HF module
forwards onto our sm_90a ops; deferred (meta-device) models are materialised unit by unit instead of torchdistx.
"""
from __future__ import annotations

import inspect
from typing import Optional

import torch
import torch.nn as nn

from .config import Config
from .utils.logger import logger


def _materialize_meta(model: nn.Module, device: torch.device) -> None:
    """Deferred init (reference accelerate.py:13-17,114-119 uses torchdistx): allocate real storage for
    meta-device parameters and run each module's ``reset_parameters`` where available."""
    has_meta = any(p.is_meta for p in model.parameters()) or any(b.is_meta for b in model.buffers())
    if not has_meta:
        return
    model.to_empty(device=device)
    if hasattr(model, "reset_parameters"):
        model.reset_parameters()
    else:
        for m in model.modules():
            if m is not model and hasattr(m, "reset_parameters"):
                m.reset_parameters()


def accelerate(model: nn.Module, dataloader=None, config: Optional[Config] = None):
    from . import get_global_context
    from .parallel import bootstrap
    from .parallel.distributed_parallel import DistributedParallel

    config = config if config is not None else Config()
    config.validate()
    get_global_context().config = config

    if config.is_distributed_parallel() or bootstrap.world_size() > 1:
        bootstrap.init_process_group(config)
        bootstrap.init_nccl_context(None)
    device = bootstrap.current_device()
    if device.type == "cuda":
        torch.cuda.set_device(device)

    loader = None
    if dataloader is not None:
        from .core.async_loader import AsyncLoader
        dl = config.dataloader
        loader = AsyncLoader(dataloader, device, buckets=dl.buckets, max_length=dl.max_length,
                             num_buckets=dl.num_buckets, pad_value_dict=dl.pad_value_dict, prefetch=dl.prefetch,
                             pin_memory=dl.pin_memory)

    from .ops import fp8 as _fp8
    if getattr(config.compute, "fp8", False):
        if device.type == "cuda" and _fp8.available():
            _fp8.enable(True)           # linear layers: MX-FP8 (e4m3 + UE8M0 block scales) wgmma GEMMs, ops/fp8.py
        else:
            from .utils.logger import logger
            logger.warning("compute.fp8 needs a CUDA device and the native library; linear layers stay in %s",
                           "bf16" if config.compute.bf16 else "fp32")
    else:
        _fp8.enable(False)
    # deterministic mode: atomic-free attention dQ and ordered gradient-norm sums (process-wide, like compute.fp8)
    from .ops import attention as _attn, optim as _optim
    _attn.set_deterministic(config.compute.deterministic)
    _optim.set_deterministic(config.compute.deterministic)
    if config.compute.acc_scaled_dot_attn:
        from .ops.sdpa import patch_sdpa
        patch_sdpa()
    if not config.compute.disable_kernel_patches:
        from .ops.liger import apply_liger_kernel
        apply_liger_kernel(model)

    orig_sig = inspect.signature(model.forward)
    _materialize_meta(model, device)

    # always the same wrapper type (reference accelerate.py:127-131): training scripts call model.clip_grad_norm_ /
    # *_optim_state_dict regardless of the world size; with one rank the engine simply has no collectives
    model = DistributedParallel(model, config, orig_forward_sig=orig_sig)
    model.to(device)
    if not isinstance(getattr(type(model), "device", None), property):   # HF models expose a read-only property
        try:
            model.device = device
        except Exception:
            object.__setattr__(model, "device", device)
    return (model, loader) if dataloader is not None else model
