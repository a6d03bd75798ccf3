"""torchacc_b200 -- an H100-native (sm_90a) training-acceleration framework with TorchAcc's capabilities.

``import torchacc_b200 as ta`` provides the reference's public surface (reference torchacc/__init__.py:4-22):
``ta.accelerate``, ``ta.Config``, ``ta.AsyncLoader``, ``ta.amp``, ``ta.dist``, ``ta.ops``, ``ta.utils``,
``ta.sync / lazy_device / is_lazy_device / is_lazy_tensor / fetch_gradients / mark_dynamic / save / mark_step``,
``ta.accelerate_hf_trainer``, ``ta.patch_qwen_model``, ``ta.get_global_context``.

Unlike the reference nothing is monkey-patched at import time (reference __init__.py:135-138): patches are
applied explicitly by ``accelerate()`` / ``ta.utils.patch``.
"""
from __future__ import annotations

from .version import __version__


class GlobalContext:
    """Process-wide state shared between layers (reference __init__.py:25-37)."""

    def __init__(self):
        self.config = None
        self.mesh = None
        self.python_dispatcher = None


_CONTEXT = None


def get_global_context() -> GlobalContext:
    global _CONTEXT
    if _CONTEXT is None:
        _CONTEXT = GlobalContext()
    return _CONTEXT


from .config import Config  # noqa: E402
from . import utils  # noqa: E402
from . import ops  # noqa: E402
from . import parallel  # noqa: E402
from . import parallel as dist  # noqa: E402  (reference name: ta.dist)
from . import models  # noqa: E402
from . import llm  # noqa: E402
from .core import (AsyncLoader, amp, fetch_gradients, is_lazy_device, is_lazy_tensor, lazy_device, mark_dynamic,  # noqa: E402
                   mark_step, save, send_cpu_data_to_device, sync)
from .core.accelerate_hf_trainer import accelerate_hf_trainer  # noqa: E402
from .accelerate import accelerate  # noqa: E402
from .llm import patch_qwen_model  # noqa: E402
from .utils import decompose, import_utils, patch  # noqa: E402
from .ops import optim  # noqa: E402

__all__ = [
    "accelerate", "Config", "AsyncLoader", "amp", "dist", "parallel", "ops", "utils", "models", "llm", "optim",
    "sync", "lazy_device", "is_lazy_device", "is_lazy_tensor", "fetch_gradients", "mark_dynamic", "mark_step",
    "save", "send_cpu_data_to_device", "accelerate_hf_trainer", "patch_qwen_model", "get_global_context",
    "__version__",
]
