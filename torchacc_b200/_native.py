"""ctypes loader for the in-tree native library (``torchacc_b200/_C.so``, built by ``build_native.py``).

Policy: on a machine with a CUDA device the native library is REQUIRED -- ops raise instead of silently
falling back to PyTorch (set ``TORCHACC_B200_ALLOW_FALLBACK=1`` to opt into the fallback explicitly).
On CPU-only hosts (the plumbing/test tier) the library is optional and every op uses its PyTorch reference.
"""
from __future__ import annotations

import ctypes
import os
from pathlib import Path
from typing import Optional

import torch

_LIB: Optional[ctypes.CDLL] = None
_TRIED = False
_SO = Path(os.environ.get("TORCHACC_B200_NATIVE_LIB") or (Path(__file__).resolve().parent / "_C.so"))   # env: A/B builds

u64, i32, i64, f32 = ctypes.c_uint64, ctypes.c_int, ctypes.c_longlong, ctypes.c_float

_SIGS = {
    "tb_abi_version": ([], i32),
    "tb_device_info": ([i32, ctypes.POINTER(i32), ctypes.POINTER(i32), ctypes.POINTER(i32), ctypes.POINTER(i64)], i32),
    "tb_gemm_bf16": ([u64, u64, u64, u64, i32, i32, i32, i64, i64, i64, i32, i32, i32, i32, i32, i32, u64, i32], i32),
    "tb_gemm_sched_mode": ([i32], i32),
    "tb_gemm_bf16_ex": ([u64, u64, u64, u64, u64, i32, i32, i32, i64, i64, i64, i64, i32, i32, i32, i32, i32, u64, i32],
                        i32),
    "tb_rmsnorm_fwd": ([u64, u64, u64, u64, u64, u64, i32, i32, f32, i32, u64, i32], i32),
    "tb_rmsnorm_bwd": ([u64, u64, u64, u64, u64, u64, u64, i32, i32, i32, i32, u64, i32], i32),
    "tb_rope_inplace": ([u64, u64, u64, u64, i64, i32, i32, i64, i32, i32, i32, u64, i32], i32),
    "tb_qk_norm_rope_fwd": ([u64, u64, u64, u64, u64, u64, u64, u64, i64, i32, i32, i32, i64, i32, f32, i32, u64, i32],
                            i32),
    "tb_qk_norm_rope_bwd": ([u64, u64, u64, u64, u64, u64, u64, i32, u64, u64, u64, i64, i32, i32, i32, i64, i32, i32,
                             u64, i32], i32),
    "tb_swiglu_fwd": ([u64, u64, u64, i64, i32, i64, i64, i32, u64, i32], i32),
    "tb_swiglu_bwd": ([u64, u64, u64, u64, u64, i64, i32, i64, i64, i64, i64, i32, u64, i32], i32),
    "tb_cross_entropy": ([u64, u64, u64, u64, i32, i32, i64, i32, u64, f32, i32, u64], i32),
    "tb_adamw_flat": ([u64, u64, i32, u64, u64, u64, i64, f32, f32, f32, f32, f32, i32, u64, u64, u64, i32, u64], i32),
    "tb_sqnorm_accumulate": ([u64, i32, i64, u64, f32, i32, u64], i32),
    "tb_scale_inplace": ([u64, i32, i64, u64, i32, u64], i32),
}
# signatures registered by optional subsystems (attention, comm) -- see register_signatures()
_EXTRA_SIGS = {}


class NativeError(RuntimeError):
    pass


def allow_fallback() -> bool:
    return os.environ.get("TORCHACC_B200_ALLOW_FALLBACK", "0") == "1"


def register_signatures(sigs: dict) -> None:
    _EXTRA_SIGS.update(sigs)
    if _LIB is not None:
        _apply(_LIB, sigs)


def _apply(lib, sigs):
    for name, (argtypes, restype) in sigs.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue
        fn.argtypes = argtypes
        fn.restype = restype


def lib() -> Optional[ctypes.CDLL]:
    """The loaded native library, or None when it is not built / not loadable."""
    global _LIB, _TRIED
    if _TRIED:
        return _LIB
    _TRIED = True
    if not _SO.exists():
        return None
    try:
        L = ctypes.CDLL(str(_SO))
    except OSError:
        return None
    L.tb_error_string.argtypes = [i32]
    L.tb_error_string.restype = ctypes.c_char_p
    _apply(L, _SIGS)
    _apply(L, _EXTRA_SIGS)
    _LIB = L
    return _LIB


def available() -> bool:
    return lib() is not None


def require() -> ctypes.CDLL:
    L = lib()
    if L is None:
        raise NativeError(
            f"torchacc_b200 native library not found at {_SO}. Build it with "
            "`python -m torchacc_b200.build_native` (or `python -c 'import __graft_entry__ as g; g.build()'`). "
            "Set TORCHACC_B200_ALLOW_FALLBACK=1 to run the PyTorch reference ops instead.")
    return L


def check(code: int, what: str) -> None:
    if code != 0:
        msg = lib().tb_error_string(code).decode() if lib() is not None else "?"
        raise NativeError(f"{what} failed: CUDA error {code} ({msg})")


def use_native(*tensors) -> bool:
    """Decide between the sm_90a kernels and the PyTorch reference path for these tensors."""
    if not tensors or not all(t.is_cuda for t in tensors if isinstance(t, torch.Tensor)):
        return False
    if os.environ.get("TORCHACC_B200_DISABLE_NATIVE", "0") == "1":   # accuracy baselines: plain PyTorch ops on the GPU
        return False
    if lib() is None:
        if allow_fallback():
            return False
        require()
    return True


_DEV_INFO = {}


def device_info(device: Optional[int] = None) -> dict:
    device = torch.cuda.current_device() if device is None else device
    if device not in _DEV_INFO:
        L = require()
        a, b, c, d = i32(), i32(), i32(), i64()
        check(L.tb_device_info(device, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c), ctypes.byref(d)),
              "tb_device_info")
        _DEV_INFO[device] = dict(num_sms=a.value, cc=(b.value, c.value), smem_optin=d.value)
    return _DEV_INFO[device]


def num_sms() -> int:
    return device_info()["num_sms"]


def stream() -> int:
    return torch.cuda.current_stream().cuda_stream


_HALF = (torch.bfloat16, torch.float16)


def is_half(*ts) -> bool:
    """All tensors share one 16-bit float dtype (the native kernels are templated on bf16 / fp16)."""
    return all(t.dtype == ts[0].dtype for t in ts) and ts[0].dtype in _HALF


def bf16_flag(t) -> int:
    return int(t.dtype == torch.bfloat16)


def set_gemm_scheduler(dynamic: bool) -> None:
    """Tile scheduling of the wgmma GEMM: static striping (fastest when the GEMM owns the GPU) or dynamic:
    one CTA per tile, placed by the block scheduler (robust when collective kernels occupy some SMs on side streams).  The env
    var ``TORCHACC_B200_GEMM_SCHED=static|dynamic`` pins the mode."""
    if os.environ.get("TORCHACC_B200_GEMM_SCHED", "auto") not in ("auto", ""):
        return
    L = lib()
    if L is not None and hasattr(L, "tb_gemm_sched_mode"):
        L.tb_gemm_sched_mode(1 if dynamic else 0)


def ptr(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


# launch counter: bench.py reports how many of OUR kernels ran inside the timed region
LAUNCHES = 0


def count_launch(n: int = 1) -> None:
    global LAUNCHES
    LAUNCHES += n
