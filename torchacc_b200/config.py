"""Configuration tree for torchacc_b200.

Same user-facing shape as the reference ``Config`` (reference torchacc/config.py:27-444): a tree of
``compute / memory / dataloader / dist{dp,tp,pp,fsdp,sp,topology}`` sections with attribute assignment,
``validate()``, ``get_mesh()`` and the ``is_*`` predicates.  Differences by design:

* validation is table-driven (each section declares ``_SPEC``: field -> (types, check)) instead of a wall of
  asserts, and every section round-trips through ``to_dict`` / ``from_dict`` / ``from_yaml`` / ``from_json``
  (the reference has a "TODO: support dict", config.py:339);
* there is no XLA ``lazy`` backend: ``backend`` accepts ``'eager'`` (and tolerates ``'lazy'`` with a warning);
* additions required by the GPU-native design: ``compute.fp8``, ``compute.fused_kernels``, ``dist.sp.mode``
  (``ulysses`` / ``ring`` / ``2d``) and ``dist.sp.ulysses_size``, ``dist.fsdp.reduce_dtype``,
  ``dist.fsdp.fused_collectives``, ``dist.tp.sequence_parallel``; ``'sp'`` is a real mesh axis;
* reference defects not reproduced: ``DataLoaderConfig.validate`` type-checking the wrong field
  (config.py:112-115) and ``SPConfig`` not being a dataclass (config.py:273).
"""
from __future__ import annotations

import copy
import json
import os
from typing import Any, Dict, Optional

import torch

_AXES = ("dp", "fsdp", "pp", "tp", "sp")


class ConfigError(ValueError):
    pass


def _is_pos_int(v):
    return isinstance(v, int) and not isinstance(v, bool) and v >= 1


class Section:
    """Base class: a flat record described by ``_SPEC = {name: (default_factory, predicate, message)}``."""
    _SPEC: Dict[str, tuple] = {}

    def __init__(self, **kwargs):
        for name, (default, _pred, _msg) in self._SPEC.items():
            value = kwargs.pop(name) if name in kwargs else (default() if callable(default) else default)
            object.__setattr__(self, name, value)
        if kwargs:
            raise ConfigError(f"{type(self).__name__}: unknown field(s) {sorted(kwargs)}")

    def __setattr__(self, name, value):
        if name not in self._SPEC and not name.startswith("_"):
            raise AttributeError(f"{type(self).__name__} has no field '{name}'")
        object.__setattr__(self, name, value)

    def validate(self):
        for name, (_default, pred, msg) in self._SPEC.items():
            value = getattr(self, name)
            if isinstance(value, Section):
                value.validate()
            elif pred is not None and not pred(value):
                raise ConfigError(f"{type(self).__name__}.{name} {msg}, got {value!r}")
        self._cross_validate()

    def _cross_validate(self):
        pass

    def to_dict(self) -> Dict[str, Any]:
        out = {}
        for name in self._SPEC:
            v = getattr(self, name)
            if isinstance(v, Section):
                out[name] = v.to_dict()
            elif isinstance(v, set):
                out[name] = sorted(v)
            elif isinstance(v, (list, tuple)):
                out[name] = [x if isinstance(x, (str, int, float, bool, type(None))) else repr(x) for x in v]
            elif callable(v):
                out[name] = getattr(v, "__qualname__", repr(v))
            else:
                out[name] = v
        return out

    @classmethod
    def from_dict(cls, d: Dict[str, Any]):
        obj = cls()
        for k, v in (d or {}).items():
            if k not in cls._SPEC:
                raise ConfigError(f"{cls.__name__}: unknown field '{k}'")
            cur = getattr(obj, k)
            if isinstance(cur, Section):
                setattr(obj, k, type(cur).from_dict(v))
            elif isinstance(cur, set) or k in ("wrap_layer_cls", "gc_cls"):
                setattr(obj, k, set(v) if v is not None else None)
            else:
                setattr(obj, k, v)
        return obj

    def __repr__(self):
        body = ", ".join(f"{k}={getattr(self, k)!r}" for k in self._SPEC)
        return f"{type(self).__name__}({body})"

    def __eq__(self, other):
        return type(self) is type(other) and all(getattr(self, k) == getattr(other, k) for k in self._SPEC)


_bool = (lambda v: isinstance(v, bool), "must be a bool")
_opt_pos_int = (lambda v: v is None or _is_pos_int(v), "must be None or an int >= 1")
_pos_int = (_is_pos_int, "must be an int >= 1")


class ComputeConfig(Section):
    """fp16/bf16 mixed precision, attention replacement, kernel patches (reference config.py:27-54).

    New: ``fp8`` enables the block-scaled fp8 GEMM path on the linear layers of native models;
    ``fused_kernels`` selects the hand-written sm_90a kernels for GEMM/attention/norm/rope/loss
    (``False`` falls back to plain PyTorch ops -- the CPU plumbing tier always does);
    ``deterministic`` makes a single-GPU training step bitwise reproducible: the attention backward computes dQ
    without atomics and the gradient-norm reduction sums in a fixed order (off by default).
    """
    _SPEC = {
        "fp16": (False, ) + _bool,
        "bf16": (False, ) + _bool,
        "fp8": (False, ) + _bool,
        "acc_scaled_dot_attn": (False, ) + _bool,
        "disable_kernel_patches": (False, ) + _bool,
        "fused_kernels": (True, ) + _bool,
        "deterministic": (False, ) + _bool,
    }

    def _cross_validate(self):
        if self.fp16 and self.bf16:
            raise ConfigError("ComputeConfig: fp16 and bf16 cannot both be True")
        if self.fp8 and self.fp16:
            raise ConfigError("ComputeConfig: fp8 GEMMs require bf16 (or fp32) activations, not fp16")

    @property
    def dtype(self) -> torch.dtype:
        return torch.bfloat16 if self.bf16 else torch.float16 if self.fp16 else torch.float32


class MemoryConfig(Section):
    """Gradient checkpointing (reference config.py:58-88) + activation CPU offload knobs."""
    _SPEC = {
        "gc": (False, ) + _bool,
        "gc_cls": (None, lambda v: v is None or (isinstance(v, set) and all(isinstance(c, str) for c in v)),
                   "must be None or a set of class names"),
        "gc_cnt": (None, lambda v: v is None or (isinstance(v, int) and not isinstance(v, bool) and v >= 0),
                   "must be None or an int >= 0"),
        "offload_activations": (False, ) + _bool,
        "offload_layers": (None, ) + _opt_pos_int,
    }


class DataLoaderConfig(Section):
    """Bucketed async loader options (reference config.py:92-127)."""
    _SPEC = {
        "buckets": (None, lambda v: v is None or (isinstance(v, list) and all(_is_pos_int(b) for b in v)),
                    "must be None or a list of positive ints"),
        "max_length": (None, ) + _opt_pos_int,
        "num_buckets": (None, ) + _opt_pos_int,
        "pad_value_dict": (None, lambda v: v is None or isinstance(v, dict), "must be None or a dict"),
        "prefetch": (2, ) + _pos_int,
        "pin_memory": (True, ) + _bool,
    }

    def _cross_validate(self):
        if self.buckets is not None and sorted(self.buckets) != list(self.buckets):
            raise ConfigError("DataLoaderConfig.buckets must be sorted ascending")


class DPConfig(Section):
    """Data parallel degree; ``None`` = infer from the world size (reference config.py:131-146, 320-324)."""
    _SPEC = {"size": (None, ) + _opt_pos_int}


class TPConfig(Section):
    """Tensor parallel degree.  ``sequence_parallel`` keeps the residual stream sharded along the sequence
    between the column- and row-parallel linears (all-gather->GEMM / GEMM->reduce-scatter kernels)."""
    _SPEC = {"size": (1, ) + _pos_int, "sequence_parallel": (True, ) + _bool}


class PPConfig(Section):
    """Pipeline parallel (reference config.py:165-221).  The model is cut *before* each split point."""
    _SPEC = {
        "size": (1, ) + _pos_int,
        "num_micro_batches": (1, ) + _pos_int,
        "input_names": (None, lambda v: v is None or (isinstance(v, list) and all(isinstance(n, str) for n in v)),
                        "must be None or a list of str"),
        "split_points": (list, lambda v: isinstance(v, list), "must be a list"),
        "broadcast_loss": (True, ) + _bool,
        "schedule": ("1f1b", lambda v: v in ("1f1b", "gpipe"), "must be '1f1b' or 'gpipe'"),
    }

    def _cross_validate(self):
        pts = self.split_points
        if pts:
            all_str = all(isinstance(p, str) for p in pts)
            all_mod = all(isinstance(p, torch.nn.Module) for p in pts)
            if not (all_str or all_mod):
                raise ConfigError("PPConfig.split_points must be all module names or all nn.Module objects")
            keys = pts if all_str else [id(p) for p in pts]
            if len(set(keys)) != len(keys):
                raise ConfigError("PPConfig.split_points contains duplicates")
        if self.size != len(pts) + 1:
            raise ConfigError(f"PPConfig: need pp.size - 1 = {self.size - 1} split points, got {len(pts)}")


class FSDPConfig(Section):
    """ZeRO-3 sharding (reference config.py:225-270).

    ``reduce_dtype``: wire/accumulate dtype of the gradient reduce-scatter (reference eager path reduces in
    fp32, dist/fsdp.py:204-208; our peer-memory kernel reads bf16 partials and accumulates in fp32).
    ``grad_dtype``: dtype of the flat gradient buffer / accumulation / wire (see the inline comment).
    ``fused_collectives``: use the symmetric-memory kernels (all-gather / reduce-scatter over NVLink peer
    memory, fused with cast and the optimizer hand-off) instead of NCCL calls.
    ``reshard_after_forward``: see the inline comment (torch FSDP's FULL_SHARD vs SHARD_GRAD_OP trade-off).
    """
    _SPEC = {
        "size": (1, ) + _pos_int,
        "wrap_layer_cls": (set, lambda v: isinstance(v, set) and all(isinstance(c, str) for c in v),
                           "must be a set of class names"),
        "flatten_parameters": (True, ) + _bool,
        "sync_module_states": (False, ) + _bool,
        "use_spmd": (False, ) + _bool,
        "shard_output_callable": (None, lambda v: v is None or callable(v), "must be None or callable"),
        "reduce_dtype": ("fp32", lambda v: v in ("fp32", "bf16"), "must be 'fp32' or 'bf16'"),
        # dtype of the FLAT gradient buffer: what the wgrad GEMM epilogues write, what micro-batches accumulate in and
        # what travels on the reduce-scatter wire.  "compute" (default) = bf16/fp16 buffer, fp32 accumulation at the
        # destination; "fp32" = fp32 end to end like the reference's fp32 reduce (dist/fsdp.py:204-208) at twice the
        # gradient bytes (the wgrad GEMM accumulates into the fp32 buffer straight from its accumulators).
        "grad_dtype": ("compute", lambda v: v in ("compute", "fp32"), "must be 'compute' or 'fp32'"),
        "fused_collectives": (True, ) + _bool,
        "prefetch": (1, lambda v: isinstance(v, int) and v >= 0, "must be an int >= 0"),
        # None = auto: keep the gathered bf16 parameters of every unit resident from the forward through the backward
        # (one all-gather per unit and step instead of two) whenever the full bf16 copy of the model is small next to
        # the device memory (<= 20 %); True = classic ZeRO-3 (free after forward, gather again for backward).
        "reshard_after_forward": (None, lambda v: v is None or isinstance(v, bool), "must be None (auto) or a bool"),
    }

    def _cross_validate(self):
        if self.use_spmd:
            from .utils.logger import logger
            logger.warning("FSDPConfig.use_spmd: the XLA SPMD partitioner does not exist in this framework; "
                           "the native FSDP engine (optionally composed with TP) is used instead")


class SPConfig(Section):
    """Sequence / context parallel.  ``mode``: 'ulysses' (all-to-all over heads), 'ring' (ring attention) or
    '2d' (ulysses inside ``ulysses_size`` ranks x ring across the rest; reference context_parallel_2d.py)."""
    _SPEC = {
        "size": (1, ) + _pos_int,
        "mode": ("ulysses", lambda v: v in ("ulysses", "ring", "2d"), "must be 'ulysses', 'ring' or '2d'"),
        "ulysses_size": (None, ) + _opt_pos_int,
        "zigzag": (True, ) + _bool,
    }

    def _cross_validate(self):
        if self.ulysses_size is not None and self.size % self.ulysses_size != 0:
            raise ConfigError("SPConfig.ulysses_size must divide SPConfig.size")


def _world_size() -> int:
    return int(os.environ.get("WORLD_SIZE", "1"))


class DistConfig(Section):
    """Parallel degrees + rank topology (reference config.py:283-336).  ``topology`` lists axes from the
    slowest-varying (largest rank stride, inter-node) to the fastest-varying (adjacent ranks, NVSwitch)."""
    _SPEC = {
        "dp": (DPConfig, None, ""),
        "tp": (TPConfig, None, ""),
        "pp": (PPConfig, None, ""),
        "fsdp": (FSDPConfig, None, ""),
        "sp": (SPConfig, None, ""),
        "topology": (lambda: ["dp", "fsdp", "pp", "sp", "tp"], lambda v: isinstance(v, list),
                     "must be a list of axis names"),
    }

    def _cross_validate(self):
        topo = list(self.topology)
        if len(set(topo)) != len(topo):
            raise ConfigError("DistConfig.topology has duplicate axes")
        for t in topo:
            if t not in _AXES:
                raise ConfigError(f"DistConfig.topology: unknown axis '{t}' (expected {_AXES})")
        # axes the user left out are appended with the reference's default relative order
        for t in _AXES:
            if t not in topo:
                if getattr(self, t).size not in (None, 1):
                    # insert just before 'tp' (fast axis) if present, else at the end
                    idx = topo.index("tp") if "tp" in topo else len(topo)
                    topo.insert(idx, t)
        object.__setattr__(self, "topology", topo)
        used = self.pp.size * self.fsdp.size * self.tp.size * self.sp.size
        world = _world_size()
        if self.dp.size is None:
            if world % used != 0:
                raise ConfigError(f"world size {world} is not divisible by pp*fsdp*tp*sp = {used}")
            self.dp.size = world // used
        elif world > 1 and self.dp.size * used != world:
            raise ConfigError(f"dp*pp*fsdp*tp*sp = {self.dp.size * used} does not match world size {world}")

    def sizes(self) -> Dict[str, int]:
        return {a: (getattr(self, a).size or 1) for a in _AXES}


class Config(Section):
    """Top-level configuration (reference config.py:341-444)."""
    _SPEC = {
        "backend": ("eager", lambda v: v in ("eager", "lazy"), "must be 'eager' (the XLA 'lazy' backend was dropped)"),
        "compute": (ComputeConfig, None, ""),
        "memory": (MemoryConfig, None, ""),
        "dist": (DistConfig, None, ""),
        "dataloader": (DataLoaderConfig, None, ""),
    }

    def _cross_validate(self):
        if self.backend == "lazy":
            from .utils.logger import logger
            logger.warning("Config.backend='lazy' requested: there is no lazy-tensor backend in torchacc_b200; "
                           "running eagerly on CUDA streams/graphs")
            object.__setattr__(self, "backend", "eager")

    # ---- mesh ---------------------------------------------------------------------------------------
    def get_mesh(self):
        """Create (once) the process-group mesh for this config (reference config.py:389-413)."""
        mesh = getattr(self, "_mesh", None)
        if mesh is not None:
            return mesh
        self.validate()
        from . import get_global_context
        from .parallel import bootstrap
        from .parallel.mesh import Mesh
        bootstrap.init_process_group(self)
        s = self.dist.sizes()
        mesh = Mesh(dp_num=s["dp"], pp_num=s["pp"], tp_num=s["tp"], fsdp_num=s["fsdp"], sp_num=s["sp"],
                    topology=self.dist.topology, sp_mode=self.dist.sp.mode, ulysses_num=self.dist.sp.ulysses_size)
        object.__setattr__(self, "_mesh", mesh)
        get_global_context().mesh = mesh
        return mesh

    # ---- predicates ---------------------------------------------------------------------------------
    def is_distributed_parallel(self) -> bool:
        return any((getattr(self.dist, a).size or 1) > 1 for a in _AXES)

    def is_tracing_enabled(self) -> bool:
        return self.dist.pp.size > 1

    def is_lazy_backend(self) -> bool:
        return False

    def is_eager_backend(self) -> bool:
        return True

    # ---- serialisation ------------------------------------------------------------------------------
    def to_json(self, path: Optional[str] = None) -> str:
        text = json.dumps(self.to_dict(), indent=2, sort_keys=True)
        if path:
            with open(path, "w") as f:
                f.write(text)
        return text

    @classmethod
    def from_json(cls, path_or_text: str) -> "Config":
        text = open(path_or_text).read() if os.path.exists(path_or_text) else path_or_text
        return cls.from_dict(json.loads(text))

    @classmethod
    def from_yaml(cls, path_or_text: str) -> "Config":
        import yaml
        text = open(path_or_text).read() if os.path.exists(path_or_text) else path_or_text
        return cls.from_dict(yaml.safe_load(text))

    def copy(self) -> "Config":
        mesh = self.__dict__.pop("_mesh", None)
        try:
            c = copy.deepcopy(self)
        finally:
            if mesh is not None:
                object.__setattr__(self, "_mesh", mesh)
        return c
