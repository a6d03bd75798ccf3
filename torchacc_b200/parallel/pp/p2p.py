"""Point-to-point transport between adjacent pipeline stages (reference torchacc/dist/pp/p2p.py:7-37 and the
metadata handshake of pp/executor.py:475-570).

* asynchronous ``isend`` / ``irecv``; receives are *posted early* and waited for right before use, so transfers
  overlap the neighbouring micro-batch's compute (the reference blocks on every ``dist.send/recv``).  Activations and
  gradients use two separate process groups: NCCL runs the p2p operations of one communicator in issue order, so an
  early-posted receive in one direction must never queue in front of a send in the other;
* tensor metadata (dtype, shape, requires_grad) travels ONCE per shape epoch as a single fixed-size int64 header
  -- one host sync per epoch on the receiver instead of five ``.item()`` syncs per tensor (executor.py:528-561).
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

_DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.int64, torch.int32, torch.int16, torch.int8,
           torch.uint8, torch.bool, torch.float64]
_MAX_TENSORS, _MAX_DIMS = 16, 6
_FIELDS = 4                      # dtype id, ndim, requires_grad, group (index of the named value * 2 + member-of-a-tuple)
_HDR = 1 + _MAX_TENSORS * (_FIELDS + _MAX_DIMS)


class Meta:
    """``group``: which named boundary value the tensor belongs to; ``in_tuple``: the value is a tuple / list of tensors
    (e.g. the (cos, sin) pair an HF rotary-embedding module hands to every decoder layer) and this is one member."""
    __slots__ = ("shape", "dtype", "requires_grad", "group", "in_tuple")

    def __init__(self, shape, dtype, requires_grad, group=0, in_tuple=False):
        self.shape, self.dtype, self.requires_grad = tuple(shape), dtype, bool(requires_grad)
        self.group, self.in_tuple = int(group), bool(in_tuple)

    def __eq__(self, o):
        return (self.shape, self.dtype, self.requires_grad, self.group, self.in_tuple) == \
            (o.shape, o.dtype, o.requires_grad, o.group, o.in_tuple)


def flatten_values(values: Sequence) -> Tuple[List[torch.Tensor], List[Tuple[int, bool]]]:
    """Named boundary values (tensors, or one-level tuples / lists of tensors) -> flat tensor list + (group, in_tuple)."""
    flat, groups = [], []
    for g, v in enumerate(values):
        if isinstance(v, (tuple, list)):
            if not all(isinstance(t, torch.Tensor) for t in v):
                raise TypeError("only tensors and flat tuples / lists of tensors can cross a pipeline stage boundary")
            flat += list(v)
            groups += [(g, True)] * len(v)
        elif isinstance(v, torch.Tensor):
            flat.append(v)
            groups.append((g, False))
        else:
            raise TypeError(f"value of type {type(v).__name__} cannot cross a pipeline stage boundary")
    return flat, groups


def unflatten_values(tensors: Sequence[torch.Tensor], metas: Sequence[Meta]) -> List:
    """Inverse of ``flatten_values`` on the receiving stage."""
    out: List = []
    for t, m in zip(tensors, metas):
        if m.in_tuple:
            if len(out) == m.group:
                out.append([t])
            else:
                out[m.group].append(t)
        else:
            out.append(t)
    return [tuple(v) if isinstance(v, list) else v for v in out]


def encode_header(tensors: Sequence[torch.Tensor], device, groups: Optional[Sequence[Tuple[int, bool]]] = None) -> torch.Tensor:
    if len(tensors) > _MAX_TENSORS:
        raise ValueError(f"at most {_MAX_TENSORS} tensors per stage boundary")
    h = [len(tensors)]
    for i, t in enumerate(tensors):
        if t.dim() > _MAX_DIMS:
            raise ValueError(f"at most {_MAX_DIMS}-d tensors cross a stage boundary")
        g, tup = groups[i] if groups is not None else (i, False)
        h += [_DTYPES.index(t.dtype), t.dim(), int(t.requires_grad), 2 * g + int(tup)] + list(t.shape) + \
            [0] * (_MAX_DIMS - t.dim())
    h += [0] * (_HDR - len(h))
    return torch.tensor(h, dtype=torch.int64, device=device)


def decode_header(h: torch.Tensor) -> List[Meta]:
    v = h.tolist()          # the one host sync of a shape epoch
    out, p = [], 1
    for _ in range(v[0]):
        dt, nd, rg, grp = v[p], v[p + 1], v[p + 2], v[p + 3]
        out.append(Meta(v[p + _FIELDS:p + _FIELDS + nd], _DTYPES[dt], rg, grp // 2, grp % 2))
        p += _FIELDS + _MAX_DIMS
    return out


class StageLink:
    """Bidirectional link of one stage with its neighbours."""

    def __init__(self, mesh, device: torch.device):
        self.mesh, self.device = mesh, device
        self.group = mesh.get_pp_proc_group()                  # activations (and their headers): stage i -> i+1
        self.bwd_group = mesh.get_pp_bwd_proc_group() if hasattr(mesh, "get_pp_bwd_proc_group") else self.group
        # gradients travel on their own communicator (see Mesh._create_groups: NCCL p2p ordering)
        self.stage, self.stages = mesh.get_stage_id(), mesh.get_pp_num()
        self.prev = mesh.stage_to_global(self.stage - 1) if self.stage > 0 else None
        self.next = mesh.stage_to_global(self.stage + 1) if self.stage < self.stages - 1 else None
        self.recv_meta: Optional[List[Meta]] = None          # activations coming from prev
        self.sent_meta: Optional[List[Meta]] = None
        self._pending: List = []
        self.warm_up()

    def warm_up(self):
        """Create both communicators' p2p channels NOW, collectively (reference dist/__init__.py:68-81 warms its PP
        send/recv for the same reason).  NCCL creates a communicator / p2p channel at its first use with a host-side
        rendezvous of both peers; inside the 1F1B schedule the two stages reach their first gradient transfer at
        different points, and the stage that arrives first blocks on the host while its neighbour's device sits in an
        early-posted receive that only the blocked stage could satisfy.
        One tiny exchange per direction and communicator, in the same order on every stage, then a device sync."""
        if self.stages <= 1 or not (dist.is_available() and dist.is_initialized()):
            return
        t = torch.zeros(1, device=self.device)
        for group, down in ((self.group, True), (self.bwd_group, False)):
            # activations flow prev -> next on `group`, gradients next -> prev on `bwd_group`; even stages talk to
            # their successor first, odd stages to their predecessor, so every pair meets without a cyclic wait
            for phase in (0, 1):
                lower = self.stage if (self.stage % 2 == phase) else self.stage - 1     # pair (lower, lower + 1)
                if lower < 0 or lower + 1 >= self.stages:
                    continue
                src, dst = (lower, lower + 1) if down else (lower + 1, lower)
                if self.stage == src:
                    dist.send(t, self.mesh.stage_to_global(dst), group=group)
                else:
                    dist.recv(t, self.mesh.stage_to_global(src), group=group)
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)

    def reset_shapes(self):
        self.recv_meta = None
        self.sent_meta = None

    # ---- activations: prev -> me -> next ---------------------------------------------------------------------
    def send_activations(self, tensors: Sequence[torch.Tensor], groups: Optional[Sequence[Tuple[int, bool]]] = None):
        groups = list(groups) if groups is not None else [(i, False) for i in range(len(tensors))]
        metas = [Meta(t.shape, t.dtype, t.requires_grad, g, tup) for t, (g, tup) in zip(tensors, groups)]
        if self.sent_meta is None or self.sent_meta != metas:
            dist.send(encode_header(tensors, self.device, groups), self.next, group=self.group)
            self.sent_meta = metas
        works = [dist.isend(t.detach().contiguous(), self.next, group=self.group) for t in tensors]
        self._pending += works

    def post_recv_activations(self) -> Tuple[List[torch.Tensor], List]:
        if self.recv_meta is None:
            h = torch.empty(_HDR, dtype=torch.int64, device=self.device)
            dist.recv(h, self.prev, group=self.group)
            self.recv_meta = decode_header(h)
        bufs = [torch.empty(m.shape, dtype=m.dtype, device=self.device) for m in self.recv_meta]
        works = [dist.irecv(b, self.prev, group=self.group) for b in bufs]
        return bufs, works

    # ---- gradients: next -> me -> prev -----------------------------------------------------------------------
    def send_grads(self, grads: Sequence[Optional[torch.Tensor]], like: Sequence[torch.Tensor]):
        """One gradient per activation that was received with requires_grad (zeros when autograd produced none,
        reference executor.py:613-615)."""
        works = []
        for g, t, m in zip(grads, like, self.recv_meta):
            if not m.requires_grad:
                continue
            if g is None:
                g = torch.zeros_like(t)
            works.append(dist.isend(g.contiguous(), self.prev, group=self.bwd_group))
        self._pending += works

    def post_recv_grads(self) -> Tuple[List[Optional[torch.Tensor]], List]:
        bufs, works = [], []
        for m in self.sent_meta:
            if m.requires_grad:
                b = torch.empty(m.shape, dtype=m.dtype, device=self.device)
                works.append(dist.irecv(b, self.next, group=self.bwd_group))
                bufs.append(b)
            else:
                bufs.append(None)
        return bufs, works

    @staticmethod
    def wait(works):
        for w in works:
            w.wait()

    def flush(self):
        for w in self._pending:
            w.wait()
        self._pending = []
