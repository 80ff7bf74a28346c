"""Flat parameter / gradient storage.

All parameters of one dtype are re-homed into ONE contiguous buffer (and their gradients into one
matching buffer, optionally carved out of NVSwitch-symmetric memory), so that

* the optimizer step is a single fused kernel per dtype (csrc/optim.cu) instead of the reference's
  one ``momentum`` op per tensor (167 for ResNet50_vd),
* gradient buckets are zero-copy slices of the flat gradient buffer (no flatten/unflatten copies as
  in Paddle's ``fuse_all_reduce_ops`` / DDP buckets), and
* elastic re-planning (new world size => new bucket/slice layout) never touches the model.

Layout order is *reverse registration order* (last layer first) so that the gradients that become
ready first during backward are contiguous at the start of the buffer -> bucket 0 can be reduced
while the rest of backward is still running.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import torch

ALIGN_ELEMS = 128  # every tensor starts on a 256-byte (bf16) / 512-byte (fp32) boundary


@dataclass
class FlatEntry:
    name: str
    param: torch.nn.Parameter
    offset: int
    numel: int
    order: int = 0   # global gradient-readiness order (0 = ready first)


@dataclass
class FlatGroup:
    dtype: torch.dtype
    entries: List[FlatEntry] = field(default_factory=list)
    numel: int = 0            # padded total
    param: torch.Tensor = None   # flat model-precision parameters (bf16 or fp32)
    grad: torch.Tensor = None    # flat gradients, same dtype
    master: Optional[torch.Tensor] = None  # fp32 master copy for low-precision groups


def _round_up(n: int, m: int) -> int:
    return (n + m - 1) // m * m


def is_sparse_param(p: torch.Tensor) -> bool:
    """A table whose gradient is row-sparse (``ops.embedding_bag_mean_sparse``; models mark it ``_edl_sparse``)."""
    return bool(getattr(p, "_edl_sparse", False))


class FlatParams:
    """Re-home ``module``'s trainable parameters into flat per-dtype buffers.

    ``grad_alloc(numel, dtype, device) -> Tensor`` lets the caller provide gradient storage (e.g.
    a slice of symmetric memory); ``pad_multiple`` pads each group so it can be split evenly across
    ranks by the two-shot all-reduce.

    Parameters marked ``_edl_sparse`` (row-sparse embedding tables, see ``is_sparse_param``) keep their own storage and
    sparse gradients: they are left out of the flat buffers."""

    def __init__(self, module: torch.nn.Module, grad_alloc: Optional[Callable] = None,
                 pad_multiple: int = 8 * 16 * 8, reverse: bool = True, direct_sinks: bool = True):
        named = [(n, p) for n, p in module.named_parameters() if p.requires_grad and not is_sparse_param(p)]
        if reverse:
            named = named[::-1]
        if not named:
            raise ValueError("module has no trainable parameters")
        self.device = named[0][1].device
        self.groups: Dict[torch.dtype, FlatGroup] = {}
        for order, (name, p) in enumerate(named):
            g = self.groups.setdefault(p.dtype, FlatGroup(dtype=p.dtype))
            off = _round_up(g.numel, ALIGN_ELEMS)
            g.entries.append(FlatEntry(name, p, off, p.numel(), order))
            g.numel = off + p.numel()
        for g in self.groups.values():
            g.numel = _round_up(g.numel, pad_multiple)
            g.param = torch.zeros(g.numel, dtype=g.dtype, device=self.device)
            if grad_alloc is not None:
                g.grad = grad_alloc(g.numel, g.dtype, self.device)
                g.grad.zero_()
            else:
                g.grad = torch.zeros(g.numel, dtype=g.dtype, device=self.device)
            for e in g.entries:
                view = g.param[e.offset:e.offset + e.numel].view(e.param.shape)
                with torch.no_grad():
                    view.copy_(e.param.data)
                e.param.data = view
                gview = g.grad[e.offset:e.offset + e.numel].view(e.param.shape)
                e.param.grad = gview
                if direct_sinks:
                    e.param._edl_grad_sink = gview
            if g.dtype != torch.float32:
                g.master = g.param.float()
        self.direct_sinks = direct_sinks

    # ------------------------------------------------------------------ helpers
    def zero_grad(self):
        """One memset per dtype group (gradients are accumulated in place by autograd / sinks)."""
        for g in self.groups.values():
            g.grad.zero_()
            for e in g.entries:
                if e.param.grad is None or e.param.grad.data_ptr() != g.grad.data_ptr() + \
                        e.offset * g.grad.element_size():
                    e.param.grad = g.grad[e.offset:e.offset + e.numel].view(e.param.shape)

    def rebind_grads(self, grad_alloc: Callable):
        """Move the gradient storage (e.g. into freshly rendezvoused symmetric memory after an
        elastic stage change).  Parameter values are untouched."""
        for g in self.groups.values():
            new = grad_alloc(g.numel, g.dtype, self.device)
            new.zero_()
            g.grad = new
            for e in g.entries:
                gview = g.grad[e.offset:e.offset + e.numel].view(e.param.shape)
                e.param.grad = gview
                if self.direct_sinks:
                    e.param._edl_grad_sink = gview

    def rebind_params(self, param_alloc: Callable, dtypes=None):
        """Move the flat model-precision parameters of the given dtype groups into storage provided by
        ``param_alloc(numel, dtype, device)`` (a window of symmetric memory: the fused reduce-scatter -> SGD ->
        all-gather kernel stores the new parameters into every rank's copy).  Values are carried over."""
        for dt, g in self.groups.items():
            if dtypes is not None and dt not in dtypes:
                continue
            new = param_alloc(g.numel, g.dtype, self.device)
            with torch.no_grad():
                new.copy_(g.param)
            g.param = new
            for e in g.entries:
                e.param.data = g.param[e.offset:e.offset + e.numel].view(e.param.shape)

    def sync_master_from_params(self):
        for g in self.groups.values():
            if g.master is not None:
                g.master.copy_(g.param.float())

    def total_numel(self) -> int:
        return sum(g.numel for g in self.groups.values())

    def entries(self):
        for g in self.groups.values():
            for e in g.entries:
                yield g, e

    def state_dict(self):
        return {str(dt): {"param": g.param, "master": g.master} for dt, g in self.groups.items()}
