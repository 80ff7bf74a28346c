"""Row-sparse embedding bags (csrc/embedding.cu): the CTR models' ``embedding(is_sparse=True) + sequence_pool(avg)``
with a gradient that holds only the rows the batch looked up.

``embedding_bag_mean_sparse(table, ids, offsets=None)`` returns ``[B, D]`` mean-pooled bags.  Its table gradient is
an uncoalesced sparse COO tensor ``[V, D]`` with one row per looked-up element (indices ``[nnz]``, values
``[nnz, D]``), the same content ``nn.EmbeddingBag(mode="mean", sparse=True)`` produces.  A table used by several
bags in one step accumulates one contribution per use (autograd adds the sparse gradients).  ``ops.SparseAdam``
(ops/optim.py) consumes it.
"""
from __future__ import annotations

import torch


def sparse_rows(indices, values, shape):
    """Uncoalesced sparse COO gradient [V, D] from row indices [n] and rows [n, D], built without validating the
    indices (that would read them back to the host: every caller produces valid ids)."""
    with torch.sparse.check_sparse_tensor_invariants(enable=False):
        return torch.sparse_coo_tensor(indices.view(1, -1), values, tuple(shape), check_invariants=False)


def _flatten_bags(ids, offsets):
    """(flat ids [nnz], bag of every element [nnz], number of bags).  ``offsets`` None: ids is [B, L]."""
    if offsets is None:
        B, L = ids.shape
        flat = ids.reshape(-1)
        bag = torch.arange(flat.numel(), device=ids.device) // max(L, 1)
        return flat, bag, B
    B = offsets.numel()
    bag = torch.searchsorted(offsets, torch.arange(ids.numel(), device=ids.device), right=True) - 1
    return ids, bag, B


def _bag_sizes(bag, B):
    return torch.bincount(bag, minlength=B).to(torch.float32)


class _EmbBagSparseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, table, ids, offsets):
        B = ids.shape[0] if offsets is None else offsets.numel()
        if table.is_cuda:
            from . import native, count_launch

            out = torch.empty(B, table.shape[1], device=table.device, dtype=torch.float32)
            native().embedding_bag_mean_fwd(table, ids, offsets, out)
            count_launch()
        else:
            flat, bag, B = _flatten_bags(ids, offsets)
            out = torch.zeros(B, table.shape[1], dtype=torch.float32).index_add_(0, bag, table[flat])
            out = out / _bag_sizes(bag, B).clamp_min(1.0)[:, None]
        ctx.save_for_backward(ids, offsets)
        ctx.table_shape = table.shape
        return out

    @staticmethod
    def backward(ctx, dout):
        ids, offsets = ctx.saved_tensors
        V, D = ctx.table_shape
        dout = dout.contiguous().float()
        nnz = ids.numel()
        if dout.is_cuda:
            from . import native, count_launch

            indices = torch.empty(nnz, device=dout.device, dtype=torch.int64)
            values = torch.empty(nnz, D, device=dout.device, dtype=torch.float32)
            native().embedding_bag_mean_bwd_sparse(dout, ids, offsets, indices, values)
            count_launch()
        else:
            flat, bag, B = _flatten_bags(ids, offsets)
            indices = flat.clone()
            values = dout[bag] / _bag_sizes(bag, B)[bag][:, None]
        return sparse_rows(indices, values, (V, D)), None, None


def embedding_bag_mean_sparse(table, ids, offsets=None):
    """out[b] = mean over bag b of table[id] with a row-sparse table gradient.  table [V, D] fp32; ids [B, L] int64
    (fixed-length bags) or ids [nnz] int64 with ``offsets`` [B] int64 (bag starts, ``nn.EmbeddingBag``'s convention;
    an empty bag yields zeros)."""
    if table.dtype != torch.float32:
        raise TypeError("embedding_bag_mean_sparse: fp32 tables only, got %s" % table.dtype)
    ids = ids.contiguous()
    if offsets is not None:
        if ids.dim() != 1:
            raise ValueError("with offsets, ids must be 1-D [nnz]")
        offsets = offsets.contiguous()
    elif ids.dim() != 2:
        raise ValueError("without offsets, ids must be [B, L]")
    return _EmbBagSparseFn.apply(table, ids, offsets)


class _EmbBagsSparseFn(torch.autograd.Function):
    """S slots of fixed-length bags in one launch each way (CUDA only).  ``slot_table[s]``: index of slot s's table in
    ``tables``; a table used by several slots gets one gradient with the rows of all its slots."""

    @staticmethod
    def forward(ctx, ids, slot_table, *tables):
        from . import native, count_launch

        B, S, _ = ids.shape
        out = torch.empty(B, S, tables[0].shape[1], device=ids.device, dtype=torch.float32)
        native().embedding_bags_mean_fwd([tables[t] for t in slot_table], ids, out)
        count_launch()
        ctx.save_for_backward(ids)
        ctx.slot_table = slot_table
        ctx.table_shapes = [t.shape for t in tables]
        return out

    @staticmethod
    def backward(ctx, dout):
        from . import native, count_launch

        (ids,) = ctx.saved_tensors
        B, S, L = ids.shape
        D = dout.shape[2]
        indices = torch.empty(S, B * L, device=ids.device, dtype=torch.int64)
        values = torch.empty(S, B * L, D, device=ids.device, dtype=torch.float32)
        native().embedding_bags_mean_bwd_sparse(dout.contiguous().float(), ids, indices, values)
        count_launch()
        grads = []
        for t, shape in enumerate(ctx.table_shapes):
            slots = [s for s, u in enumerate(ctx.slot_table) if u == t]
            if len(slots) == 1:
                grads.append(sparse_rows(indices[slots[0]], values[slots[0]], shape))
            else:
                grads.append(sparse_rows(torch.cat([indices[s] for s in slots]),
                                         torch.cat([values[s] for s in slots]), shape))
        return (None, None, *grads)


def embedding_bags_mean_sparse(tables, ids):
    """One ``embedding_bag_mean_sparse`` per slot for fixed-length bags: ``tables[s]`` (fp32 [V, D], one entry per slot,
    the same table may repeat) pooled over ``ids[:, s]`` of ids [B, S, L] -> list of S [B, D] tensors.  On a GPU all
    slots (at most 64, of one width D) share one forward and one backward launch; gradients are the same row-sparse
    tensors as the per-slot op's."""
    if not ids.is_cuda or len(tables) > 64:
        return [embedding_bag_mean_sparse(t, ids[:, s]) for s, t in enumerate(tables)]
    uniq, slot_table = [], []
    for t in tables:
        for i, u in enumerate(uniq):
            if u is t:
                slot_table.append(i)
                break
        else:
            if t.dtype != torch.float32:
                raise TypeError("embedding_bags_mean_sparse: fp32 tables only, got %s" % t.dtype)
            slot_table.append(len(uniq))
            uniq.append(t)
    out = _EmbBagsSparseFn.apply(ids.contiguous(), tuple(slot_table), *uniq)
    return list(out.unbind(1))
