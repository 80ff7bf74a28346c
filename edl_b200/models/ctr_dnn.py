"""CTR-DNN (Criteo click-through model) -- the reference's CTR example network:
26 sparse-slot embeddings ([1 000 001, 10] each, average-pooled per slot) + 13 dense features
-> concat(273) -> FC400 x3 (ReLU) -> FC2 -> softmax, trained with Adam 1e-4, AUC metric
(example/ctr/ctr/save_program.py:75-144, train.py:234).  The reference runs it CPU-only in
parameter-server mode; here it is an elastic data-parallel GPU model whose embedding gradients are
all-reduced densely (the BASELINE "embedding all-reduce bandwidth sweep" config) or, with ``sparse_grad=True``,
kept row-sparse like the reference's ``is_sparse=True`` tables: only the looked-up rows get a gradient, the
data-parallel engine all-gathers those rows and ``ops.SparseAdam`` updates only them."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F


class CtrDnn(nn.Module):
    def __init__(self, sparse_feature_dim=1000001, embedding_size=10, num_sparse=26, num_dense=13,
                 hidden=(400, 400, 400), shared_table=False, sparse_grad=False):
        super().__init__()
        self.num_sparse, self.num_dense = num_sparse, num_dense
        self.sparse_grad = sparse_grad
        n_tables = 1 if shared_table else num_sparse
        self.tables = nn.ModuleList([nn.EmbeddingBag(sparse_feature_dim, embedding_size, mode="mean", sparse=False)
                                     for _ in range(n_tables)])
        for t in self.tables:
            nn.init.uniform_(t.weight, -1.0 / math.sqrt(sparse_feature_dim), 1.0 / math.sqrt(sparse_feature_dim))
            if sparse_grad:
                t.weight._edl_sparse = True        # kept out of the flat buffers (parallel/flat.py)
        dims = [num_sparse * embedding_size + num_dense] + list(hidden)
        self.fcs = nn.ModuleList([nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])])
        for fc in self.fcs:
            nn.init.normal_(fc.weight, 0.0, 1.0 / math.sqrt(fc.in_features))
        self.out = nn.Linear(dims[-1], 2)

    def forward(self, dense, sparse_ids, sparse_offsets=None):
        """dense [B, 13] float; sparse_ids [B, 26, L] int64 (L ids per slot, average pooled) or, with
        ``sparse_offsets``, a list of 26 (ids, offsets) bags."""
        x = torch.cat(self.slot_embeddings(sparse_ids, sparse_offsets) + [dense], dim=1)
        for fc in self.fcs:
            x = F.relu(fc(x))
        return self.out(x)

    def slot_embeddings(self, sparse_ids, sparse_offsets=None):
        """One pooled [B, D] embedding per sparse slot.  Fixed-length bags on a GPU go through the
        hand-written embedding-bag kernels (csrc/misc.cu: gather-mean forward, scatter-add backward into
        a dense fp32 table gradient that elastic DP all-reduces like any other parameter).  With ``sparse_grad``
        every bag, fixed-length or CSR, on GPU or CPU, goes through ``ops.embedding_bag_mean_sparse``."""
        from ..ops import embedding_bag_mean

        if self.sparse_grad and sparse_offsets is None:
            return _sparse_bags(self.tables, self.num_sparse, sparse_ids)
        embs = []
        for s in range(self.num_sparse):
            table = self.tables[s % len(self.tables)]
            if self.sparse_grad:
                embs.append(_sparse_bag(table, s, sparse_ids, sparse_offsets))
            elif sparse_offsets is not None:
                embs.append(table(sparse_ids[s], sparse_offsets[s]))
            elif table.weight.is_cuda:
                embs.append(embedding_bag_mean(table.weight, sparse_ids[:, s]))
            else:
                embs.append(table(sparse_ids[:, s]))
        return embs


def _sparse_bags(tables, num_sparse, sparse_ids):
    """Every slot's fixed-length bags at once (one launch per direction on a GPU)."""
    from ..ops import embedding_bags_mean_sparse

    return embedding_bags_mean_sparse([tables[s % len(tables)].weight for s in range(num_sparse)], sparse_ids)


def _sparse_bag(table, s, sparse_ids, sparse_offsets):
    from ..ops import embedding_bag_mean_sparse

    if sparse_offsets is None:
        return embedding_bag_mean_sparse(table.weight, sparse_ids[:, s])
    return embedding_bag_mean_sparse(table.weight, sparse_ids[s], sparse_offsets[s])


class DeepFM(CtrDnn):
    """DeepFM on the same inputs (BASELINE.json names the CTR config "DeepFM"; the reference network is
    the plain CTR-DNN above, BASELINE.md "What is not published").  Shares the slot embeddings between
    the factorisation-machine part and the DNN:

        logit = w0 + sum_s w_s[id_s] + <dense, w_d>                    (first order)
              + 0.5 * sum_d ((sum_s e_s)^2 - sum_s e_s^2)_d            (second order, pairwise <e_i, e_j>)
              + DNN(concat(e_1..e_S, dense))                           (deep part, 1 output)

    Returns 2-class logits ``[0, logit]`` so that the loss / AUC code of the CTR-DNN example is unchanged."""

    def __init__(self, sparse_feature_dim=1000001, embedding_size=10, num_sparse=26, num_dense=13,
                 hidden=(400, 400, 400), shared_table=False, sparse_grad=False):
        super().__init__(sparse_feature_dim, embedding_size, num_sparse, num_dense, hidden, shared_table, sparse_grad)
        self.first_order = nn.ModuleList([nn.EmbeddingBag(sparse_feature_dim, 1, mode="mean", sparse=False)
                                          for _ in range(len(self.tables))])
        for t in self.first_order:
            nn.init.zeros_(t.weight)
            if sparse_grad:
                t.weight._edl_sparse = True
        self.dense_first = nn.Linear(num_dense, 1)
        self.out = nn.Linear(self.fcs[-1].out_features, 1)

    def forward(self, dense, sparse_ids, sparse_offsets=None):
        embs = self.slot_embeddings(sparse_ids, sparse_offsets)
        first = self.dense_first(dense)
        firsts = (_sparse_bags(self.first_order, self.num_sparse, sparse_ids)
                  if self.sparse_grad and sparse_offsets is None else None)
        for s in range(self.num_sparse):
            t = self.first_order[s % len(self.first_order)]
            if firsts is not None:
                first = first + firsts[s]
            elif self.sparse_grad:
                first = first + _sparse_bag(t, s, sparse_ids, sparse_offsets)
            else:
                first = first + (t(sparse_ids[:, s]) if sparse_offsets is None else t(sparse_ids[s], sparse_offsets[s]))
        e = torch.stack(embs, dim=1).float()                      # [B, S, D]
        second = 0.5 * (e.sum(1).pow(2) - e.pow(2).sum(1)).sum(1, keepdim=True)
        x = torch.cat(embs + [dense], dim=1)
        for fc in self.fcs:
            x = F.relu(fc(x))
        logit = first + second.to(first.dtype) + self.out(x)
        return torch.cat([torch.zeros_like(logit), logit], dim=1)


def auc(scores, labels, num_thresholds=4096):
    """Streaming-friendly AUC from score histograms (what the ``auc`` op of the reference computes)."""
    s = scores.detach().float().clamp(0, 1)
    idx = (s * (num_thresholds - 1)).long()
    pos = torch.zeros(num_thresholds, device=s.device).index_add_(0, idx, labels.float())
    neg = torch.zeros(num_thresholds, device=s.device).index_add_(0, idx, 1.0 - labels.float())
    tp = torch.flip(torch.cumsum(torch.flip(pos, [0]), 0), [0])
    fp = torch.flip(torch.cumsum(torch.flip(neg, [0]), 0), [0])
    tot_p, tot_n = pos.sum().clamp_min(1), neg.sum().clamp_min(1)
    tpr = torch.cat([tp / tot_p, tp.new_zeros(1)])
    fpr = torch.cat([fp / tot_n, fp.new_zeros(1)])
    return torch.trapz(torch.flip(tpr, [0]), torch.flip(fpr, [0]))
