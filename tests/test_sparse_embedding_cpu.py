"""Row-sparse embedding bags and lazy Adam on CPU: the plain-torch path of ``ops.embedding_bag_mean_sparse`` against
``nn.EmbeddingBag(sparse=True)``, ``ops.SparseAdam`` against FlatAdam, and a 2-rank gloo run of the sparse CTR model
whose replicas must stay bitwise equal and match one process on the concatenated batch."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models.ctr_dnn import CtrDnn, DeepFM
from edl_b200.parallel import ElasticDataParallel, FlatParams


def _csr(B, V, max_len, gen):
    lens = torch.randint(0, max_len + 1, (B,), generator=gen)
    lens[0] = 0                                            # at least one empty bag
    ids = torch.randint(0, V, (int(lens.sum()),), generator=gen)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)[:-1]])
    return ids, offsets


@pytest.mark.parametrize("D", [1, 10])
@pytest.mark.parametrize("csr", [False, True])
def test_cpu_path_matches_embedding_bag(D, csr):
    gen = torch.Generator().manual_seed(D)
    V, B = 37, 9
    ref = torch.nn.EmbeddingBag(V, D, mode="mean", sparse=True)
    table = ref.weight.detach().clone().requires_grad_(True)
    if csr:
        ids, offsets = _csr(B, V, 4, gen)
        want = ref(ids, offsets)
        got = ops.embedding_bag_mean_sparse(table, ids, offsets)
    else:
        ids, offsets = torch.randint(0, V, (B, 3), generator=gen), None
        want = ref(ids)
        got = ops.embedding_bag_mean_sparse(table, ids)
    assert torch.allclose(got, want, atol=1e-6)
    dout = torch.randn(B, D, generator=gen)
    want.backward(dout)
    got.backward(dout)
    g = table.grad
    assert g.is_sparse and g._indices().shape[1] == ids.numel() and g._values().shape == (ids.numel(), D)
    assert torch.equal(g._indices()[0], ids.reshape(-1))
    assert torch.allclose(g.coalesce().to_dense(), ref.weight.grad.coalesce().to_dense(), atol=1e-6)


def test_shared_table_accumulates_one_contribution_per_use():
    torch.manual_seed(0)
    kw = dict(sparse_feature_dim=20, embedding_size=4, num_sparse=3, num_dense=2, hidden=(8,), shared_table=True)
    m, ref = CtrDnn(sparse_grad=True, **kw), CtrDnn(**kw)
    ref.load_state_dict(m.state_dict())
    ids, x = torch.randint(0, 20, (5, 3, 2)), torch.rand(5, 2)
    m(x, ids).sum().backward()
    ref(x, ids).sum().backward()
    g = m.tables[0].weight.grad
    assert g.is_sparse
    assert torch.allclose(g.coalesce().to_dense(), ref.tables[0].weight.grad, atol=1e-6)


def test_sparse_adam_matches_flat_adam_when_every_row_is_touched():
    torch.manual_seed(0)
    V, D = 16, 3
    dense = torch.nn.Parameter(torch.randn(V, D))
    sparse = torch.nn.Parameter(dense.detach().clone())
    flat = FlatParams(torch.nn.ParameterList([dense]))
    fa = ops.FlatAdam(flat, lr=1e-2)
    sa = ops.SparseAdam([sparse], lr=1e-2)
    for _ in range(5):
        ids = torch.cat([torch.randperm(V), torch.randint(0, V, (7,))])
        vals = torch.randn(ids.numel(), D)
        g = torch.sparse_coo_tensor(ids[None], vals, (V, D))
        flat.zero_grad()
        dense.grad.copy_(g.to_dense())
        sparse.grad = g
        fa.step()
        sa.step()
    assert torch.allclose(sparse, dense, atol=1e-6)
    assert torch.allclose(sa.state[0]["m"], fa.state[torch.float32]["m"][:V * D].view(V, D), atol=1e-6)


def test_sparse_adam_leaves_other_rows_untouched():
    torch.manual_seed(0)
    p = torch.nn.Parameter(torch.randn(50, 4))
    opt = ops.SparseAdam([p], lr=1e-2)
    touched = torch.tensor([3, 7, 7, 41])
    for _ in range(3):
        w0 = p.detach().clone()
        m0, v0 = opt.state[0]["m"].clone(), opt.state[0]["v"].clone()
        p.grad = torch.sparse_coo_tensor(touched[None], torch.randn(4, 4), (50, 4))
        opt.step()
        keep = torch.ones(50, dtype=torch.bool)
        keep[touched] = False
        assert torch.equal(p[keep], w0[keep])
        assert torch.equal(opt.state[0]["m"][keep], m0[keep]) and torch.equal(opt.state[0]["v"][keep], v0[keep])
        assert not torch.equal(p[~keep], w0[~keep])
    sd = opt.state_dict()
    opt2 = ops.SparseAdam([torch.nn.Parameter(p.detach().clone())], lr=1.0)
    opt2.load_state_dict(sd)
    assert opt2.lr == opt.lr and torch.equal(opt2.step_t, opt.step_t)
    assert torch.equal(opt2.state[0]["v"], opt.state[0]["v"])


def test_first_sparse_step_equals_dense_step():
    """On the first step the dense Adam moves no row that has a zero gradient, so both paths agree."""
    torch.manual_seed(0)
    kw = dict(sparse_feature_dim=30, embedding_size=4, num_sparse=3, num_dense=2, hidden=(8,))
    dense, sparse = DeepFM(**kw), DeepFM(sparse_grad=True, **kw)
    sparse.load_state_dict(dense.state_dict())
    for t in sparse.first_order:
        torch.nn.init.normal_(t.weight)
    dense.load_state_dict(sparse.state_dict())
    x, ids = torch.rand(6, 2), torch.randint(0, 30, (6, 3, 2))
    y = torch.randint(0, 2, (6,))
    dp_d, dp_s = ElasticDataParallel(dense), ElasticDataParallel(sparse)
    assert len(dp_s.sparse_params) == 6 and not dp_d.sparse_params
    assert not [e.name for _, e in dp_s.flat.entries() if "tables" in e.name or "first_order" in e.name]
    assert dp_s.flat.total_numel() < dp_d.flat.total_numel()
    opt_d = ops.FlatAdam(dp_d.flat, lr=1e-2)
    opt_s, opt_t = ops.FlatAdam(dp_s.flat, lr=1e-2), ops.SparseAdam(dp_s.sparse_params, lr=1e-2)
    for dp, opts, model in ((dp_d, [opt_d], dense), (dp_s, [opt_s, opt_t], sparse)):
        dp.zero_grad()
        F.cross_entropy(dp(x, ids), y).backward()
        dp.finish()
        for o in opts:
            o.step()
    for (n, a), (_, b) in zip(dense.named_parameters(), sparse.named_parameters()):
        assert torch.allclose(a, b, atol=1e-6), n


# ---------------------------------------------------------------------------------------------- 2 ranks, gloo
V, S, D, B, STEPS = 40, 3, 4, 6, 4


def _batches(rank, step):
    gen = torch.Generator().manual_seed(1000 * rank + step)
    ids, offs = zip(*[_csr(B, V, 2 + rank, gen) for _ in range(S)])   # rank 1 has longer bags: different nnz
    return torch.rand(B, 2, generator=gen), list(ids), list(offs), torch.randint(0, 2, (B,), generator=gen)


def _model():
    torch.manual_seed(0)
    m = DeepFM(sparse_feature_dim=V, embedding_size=D, num_sparse=S, num_dense=2, hidden=(8,), sparse_grad=True)
    for t in m.first_order:
        torch.nn.init.normal_(t.weight, 0.0, 0.1)
    return m


def _train(dp, batches):
    dense_opt = ops.FlatAdam(dp.flat, lr=1e-2)
    sparse_opt = ops.SparseAdam(dp.sparse_params, lr=1e-2)
    for x, ids, offs, y in batches:
        dp.zero_grad()
        F.cross_entropy(dp(x, ids, offs), y).backward()
        dp.finish()
        dense_opt.step()
        sparse_opt.step()
    return sparse_opt


def _state(model, sparse_opt):
    tabs = torch.cat([p.detach().reshape(-1) for p in sparse_opt.params])
    mv = torch.cat([t.reshape(-1) for st in sparse_opt.state for t in (st["m"], st["v"])])
    rest = torch.cat([p.detach().reshape(-1) for n, p in model.named_parameters() if "tables" not in n
                      and "first_order" not in n])
    return tabs, mv, rest


def _gloo_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    model = _model()
    dp = ElasticDataParallel(model)
    if rank == 1:
        with torch.no_grad():
            for p in dp.sparse_params:
                p.add_(1.0)                                  # broadcast_parameters() must undo this
    dp.broadcast_parameters()
    opt = _train(dp, [_batches(rank, s) for s in range(STEPS)])
    nnz = [p.grad._nnz() for p in dp.sparse_params]
    # numpy arrays travel by value: shared-memory tensors would need this process alive until the parent reads them
    q.put((rank, [t.numpy().copy() for t in _state(model, opt)], dp.last_sparse_bytes, nnz))
    dist.destroy_process_group()


def test_gloo_two_ranks_sparse_tables_bitwise_equal():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 777) % 2000
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r, (st, nbytes, nnz)) for r, st, nbytes, nnz in (q.get(timeout=240) for _ in range(2)))
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    (s0, b0, nnz0), (s1, b1, nnz1) = res[0], res[1]
    s0, s1 = [torch.from_numpy(a) for a in s0], [torch.from_numpy(a) for a in s1]
    for a, b in zip(s0, s1):
        assert torch.equal(a, b)                                     # replicas bitwise identical
    assert b0 != b1                                                  # the ranks sent different nnz
    assert nnz0 == nnz1
    # one process on the concatenated batch of both ranks
    model = _model()
    dp = ElasticDataParallel(model)
    batches = []
    for s in range(STEPS):
        x0, i0, o0, y0 = _batches(0, s)
        x1, i1, o1, y1 = _batches(1, s)
        batches.append((torch.cat([x0, x1]), [torch.cat([a, b]) for a, b in zip(i0, i1)],
                        [torch.cat([oa, ob + ia.numel()]) for oa, ob, ia in zip(o0, o1, i0)], torch.cat([y0, y1])))
    opt = _train(dp, batches)
    for a, b in zip(s0, _state(model, opt)):
        assert torch.allclose(a, b, atol=2e-5, rtol=1e-4)
