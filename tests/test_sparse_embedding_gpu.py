"""Row-sparse embedding bags and lazy Adam on the H100 (csrc/embedding.cu) against nn.EmbeddingBag(sparse=True), the
plain-torch CPU path and FlatAdam."""
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models.ctr_dnn import CtrDnn, DeepFM
from edl_b200.parallel import ElasticDataParallel

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
BIG_V = 1000001


def _csr(B, V, max_len, gen, device="cpu"):
    lens = torch.randint(0, max_len + 1, (B,), generator=gen)
    lens[::7] = 0                                          # empty bags, including the first one
    ids = torch.randint(0, V, (int(lens.sum()),), generator=gen)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)[:-1]])
    return ids.to(device), offsets.to(device)


@pytest.mark.parametrize("D", [1, 10, 64])
@pytest.mark.parametrize("csr", [False, True])
def test_forward_and_gradient_match_embedding_bag(D, csr):
    gen = torch.Generator().manual_seed(D + csr)
    B = 1000
    ref = torch.nn.EmbeddingBag(BIG_V, D, mode="mean", sparse=True).to(DEV)
    table = ref.weight.detach().clone().requires_grad_(True)
    if csr:
        ids, offsets = _csr(B, BIG_V, 5, gen, DEV)
        want, got = ref(ids, offsets), ops.embedding_bag_mean_sparse(table, ids, offsets)
    else:
        ids = torch.randint(0, BIG_V, (B, 3), generator=gen).to(DEV)
        ids[:10, :] = 12345                                # repeated ids
        want, got = ref(ids), ops.embedding_bag_mean_sparse(table, ids)
    torch.testing.assert_close(got, want, atol=1e-6, rtol=1e-5)
    dout = torch.randn(B, D, generator=gen).to(DEV)
    want.backward(dout)
    got.backward(dout)
    g = table.grad
    assert g.is_sparse and g._nnz() == ids.numel() and g._values().shape == (ids.numel(), D)
    assert torch.equal(g._indices()[0], ids.reshape(-1))
    gc, rc = g.coalesce(), ref.weight.grad.coalesce()
    assert torch.equal(gc.indices(), rc.indices())
    torch.testing.assert_close(gc.values(), rc.values(), atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("D", [1, 10])
def test_all_slots_at_once_equal_one_slot_at_a_time(shared, D):
    gen = torch.Generator().manual_seed(9)
    S, B, L = 26, 1000, 2
    tables = [torch.nn.Parameter(torch.randn(BIG_V if shared else 5003, D).to(DEV)) for _ in range(1 if shared else S)]
    slots = [tables[s % len(tables)] for s in range(S)]
    ids = torch.randint(0, tables[0].shape[0], (B, S, L), generator=gen).to(DEV)
    dout = torch.randn(B, S, D, generator=gen).to(DEV)
    outs = ops.embedding_bags_mean_sparse(slots, ids)
    torch.stack(outs, 1).backward(dout)
    grads = [t.grad for t in tables]
    for t in tables:
        t.grad = None
    for s in range(S):
        ref = ops.embedding_bag_mean_sparse(slots[s], ids[:, s])
        assert torch.equal(outs[s], ref)
        ref.backward(dout[:, s])
    for g, t in zip(grads, tables):
        assert g.is_sparse and g._nnz() == t.grad._nnz() == B * L * (S if shared else 1)
        torch.testing.assert_close(g.coalesce().to_dense(), t.grad.coalesce().to_dense(), atol=1e-6, rtol=1e-5)


def _lazy_adam_run(device, V, D, steps, lr=1e-2):
    """SparseAdam over ``steps``: each a list of (ids, offsets or None, dout) bag sets looked up in ONE table (a table
    shared by several slots); returns table, m, v on the CPU."""
    torch.manual_seed(0)
    table = torch.nn.Parameter(torch.randn(V, D).to(device))
    opt = ops.SparseAdam([table], lr=lr)
    for bag_sets in steps:
        table.grad = None
        for ids, offs, dout in bag_sets:
            out = ops.embedding_bag_mean_sparse(table, ids.to(device), None if offs is None else offs.to(device))
            out.backward(dout.to(device))
        opt.step()
    return table.detach().cpu(), opt.state[0]["m"].cpu(), opt.state[0]["v"].cpu()


def _adam_steps(V, D, n_steps=6):
    gen = torch.Generator().manual_seed(7)
    steps = []
    for s in range(n_steps):
        fixed = torch.randint(0, 1000, (100000, 2), generator=gen)     # short runs of repeated ids
        fixed[:, 0] = 4242                                             # one id repeated 10^5 times
        ids, offs = _csr(3000, V, 4, gen)
        bag_sets = [(ids, offs, torch.randn(3000, D, generator=gen)),
                    (ids.flip(0).contiguous(), offs, torch.randn(3000, D, generator=gen))]
        if s % 2 == 0:
            bag_sets.append((fixed, None, torch.randn(100000, D, generator=gen)))
        steps.append(bag_sets)
    return steps


def test_sparse_adam_matches_cpu_reference():
    V, D = BIG_V, 10
    steps = _adam_steps(V, D)
    w, m, v = _lazy_adam_run(DEV, V, D, steps)
    w_ref, m_ref, v_ref = _lazy_adam_run("cpu", V, D, steps)
    torch.testing.assert_close(m, m_ref, atol=1e-5, rtol=1e-4)
    torch.testing.assert_close(v, v_ref, atol=1e-6, rtol=1e-4)
    torch.testing.assert_close(w, w_ref, atol=1e-5, rtol=1e-5)
    # rows outside every gradient: weights bitwise as initialised, m / v bitwise zero
    touched = torch.zeros(V, dtype=torch.bool)
    for bag_sets in steps:
        for ids, _, _ in bag_sets:
            touched[ids.reshape(-1)] = True
    torch.manual_seed(0)
    w0 = torch.randn(V, D)
    assert (~touched).sum() > V // 2
    assert torch.equal(w[~touched], w0[~touched])
    assert torch.equal(m[~touched], torch.zeros_like(m[~touched]))
    assert torch.equal(v[~touched], torch.zeros_like(v[~touched]))
    # deterministic: a second identical run is bitwise equal
    w2, m2, v2 = _lazy_adam_run(DEV, V, D, steps)
    assert torch.equal(w, w2) and torch.equal(m, m2) and torch.equal(v, v2)


def test_sparse_adam_many_tables_of_two_widths():
    """70 tables of width 3 (two launches of up to 64) and 5 of width 1, some without a gradient, against the CPU path."""
    shapes = [(200 + t, 3) for t in range(70)] + [(50, 1)] * 5
    runs = []
    for dev in ("cpu", DEV):
        torch.manual_seed(0)
        params = [torch.nn.Parameter(torch.randn(*s).to(dev)) for s in shapes]
        opt = ops.SparseAdam(params, lr=1e-2)
        g = torch.Generator().manual_seed(5)                           # the same gradients for both runs
        for _ in range(5):
            for t, p in enumerate(params):
                if t % 9 == 4:
                    p.grad = None
                    continue
                ids = torch.randint(0, p.shape[0], (40,), generator=g)
                vals = torch.randn(40, p.shape[1], generator=g)
                p.grad = torch.sparse_coo_tensor(ids[None], vals, p.shape).to(dev)
            opt.step()
        runs.append([torch.cat([p.detach().cpu().reshape(-1), st["m"].cpu().reshape(-1), st["v"].cpu().reshape(-1)])
                     for p, st in zip(params, opt.state)])
    for a, b in zip(*runs):
        torch.testing.assert_close(b, a, atol=1e-5, rtol=1e-4)


def test_untouched_rows_bitwise_unchanged_between_steps():
    V, D = BIG_V, 10
    torch.manual_seed(1)
    table = torch.nn.Parameter(torch.randn(V, D, device=DEV))
    opt = ops.SparseAdam([table], lr=1e-2)
    for s in range(5):
        ids = torch.randint(0, V, (1000, 26), device=DEV)
        w0, m0, v0 = table.detach().clone(), opt.state[0]["m"].clone(), opt.state[0]["v"].clone()
        table.grad = None
        ops.embedding_bag_mean_sparse(table, ids).sum().backward()
        opt.step()
        keep = torch.ones(V, dtype=torch.bool, device=DEV)
        keep[ids.reshape(-1)] = False
        assert torch.equal(table[keep], w0[keep])
        assert torch.equal(opt.state[0]["m"][keep], m0[keep]) and torch.equal(opt.state[0]["v"][keep], v0[keep])
        assert not torch.equal(table[~keep], w0[~keep])


def test_every_row_touched_reproduces_flat_adam():
    from edl_b200.parallel import FlatParams

    V, D = 4096, 10
    torch.manual_seed(2)
    dense = torch.nn.Parameter(torch.randn(V, D, device=DEV))
    sparse = torch.nn.Parameter(dense.detach().clone())
    flat = FlatParams(torch.nn.ParameterList([dense]))
    fa, sa = ops.FlatAdam(flat, lr=1e-2), ops.SparseAdam([sparse], lr=1e-2)
    for _ in range(6):
        ids = torch.cat([torch.randperm(V, device=DEV), torch.randint(0, V, (V,), device=DEV)]).view(-1, 2)
        dout = torch.randn(ids.shape[0], D, device=DEV)
        flat.zero_grad()
        sparse.grad = None
        ops.embedding_bag_mean_sparse(sparse, ids).backward(dout)
        dense.grad.copy_(sparse.grad.coalesce().to_dense())
        fa.step()
        sa.step()
    torch.testing.assert_close(sparse.detach(), dense.detach(), atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(sa.state[0]["v"], fa.state[torch.float32]["v"][:V * D].view(V, D), atol=1e-7, rtol=1e-4)


def test_no_host_sync_in_forward_backward_step():
    V, D = BIG_V, 10
    table = torch.nn.Parameter(torch.randn(V, D, device=DEV))
    first = torch.nn.Parameter(torch.zeros(V, 1, device=DEV))
    opt = ops.SparseAdam([table, first], lr=1e-3)
    gen = torch.Generator().manual_seed(3)
    ids, offsets = _csr(1000, V, 3, gen, DEV)
    fixed = torch.randint(0, V, (1000, 1), generator=gen).to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for _ in range(2):
            table.grad = first.grad = None
            y = ops.embedding_bag_mean_sparse(table, ids, offsets).sum(1)
            y = y + ops.embedding_bag_mean_sparse(table, fixed).sum(1)            # shared table
            y = y + ops.embedding_bag_mean_sparse(first, fixed)[:, 0]
            y.sum().backward()
            opt.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(table).all()


@pytest.mark.parametrize("cls", [CtrDnn, DeepFM])
@pytest.mark.parametrize("csr", [False, True])
def test_sparse_model_in_data_parallel_matches_cpu(cls, csr):
    kw = dict(sparse_feature_dim=5003, embedding_size=10, num_sparse=26, num_dense=13, hidden=(64, 64),
              sparse_grad=True)
    torch.manual_seed(0)
    cpu_model = cls(**kw)
    if cls is DeepFM:
        for t in cpu_model.first_order:
            torch.nn.init.normal_(t.weight, 0.0, 0.01)
    gpu_model = cls(**kw)
    gpu_model.load_state_dict(cpu_model.state_dict())
    gpu_model = gpu_model.to(DEV)
    runs = []
    gen = torch.Generator().manual_seed(11)
    batches = []
    for _ in range(3):
        x = torch.rand(256, 13, generator=gen)
        y = torch.randint(0, 2, (256,), generator=gen)
        if csr:
            bags = [_csr(256, 5003, 3, gen) for _ in range(26)]
            batches.append((x, [b[0] for b in bags], [b[1] for b in bags], y))
        else:
            batches.append((x, torch.randint(0, 5003, (256, 26, 2), generator=gen), None, y))
    for model, dev in ((cpu_model, torch.device("cpu")), (gpu_model, DEV)):
        dp = ElasticDataParallel(model)
        assert len(dp.sparse_params) == (52 if cls is DeepFM else 26)
        assert not [e.name for _, e in dp.flat.entries() if "tables" in e.name or "first_order" in e.name]
        fa, sa = ops.FlatAdam(dp.flat, lr=1e-4), ops.SparseAdam(dp.sparse_params, lr=1e-4)
        losses = []
        for x, ids, offs, y in batches:
            ids_d = [i.to(dev) for i in ids] if csr else ids.to(dev)
            offs_d = [o.to(dev) for o in offs] if csr else None
            dp.zero_grad()
            loss = F.cross_entropy(dp(x.to(dev), ids_d, offs_d), y.to(dev))
            loss.backward()
            dp.finish()
            fa.step()
            sa.step()
            losses.append(float(loss))
        runs.append((losses, {k: v.detach().cpu() for k, v in model.state_dict().items()}))
    (l_cpu, sd_cpu), (l_gpu, sd_gpu) = runs
    assert l_gpu == pytest.approx(l_cpu, rel=1e-4, abs=1e-5)
    for k in sd_cpu:
        torch.testing.assert_close(sd_gpu[k], sd_cpu[k], atol=1e-3 if "fcs" in k or "out" in k else 3e-4, rtol=1e-3)
