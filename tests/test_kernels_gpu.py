"""Numerics of every hand-written sm_90a kernel against a plain PyTorch reference (float64 element-wise bounds of
tests/f64_bounds.py for BatchNorm and pooling)."""
import pytest
import torch
import torch.nn.functional as F

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.ops import bn as bnmod

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize("shape", [(4, 32, 28, 28), (2, 64, 56, 56), (3, 256, 14, 14), (2, 2048, 7, 7),
                                   (1, 1000 // 8 * 8, 5, 5), (32, 128, 28, 28), (16, 64, 112, 112)])
@pytest.mark.parametrize("relu,res", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("path", ["fused", "stream", "regs"])
def test_bn_fwd_bwd(shape, relu, res, path):
    """path: SM-resident fused kernels / cp.async.bulk streaming kernels / register kernels."""
    ops.set_fused_bn(path == "fused")
    ops.native().bn_set_stream_kernels(path != "regs")
    try:
        _bn_fwd_bwd(shape, relu, res)
    finally:
        ops.set_fused_bn(False)
        ops.native().bn_set_stream_kernels(True)


def _bn_fwd_bwd(shape, relu, res):
    torch.manual_seed(0)
    n, c, h, w = shape
    m = n * h * w
    x = _cl((torch.randn(shape, device=DEV) * 2 + 0.5).bfloat16()).requires_grad_(True)
    r = _cl(torch.randn(shape, device=DEV).bfloat16()).requires_grad_(True) if res else None
    gamma = (torch.rand(c, device=DEV) + 0.5).requires_grad_(True)
    beta = (torch.randn(c, device=DEV) * 0.1).requires_grad_(True)
    rm, rv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    y = ops.batch_norm_act(x, gamma, beta, rm, rv, residual=r, relu=relu, training=True)
    _, _, _, mean, rstd, _ = y.grad_fn.saved_tensors      # the saved statistics, read before backward frees them
    dy = _cl(torch.randn(shape, device=DEV).bfloat16())
    y.backward(dy)
    # float64 BatchNorm with the exact statistics of the bf16 input; the ReLU mask of the stored output, like the kernels
    ex = fb.bn_exact(x.detach(), gamma.detach(), beta.detach(), 1e-5, r.detach() if res else None, relu,
                     y=y.detach(), dy=dy)
    what = "bn %s relu %d res %d" % (shape, relu, res)
    # the saved statistics: within the bound propagated from the reductions' rounding of any of the three paths
    tau_s = max(fb.bn_reduce_tau(p, m, c) for p in ("regs", "stream", "fused"))
    fb.check_bn_stats_e2e(x.detach(), mean, rstd, 1e-5, tau_s, what=what)
    if m >= fb.E2E_MIN_ROWS:
        fb.check_bf16(y.detach(), *ex["y"], criteria=(2,), what=what + " y")
        fb.check_bf16(x.grad, *ex["dx"], criteria=(2,), what=what + " dx")
    else:
        # too few rows per channel for criterion 2: criterion 1 from the saved statistics, with the float64 dsums
        # standing in for the kernel's (their error bound folded into dx's slack)
        xd, yd = fb.rows(x.detach()), fb.rows(y.detach())
        keep = yd > 0 if relu else None
        fb.check_bf16(y.detach(), *fb.bn_y_ref(xd, mean, rstd, gamma.detach(), beta.detach(),
                                               fb.rows(r.detach()) if res else None, relu),
                      tau=fb.BN_Y_TAU, criteria=(1,), what=what + " y")
        ds, ds_mag, _ = fb.bn_dsums_ref(fb.rows(dy), xd, mean, rstd, gamma, beta, relu, y=yd if relu else None)
        fb.check_bf16(x.grad, *fb.bn_dx_ref(fb.rows(dy), xd, mean, rstd, gamma.detach(), ds, m, keep,
                                           dsums_err=tau_s * ds_mag), tau=fb.BN_DX_TAU, criteria=(1,), what=what + " dx")
    for name, got in (("dgamma", gamma.grad), ("dbeta", beta.grad)):
        # the exact statistics differ from the kernel's by their fp32 rounding, far below 2^-12 of the sum of |terms|
        fb.check_sums(got, *ex[name], m, tau_s=2 ** -12, what=what + " " + name)
    if res:
        fb.check_exact(r.grad, fb.rows(ex["dres"][0]).reshape(n, h, w, c).permute(0, 3, 1, 2), what=what + " dres")
    mu, var, _, _ = fb.bn_exact_stats(x.detach())
    rm_ref, rv_ref = 0.1 * mu, 0.9 + 0.1 * var * (m / (m - 1))
    fb.check_sums(rm, rm_ref, rm_ref.abs(), m, tau_s=2 ** -12, what=what + " running mean")
    fb.check_sums(rv, rv_ref, rv_ref.abs(), m, tau_s=2 ** -12, what=what + " running var")


def test_bn_sinks_and_eval():
    torch.manual_seed(0)
    m = bnmod.BatchNormAct2d(64, relu=True).to(DEV)
    x = _cl(torch.randn(4, 64, 8, 8, device=DEV).bfloat16()).requires_grad_(True)
    sg, sb = torch.zeros(64, device=DEV), torch.zeros(64, device=DEV)
    m.weight._edl_grad_sink, m.bias._edl_grad_sink = sg, sb
    y = m(x)
    y.float().sum().backward()
    assert m.weight.grad is None and sg.abs().sum() > 0
    m.eval()
    ye = m(x.detach())
    scale = m.weight * torch.rsqrt(m.running_var + m.eps)
    ref = torch.relu(x.detach().float() * scale[None, :, None, None]
                     + (m.bias - m.running_mean * scale)[None, :, None, None])
    assert _rel(ye, ref) < 1e-2


@pytest.mark.parametrize("kind", ["probs", "logits", "labels"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_soft_ce(kind, dtype):
    torch.manual_seed(0)
    n, c = 32, 1000
    z = (torch.randn(n, c, device=DEV) * 3).to(dtype).requires_grad_(True)
    if kind == "probs":
        t = torch.softmax(torch.randn(n, c, device=DEV) * 2, -1).to(dtype)
    elif kind == "logits":
        t = (torch.randn(n, c, device=DEV) * 2).to(dtype)
    else:
        t = torch.randint(0, c, (n,), device=DEV)
    loss = ops.soft_cross_entropy(z, t, target_kind=kind, student_temperature=1.0, teacher_temperature=2.0)
    loss.backward()
    zr = z.detach().float().requires_grad_(True)
    ref = ops.loss._ref_loss(zr, t, {"probs": 0, "logits": 1, "labels": 2}[kind], 1.0, 2.0, 0.0, False, 1.0)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 2e-3 * max(1.0, abs(ref.item()))
    assert _rel(z.grad, zr.grad) < (2e-2 if dtype == torch.bfloat16 else 1e-4)


def test_kl_temperature_and_smoothing():
    torch.manual_seed(1)
    z = (torch.randn(16, 100, device=DEV)).requires_grad_(True)
    t = torch.randn(16, 100, device=DEV)
    loss = ops.soft_cross_entropy(z, t, "logits", 2.0, 2.0, kl=True, loss_scale=4.0)
    ref = F.kl_div(F.log_softmax(z.detach() / 2, -1), F.softmax(t / 2, -1), reduction="batchmean") * 4.0
    assert abs(loss.item() - ref.item()) < 1e-4
    lab = torch.randint(0, 100, (16,), device=DEV)
    l2 = ops.soft_cross_entropy(z, lab, "labels", label_smoothing=0.1)
    r2 = F.cross_entropy(z.detach(), lab, label_smoothing=0.1)
    assert abs(l2.item() - r2.item()) < 1e-4


def test_topk():
    torch.manual_seed(0)
    z = torch.randn(64, 1000, device=DEV).bfloat16()
    lab = torch.randint(0, 1000, (64,), device=DEV)
    z[torch.arange(0, 64, 2), lab[::2]] = 50.0
    got = ops.topk_accuracy(z, lab).cpu()
    ref = ops.topk_accuracy(z.cpu().float(), lab.cpu())
    assert torch.allclose(got, ref)


@pytest.mark.parametrize("shape", [(2, 64, 112, 112), (3, 32, 17, 19)])
def test_maxpool(shape):
    torch.manual_seed(0)
    x = _cl(torch.randn(shape, device=DEV).bfloat16()).requires_grad_(True)
    y = ops.max_pool_3x3_s2(x)
    dy = _cl(torch.randn_like(y))
    y.backward(dy)
    ref, idx = fb.maxpool_ref(x.detach())
    fb.check_exact(y.detach().double(), ref, what="maxpool y")
    fb.check_bf16(x.grad, *fb.maxpool_bwd_ref(dy, idx, shape), tau=3 * fb.EPS32, what="maxpool dx")


@pytest.mark.parametrize("shape", [(2, 256, 56, 56), (2, 64, 7, 9)])
def test_avgpool_gap(shape):
    torch.manual_seed(0)
    x = _cl(torch.randn(shape, device=DEV).bfloat16()).requires_grad_(True)
    y = ops.avg_pool_2x2(x)
    dy = _cl(torch.randn_like(y))
    y.backward(dy)
    fb.check_bf16(y.detach(), *fb.avgpool_ref(x.detach()), tau=3 * fb.EPS32, what="avgpool y")
    fb.check_bf16(x.grad, *fb.avgpool_bwd_ref(dy, shape), tau=fb.EPS32, what="avgpool dx")
    x2 = _cl(torch.randn(shape, device=DEV).bfloat16()).requires_grad_(True)
    g = ops.global_avg_pool(x2)
    dg = torch.randn_like(g)
    g.backward(dg)
    fb.check_bf16(g.detach(), *fb.gap_ref(x2.detach()), tau=fb.gap_tau(shape[2] * shape[3]), what="gap y")
    fb.check_bf16(x2.grad, *fb.gap_bwd_ref(dg, shape), tau=2 * fb.EPS32, what="gap dx")


def test_fused_sgd_matches_reference():
    torch.manual_seed(0)
    from edl_b200.parallel import FlatParams

    lin = torch.nn.Sequential(torch.nn.Linear(300, 257), torch.nn.Linear(257, 10)).to(DEV)
    lin[0].weight.data = lin[0].weight.data.bfloat16()
    lin[1].weight.data = lin[1].weight.data.bfloat16()
    ref_master = [p.detach().float().clone() for p in lin.parameters()]
    flat = FlatParams(lin)
    opt = ops.FlatSGDMomentum(flat, lr=0.1, momentum=0.9, weight_decay=1e-2)
    mom = [torch.zeros_like(m) for m in ref_master]
    for it in range(3):
        flat.zero_grad()
        grads = []
        for p in lin.parameters():
            g = torch.randn_like(p.float()).to(p.dtype)
            p.grad.copy_(g)
            grads.append(g.float())
        opt.step()
        for i, (m, g) in enumerate(zip(ref_master, grads)):
            gg = g + 1e-2 * m
            mom[i] = 0.9 * mom[i] + gg
            ref_master[i] = m - 0.1 * mom[i]
    for p, m in zip(lin.parameters(), ref_master):
        tol = 1e-2 if p.dtype == torch.bfloat16 else 1e-5
        assert _rel(p, m) < tol


def test_fused_adam():
    torch.manual_seed(0)
    from edl_b200.parallel import FlatParams

    lin = torch.nn.Linear(64, 33).to(DEV)
    ref = torch.nn.Linear(64, 33).to(DEV)
    ref.load_state_dict(lin.state_dict())
    flat = FlatParams(lin)
    opt = ops.FlatAdam(flat, lr=1e-2, weight_decay=0.01, decoupled=True)
    ropt = torch.optim.AdamW(ref.parameters(), lr=1e-2, weight_decay=0.01)
    for _ in range(4):
        flat.zero_grad()
        for p, q in zip(lin.parameters(), ref.parameters()):
            g = torch.randn_like(p)
            p.grad.copy_(g)
            q.grad = g.clone()
        opt.step()
        ropt.step()
    for p, q in zip(lin.parameters(), ref.parameters()):
        assert _rel(p, q) < 1e-4


def test_rope_fwd_bwd():
    torch.manual_seed(0)
    t, h, d = 77, 8, 64
    cos, sin = ops.rope_tables(t, d, device=DEV)
    x = torch.randn(t, h, d, device=DEV).bfloat16().requires_grad_(True)
    y = ops.rope(x, cos, sin)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    yr = ops.misc._rope_ref(xr, cos, sin)
    yr.backward(dy.float())
    assert _rel(y, yr) < 1e-2 and _rel(x.grad, xr.grad) < 1e-2
    # rotation preserves the norm of every (x1_j, x2_j) pair
    assert abs(y.float().norm().item() - x.float().norm().item()) / x.float().norm().item() < 1e-2


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_embedding_bag(dtype):
    torch.manual_seed(0)
    table = torch.randn(5000, 10, device=DEV).to(dtype).requires_grad_(True)
    ids = torch.randint(0, 5000, (1000, 3), device=DEV)
    out = ops.embedding_bag_mean(table, ids)
    g = torch.randn_like(out)
    out.backward(g)
    tr = table.detach().float().requires_grad_(True)
    ref = tr[ids].mean(1)
    ref.backward(g.float())
    assert _rel(out, ref) < 1e-2 and _rel(table.grad, tr.grad) < 2e-2


@pytest.mark.parametrize("cls", ["CtrDnn", "DeepFM"])
def test_ctr_models_use_native_embedding_bag(cls):
    """The CTR networks on a GPU (own gather-mean / scatter-add kernels) against the same weights on the CPU."""
    import copy

    from edl_b200.models import ctr_dnn

    torch.manual_seed(0)
    cpu = getattr(ctr_dnn, cls)(sparse_feature_dim=997, embedding_size=10, num_sparse=6, hidden=(32, 32))
    gpu = copy.deepcopy(cpu).to(DEV)
    dense = torch.rand(64, 13)
    ids = torch.randint(0, 997, (64, 6, 2))
    ops.reset_launches()
    out = gpu(dense.to(DEV), ids.to(DEV))
    assert ops.launches() >= 6, "embedding-bag kernels were not launched"
    ref = cpu(dense, ids)
    assert _rel(out.cpu(), ref) < 1e-3
    out[:, 1].sum().backward()
    ref[:, 1].sum().backward()
    for a, b in zip(gpu.tables, cpu.tables):
        assert _rel(a.weight.grad.cpu(), b.weight.grad) < 1e-3


def test_normalize_u8():
    torch.manual_seed(0)
    x = torch.randint(0, 256, (4, 20, 24, 3), device=DEV, dtype=torch.uint8)
    flip = torch.tensor([0, 1, 0, 1], device=DEV, dtype=torch.uint8)
    y = ops.normalize_u8(x, flip=flip)
    ref = ops.normalize_u8(x.cpu(), flip=flip.cpu())
    assert y.shape == (4, 3, 20, 24) and y.is_contiguous(memory_format=torch.channels_last)
    assert _rel(y.cpu(), ref) < 1e-2
