"""ReLU mask bits of the residual BatchNorms (ops/bn.py ``set_relu_mask``): the streaming apply kernel writes
uint8 [M, C/8] with bit b of byte j = (stored y[:, 8 j + b] > 0); a 1x1 dgrad that carries the BN's backward reduction
stores its gradient already masked, and the BN backward then returns that gradient as the residual gradient."""
import numpy as np
import pytest
import torch

from edl_b200 import ops

DEV = "cuda"
gpu = pytest.mark.gpu


def pack_mask(y2):
    """Reference packing: y2 [M, C] -> uint8 [M, C/8], bit b of byte j set iff y2[:, 8 j + b] > 0."""
    m, c = y2.shape
    bits = (y2 > 0).reshape(m, c // 8, 8).to(torch.int32)
    return (bits << torch.arange(8, device=y2.device, dtype=torch.int32)).sum(-1).to(torch.uint8)


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def test_pack_mask_reference_matches_numpy():
    g = torch.Generator().manual_seed(0)
    y = torch.randn(37, 256, generator=g).bfloat16()
    y[0, :16] = 0.0
    y[1, :16] = -0.0
    ref = np.packbits((y.float() > 0).numpy(), axis=1, bitorder="little")
    assert np.array_equal(pack_mask(y).numpy(), ref)


def _stage_inputs(m, c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(m, c, device=DEV, generator=g).bfloat16()
    res = torch.randn(m, c, device=DEV, generator=g).bfloat16()
    gamma = torch.rand(c, device=DEV, generator=g) + 0.5
    beta = torch.randn(c, device=DEV, generator=g) * 0.2
    # channels whose fp32 output is a positive value below bf16's range (stored as +0) or a negative one (-> 0)
    gamma[:8] = 0.0
    beta[:4] = 1e-42
    beta[4:8] = -1e-42
    res[:, :8] = 0.0
    return x, res, gamma, beta


def _sums(x):
    sums = torch.zeros(2 * x.shape[1], device=DEV)
    ops.native().bn_stats(x, sums)
    return sums


def _apply(x, res, gamma, beta, mask=None, sums=None):
    m, c = x.shape
    nat = ops.native()
    sums = _sums(x) if sums is None else sums
    y = torch.empty_like(x)
    mean, rstd = torch.empty(c, device=DEV), torch.empty(c, device=DEV)
    nat.bn_apply(x, res, y, sums, gamma, beta, None, None, mean, rstd, 1e-5, 0.1, True, mask)
    return y, mean, rstd


# the four residual-BN shapes of ResNet50_vd at batch 32, and an M whose last 16 KB chunk is partial
SHAPES = [(32 * 56 * 56, 256), (32 * 28 * 28, 512), (32 * 14 * 14, 1024), (32 * 7 * 7, 2048), (1000, 256)]


@gpu
@pytest.mark.parametrize("m,c", SHAPES)
def test_apply_writes_the_mask_of_the_stored_output(m, c):
    x, res, gamma, beta = _stage_inputs(m, c, 1)
    assert ops.native().bn_relu_mask_supported(m, c)
    mask = torch.full((m, c // 8), 0xA5, device=DEV, dtype=torch.uint8)
    sums = _sums(x)
    y, _, _ = _apply(x, res, gamma, beta, mask, sums)
    y_ref, _, _ = _apply(x, res, gamma, beta, None, sums)
    assert torch.equal(y, y_ref)                       # the output itself is unchanged
    assert (y[:, :8] == 0).all()
    assert torch.equal(mask, pack_mask(y))


@gpu
@pytest.mark.parametrize("m,c", SHAPES)
def test_backward_from_mask_bits_matches_backward_from_y(m, c):
    nat = ops.native()
    x, res, gamma, beta = _stage_inputs(m, c, 2)
    mask = torch.empty((m, c // 8), device=DEV, dtype=torch.uint8)
    y, mean, rstd = _apply(x, res, gamma, beta, mask)
    dy = torch.randn(m, c, device=DEV).bfloat16()
    # reduction: same sums up to the order of the fp32 atomics
    ds_y, ds_m = torch.zeros(2 * c, device=DEV), torch.zeros(2 * c, device=DEV)
    nat.bn_bwd_reduce(dy, x, y, gamma, beta, mean, rstd, ds_y, True)
    nat.bn_bwd_reduce(dy, x, mask, gamma, beta, mean, rstd, ds_m, True)
    assert _rel(ds_m, ds_y) < 1e-4
    # apply with the same dsums: bit-identical dx and dres
    outs = []
    for ym in (y, mask):
        dx, dres = torch.empty_like(x), torch.empty_like(x)
        dg, db = torch.empty_like(gamma), torch.empty_like(gamma)
        nat.bn_bwd_apply(dy, x, ym, gamma, beta, mean, rstd, ds_y, dx, dres, dg, db, True, False)
        outs.append((dx, dres, dg, db))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert torch.equal(outs[1][1], torch.where(y > 0, dy, torch.zeros_like(dy)))


def _hook(x, n, y=None, mask=None):
    from edl_b200.ops.bn import BNBackwardHook

    g = torch.Generator(device=DEV).manual_seed(3)
    h = BNBackwardHook()
    h.x, h.y, h.mask, h.relu = x, y, mask, True
    h.mean, h.rstd = torch.randn(n, device=DEV, generator=g) * 0.1, torch.rand(n, device=DEV, generator=g) + 0.5
    h.gamma, h.beta = torch.rand(n, device=DEV, generator=g) + 0.5, torch.randn(n, device=DEV, generator=g) * 0.2
    h.dsums = torch.zeros(2 * n, device=DEV)
    return h


@gpu
@pytest.mark.parametrize("m,k,n", [(6272, 64, 256), (25088, 128, 512), (5000, 256, 1024), (1568, 512, 2048)])
def test_dgrad_epilogue_stores_the_masked_gradient(m, k, n):
    torch.manual_seed(4)
    a = torch.randn(m, k, device=DEV).bfloat16()
    w = (torch.randn(k, n, device=DEV) * 0.1).bfloat16()
    x = torch.randn(m, n, device=DEV).bfloat16()
    y = torch.relu(torch.randn(m, n, device=DEV)).bfloat16()
    add = torch.randn(m, n, device=DEV).bfloat16()
    hy, hm = _hook(x, n, y=y), _hook(x, n, mask=pack_mask(y))
    d_y = ops.gemm_bf16(a, w, b_mn_major=True, bn=hy, add=add)
    d_m = ops.gemm_bf16(a, w, b_mn_major=True, bn=hm, add=add)
    assert hy.done and hm.done
    assert torch.equal(d_m, torch.where(y > 0, d_y, torch.zeros_like(d_y)))
    assert _rel(hm.dsums, hy.dsums) < 1e-4


def _block(relu_mask, seed=5):
    """z = relu(bn(x) + res) feeding a forked 1x1 convolution, as in a bottleneck: returns the gradients, the
    BN's hook and the gradient tensors that reached z and res."""
    ops.set_relu_mask(relu_mask)
    try:
        torch.manual_seed(seed)
        n, c, h, wd = 8, 256, 28, 28
        x = torch.randn(n, c, h, wd, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_()
        res = torch.randn(n, c, h, wd, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_()
        w = (torch.randn(64, 1, 1, c, device=DEV) * 0.05).bfloat16().requires_grad_()
        bn = ops.BatchNormAct2d(c, relu=True).to(DEV)
        z = bn(x, residual=res)
        hook = z._edl_bn_hook
        seen = {}
        z.register_hook(lambda g: seen.__setitem__("dz", g))
        res.register_hook(lambda g: seen.__setitem__("dres", g))
        y, za = ops.conv1x1(z, w, None, fork=True)
        gy = torch.randn_like(y)
        gz = torch.randn_like(za)
        torch.autograd.backward([y, za], [gy, gz])
        grads = [x.grad, res.grad, w.grad, bn.weight.grad, bn.bias.grad]
        return grads, hook, seen
    finally:
        ops.set_relu_mask(True)


@gpu
def test_fused_block_returns_the_stored_gradient_as_residual_gradient():
    g_off, h_off, s_off = _block(False)
    g_on, h_on, s_on = _block(True)
    assert h_off.mask is None and h_off.y is not None and h_off.done
    assert h_on.mask is not None and h_on.y is None and h_on.done
    # the residual gradient IS the stored (masked) dgrad output: same storage, no copy
    assert s_on["dres"].data_ptr() == s_on["dz"].data_ptr()
    assert s_off["dres"].data_ptr() != s_off["dz"].data_ptr()
    # masked dy: bit for bit what the y-path returned as dres
    assert torch.equal(s_on["dres"], s_off["dres"])
    assert torch.equal(g_on[1], g_off[1])
    for a, b in zip(g_on, g_off):                      # dx and the parameter gradients: fp32 atomics in the sums
        assert _rel(a, b) < 1e-2


def _train_step(relu_mask, graph, x, t):
    from edl_b200.models import ResNet50_vd, to_train_dtype
    from edl_b200.trainer import StudentTrainer

    ops.set_relu_mask(relu_mask)
    try:
        torch.manual_seed(0)
        m = to_train_dtype(ResNet50_vd(), torch.bfloat16, torch.device(DEV)).train()
        tr = StudentTrainer(m, batch_size=x.shape[0], image_shape=tuple(x.shape[1:]), lr=0.01, use_graph=graph)
        ops.reset_launches()
        loss = float(tr.step(x, t).item())
        torch.cuda.synchronize()
        launches = ops.launches()
        sd = tr.opt.state_dict()
        # fp32 momentum (the gradients plus weight decay, accumulated over the steps taken) and fp32 master weights
        state = [v.detach().float().clone() for k in ("momentum", "master") for v in sd[k].values()]
        bufs = [b.detach().float().clone() for b in m.buffers()]
        return loss, launches, state, bufs
    finally:
        ops.set_relu_mask(True)


@gpu
@pytest.mark.parametrize("graph", [False, True])
def test_resnet50_vd_step_with_and_without_mask_bits(graph):
    torch.manual_seed(7)
    x = torch.randn(8, 3, 128, 128).bfloat16().contiguous(memory_format=torch.channels_last).pin_memory()
    t = torch.softmax(torch.randn(8, 1000), -1).bfloat16().pin_memory()
    # the yardstick is the run-to-run spread: a second run of the same path (fp32 atomics, bf16 roundings that flip)
    l_off, n_off, u_off, b_off = _train_step(False, graph, x, t)
    l_ctl, _, u_ctl, b_ctl = _train_step(False, graph, x, t)
    l_on, n_on, u_on, b_on = _train_step(True, graph, x, t)
    assert n_on == n_off
    assert abs(l_on - l_off) <= max(1e-3 * abs(l_off), 3 * abs(l_ctl - l_off))
    assert len(u_on) >= 2 and len(u_on) == len(u_off)
    for a, b, c in zip(u_on, u_off, u_ctl):
        assert _rel(a, b) <= max(1e-2, 3 * _rel(c, b)), (_rel(a, b), _rel(c, b))
    for a, b, c in zip(b_on, b_off, b_ctl):
        assert _rel(a, b) <= max(1e-3, 3 * _rel(c, b)), (_rel(a, b), _rel(c, b))
