"""wgmma GEMM / 1x1-conv kernel numerics vs fp32 PyTorch matmul / conv2d."""
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (300, 128, 64), (1568, 2048, 512), (257, 64, 256),
                                   (32, 1000, 2048), (6272, 256, 1024), (100, 192, 72)])
def test_gemm_tn(m, n, k):
    torch.manual_seed(0)
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(n, k, device=DEV).bfloat16()
    d = ops.gemm_bf16(a, b)
    ref = a.float() @ b.float().t()
    assert _rel(d, ref) < 1e-2


def test_gemm_epilogue_scale_shift_relu_stats():
    torch.manual_seed(0)
    m, n, k = 777, 256, 128
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(n, k, device=DEV).bfloat16()
    scale = torch.rand(n, device=DEV) + 0.5
    shift = torch.randn(n, device=DEV)
    stats = torch.zeros(2 * n, device=DEV)
    d = ops.gemm_bf16(a, b, col_scale=scale, col_shift=shift, relu=True, col_stats=stats)
    ref = torch.relu((a.float() @ b.float().t()) * scale + shift)
    assert _rel(d, ref) < 1e-2
    assert _rel(stats[:n], d.float().sum(0)) < 1e-3
    assert _rel(stats[n:], (d.float() ** 2).sum(0)) < 1e-3


@pytest.mark.parametrize("m,n,k", [(300, 128, 64), (1568, 512, 2048), (500, 64, 256), (32, 2048, 1000)])
def test_gemm_b_mn_major(m, n, k):
    torch.manual_seed(0)
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(k, n, device=DEV).bfloat16()
    d = ops.gemm_bf16(a, b, b_mn_major=True)
    assert _rel(d, a.float() @ b.float()) < 1e-2


@pytest.mark.parametrize("m,n,k,split", [(256, 64, 1000, 4), (512, 128, 6272, 16), (64, 64, 100352 // 8, 32),
                                         (1000, 2048, 32, 1)])
def test_gemm_wgrad_bf16_splitk(m, n, k, split):
    from edl_b200.ops import gemm as G

    torch.manual_seed(0)
    a = torch.randn(k, m, device=DEV).bfloat16()   # [K, M]
    b = torch.randn(k, n, device=DEV).bfloat16()   # [K, N]
    ref = a.float().t() @ b.float()
    ops.reset_launches()
    d = G._wgrad_impl(a, b, (m, n), None, split_k=split)
    assert ops.launches() == 1                      # the wgmma kernel, not the library fallback
    assert d.dtype == torch.bfloat16 and _rel(d, ref) < 5e-3
    # accumulate into a prefilled output (a window of the flat gradient bucket)
    sink = torch.randn(m * n, device=DEV).bfloat16()
    want = sink.float().view(m, n) + ref
    assert G._wgrad_impl(a, b, (m, n), sink, split_k=split) is None
    assert _rel(sink.view(m, n), want) < 5e-3


@pytest.mark.parametrize("n,cin,cout,hw", [(2, 64, 256, 56), (4, 256, 64, 14), (3, 512, 2048, 7), (2, 1024, 256, 14)])
def test_conv1x1_fwd_bwd(n, cin, cout, hw):
    torch.manual_seed(0)
    x = (torch.randn(n, cin, hw, hw, device=DEV)).bfloat16().contiguous(memory_format=torch.channels_last)
    x.requires_grad_(True)
    w = (torch.randn(cout, 1, 1, cin, device=DEV) * 0.05).bfloat16().requires_grad_(True)
    stats = torch.zeros(2 * cout, device=DEV)
    y = ops.conv1x1(x, w, stats)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    wr = w.detach().float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yr = F.conv2d(xr, wr)
    yr.backward(dy.float())
    assert _rel(y, yr) < 1e-2
    assert _rel(x.grad, xr.grad) < 1e-2
    assert _rel(w.grad.permute(0, 3, 1, 2), wr.grad) < 1e-2
    assert _rel(stats[:cout], y.float().sum((0, 2, 3))) < 1e-3


def test_linear_bf16():
    torch.manual_seed(0)
    x = torch.randn(32, 2048, device=DEV).bfloat16().requires_grad_(True)
    w = (torch.randn(1000, 2048, device=DEV) * 0.02).bfloat16().requires_grad_(True)
    b = torch.randn(1000, device=DEV).requires_grad_(True)
    y = ops.linear_bf16(x, w, b)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr, wr, br = [t.detach().float().requires_grad_(True) for t in (x, w, b)]
    yr = F.linear(xr, wr, br)
    yr.backward(dy.float())
    assert _rel(y, yr) < 1e-2 and _rel(x.grad, xr.grad) < 1e-2
    assert _rel(w.grad, wr.grad) < 1e-2 and _rel(b.grad, br.grad) < 1e-2
