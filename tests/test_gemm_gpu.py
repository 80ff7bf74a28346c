"""wgmma GEMM / 1x1-conv kernel numerics against float64 references, element by element (tests/f64_bounds.py)."""
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.ops import gemm as G

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (300, 128, 64), (1568, 2048, 512), (257, 64, 256),
                                   (32, 1000, 2048), (6272, 256, 1024), (100, 192, 72)])
def test_gemm_tn(m, n, k):
    torch.manual_seed(0)
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(n, k, device=DEV).bfloat16()
    d = ops.gemm_bf16(a, b)
    fb.check_bf16(d, *fb.gemm_ref(a, b), k, what="gemm")


def test_gemm_epilogue_scale_shift_relu_stats():
    torch.manual_seed(0)
    m, n, k = 777, 256, 128
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(n, k, device=DEV).bfloat16()
    scale = torch.rand(n, device=DEV) + 0.5
    shift = torch.randn(n, device=DEV)
    stats = torch.zeros(2 * n, device=DEV)
    d = ops.gemm_bf16(a, b, col_scale=scale, col_shift=shift, relu=True, col_stats=stats)
    fb.check_bf16(d, *fb.gemm_ref(a, b, scale=scale, shift=shift, relu=True), k, what="gemm ssr")
    fb.check_sums(stats, *fb.stats_ref(d), m, what="gemm stats")


@pytest.mark.parametrize("m,n,k", [(300, 128, 64), (1568, 512, 2048), (500, 64, 256), (32, 2048, 1000)])
def test_gemm_b_mn_major(m, n, k):
    torch.manual_seed(0)
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(k, n, device=DEV).bfloat16()
    d = ops.gemm_bf16(a, b, b_mn_major=True)
    fb.check_bf16(d, *fb.gemm_ref(a, b, b_mn_major=True), k, what="dgrad gemm")


@pytest.mark.parametrize("m,n,k,split", [(256, 64, 1000, 4), (512, 128, 6272, 16), (64, 64, 100352 // 8, 32),
                                         (1000, 2048, 32, 1)])
def test_gemm_wgrad_bf16_splitk(m, n, k, split):
    torch.manual_seed(0)
    a = torch.randn(k, m, device=DEV).bfloat16()   # [K, M]
    b = torch.randn(k, n, device=DEV).bfloat16()   # [K, N]
    ops.reset_launches()
    d = G._wgrad_impl(a, b, (m, n), None, split_k=split)
    assert ops.launches() == 1                      # the wgmma kernel, not the library fallback
    assert d.dtype == torch.bfloat16
    fb.check_bf16(d, *fb.gemm_ref(a, b, a_mn_major=True, b_mn_major=True), k, split, what="wgrad gemm")
    # accumulate into a prefilled output (a window of the flat gradient bucket)
    sink = torch.randn(m * n, device=DEV).bfloat16()
    want = fb.gemm_ref(a, b, a_mn_major=True, b_mn_major=True, add=sink.view(m, n))
    assert G._wgrad_impl(a, b, (m, n), sink, split_k=split) is None
    fb.check_bf16(sink.view(m, n), *want, k, split, what="wgrad gemm sink")


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
    xd, wd = x.detach(), w.detach()
    fb.check_bf16(y, *fb.conv_ref(xd, wd, padding=0), cin, what="conv1x1 fprop")
    fb.check_sums(stats, *fb.stats_ref(y), y.numel() // cout, what="conv1x1 stats")
    fb.check_bf16(x.grad, *fb.dgrad_ref(dy, wd, x.shape, padding=0), cout, what="conv1x1 dgrad")
    m = n * hw * hw
    fb.check_bf16(w.grad.reshape(cout, cin), *fb.gemm_ref(fb.rows(dy), fb.rows(xd), a_mn_major=True, b_mn_major=True), m,
                  G._split_k_for(cout, cin, m), what="conv1x1 wgrad")


def test_linear_bf16():
    torch.manual_seed(0)
    x = torch.randn(32, 2048, device=DEV).bfloat16().requires_grad_(True)
    w = (torch.randn(1000, 2048, device=DEV) * 0.02).bfloat16().requires_grad_(True)
    b = torch.randn(1000, device=DEV).requires_grad_(True)
    y = ops.linear_bf16(x, w, b)
    dy = torch.randn_like(y)
    y.backward(dy)
    xd, wd = x.detach(), w.detach()
    fb.check_bf16(y, *fb.gemm_ref(xd, wd, shift=b.detach().float()), 2048, what="linear")
    fb.check_bf16(x.grad, *fb.gemm_ref(dy, wd, b_mn_major=True), 1000, what="linear dgrad")
    fb.check_bf16(w.grad, *fb.gemm_ref(dy, xd, a_mn_major=True, b_mn_major=True), 32, G._split_k_for(1000, 2048, 32),
                  what="linear wgrad")
    # the bias gradient is an fp32 column sum of dy (one rounding per row)
    fb.check_sums(b.grad, dy.double().sum(0), dy.double().abs().sum(0), 32, what="linear bias grad", tau_s=33 * fb.EPS32)
