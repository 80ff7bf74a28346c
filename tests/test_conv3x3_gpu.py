"""wgmma implicit-GEMM 3x3 convolution (csrc/conv3x3.cu): fprop + fused BN statistics + dgrad vs the
fp32 PyTorch convolution; autograd wrapper incl. the side-stream library wgrad."""
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


SHAPES = [  # n, cin, cout, h, w
    (2, 64, 64, 56, 56), (3, 128, 128, 28, 28), (4, 256, 256, 14, 14), (5, 512, 512, 7, 7),
    (2, 64, 128, 10, 12), (1, 128, 64, 9, 30), (3, 64, 192, 5, 5), (2, 64, 64, 33, 128), (2, 64, 64, 11, 20)]


@pytest.mark.parametrize("n,cin,cout,h,w", SHAPES)
def test_conv3x3_fprop_and_stats(n, cin, cout, h, w):
    torch.manual_seed(0)
    x = torch.randn(n, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 3, 3, cin, device=DEV) * 0.05).bfloat16()
    assert ops.conv3x3_supported(x, wt)
    stats = torch.zeros(2 * cout, device=DEV)
    y = ops.conv3x3(x, wt, stats)
    ref = fb.conv_ref(x, wt)
    assert y.shape == ref[0].shape and y.is_contiguous(memory_format=torch.channels_last)
    fb.check_bf16(y, *ref, 9 * cin, what="conv3x3 fprop")
    fb.check_sums(stats, *fb.stats_ref(y), n * h * w, what="conv3x3 stats")


@pytest.mark.parametrize("n,cin,cout,h,w", [s for s in SHAPES if s[1] % 64 == 0 and (s[1] <= 64 or s[1] % 128 == 0)])
def test_conv3x3_dgrad_and_wgrad(n, cin, cout, h, w):
    torch.manual_seed(1)
    x = torch.randn(n, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    wt = (torch.randn(cout, 3, 3, cin, device=DEV) * 0.05).bfloat16().requires_grad_(True)
    y = ops.conv3x3(x, wt)
    dy = torch.randn_like(y)
    y.backward(dy)
    xd, wd = x.detach(), wt.detach()
    fb.check_bf16(x.grad, *fb.dgrad_ref(dy, wd, x.shape), 9 * cout, what="conv3x3 dgrad")
    # the weight gradient of this path is the library's (EDL_OWN_WGRAD3 off): its split-K is unknown, so allow one
    # partial per 64-pixel block
    k = n * h * w
    fb.check_bf16(wt.grad.view(cout, -1), *[t.reshape(cout, -1) for t in fb.wgrad_ref(xd, dy, wd.shape)], k, k // 64 + 1,
                  what="conv3x3 library wgrad")


def test_conv3x3_unsupported_shapes_are_reported():
    x = torch.randn(2, 32, 8, 8, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    assert not ops.conv3x3_supported(x, torch.randn(64, 3, 3, 32, device=DEV).bfloat16())      # Cin % 64
    x = torch.randn(2, 64, 8, 200, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    assert not ops.conv3x3_supported(x, torch.randn(64, 3, 3, 64, device=DEV).bfloat16())      # W > 128
