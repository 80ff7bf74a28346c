"""Split-K weight gradients through partial tiles (csrc/gemm.cu EPI 1, csrc/conv3x3_wgrad.cu): every split is summed
by one reduce kernel in a fixed order, so repeated calls give the same bits; the partial-tile buffer grows for splits
that do not fit it; a split without (enough) partial tiles is an error, never a different path."""
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.ops import gemm as G

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _wref(x, dy, shape, stride=1):
    return [t.reshape(shape[0], -1) for t in fb.wgrad_ref(x, dy, shape, stride)]


def _nhwc(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).bfloat16().contiguous(memory_format=torch.channels_last)


def test_wgrad1x1_splitk_bitwise_reproducible():
    torch.manual_seed(0)
    m, n, k, split = 512, 128, 6272, 16
    a = torch.randn(k, m, device=DEV).bfloat16()
    b = torch.randn(k, n, device=DEV).bfloat16()
    d1 = G._wgrad_impl(a, b, (m, n), None, split_k=split)
    d2 = G._wgrad_impl(a, b, (m, n), None, split_k=split)
    assert torch.equal(d1, d2)
    sinks = [torch.full((m * n,), 0.5, device=DEV, dtype=torch.bfloat16) for _ in range(2)]
    for s in sinks:
        G._wgrad_impl(a, b, (m, n), s, split_k=split)
    assert torch.equal(sinks[0], sinks[1])
    fb.check_bf16(d1, *fb.gemm_ref(a, b, a_mn_major=True, b_mn_major=True), k, split, what="wgrad gemm")
    fb.check_bf16(sinks[0].view(m, n), *fb.gemm_ref(a, b, a_mn_major=True, b_mn_major=True,
                                                     add=torch.full((m, n), 0.5, device=DEV)), k, split,
                  what="wgrad gemm sink")


def test_wgrad3x3_stride2_bitwise_reproducible():
    torch.manual_seed(0)
    n, cin, cout, ho, wo = 8, 64, 128, 14, 14
    if not ops.native().conv3x3_wgrad_s2_supported(n, ho, wo, cin, cout):
        pytest.skip("geometry not supported by the stride-2 weight-gradient planner")
    x = _nhwc(n, cin, 2 * ho, 2 * wo)
    dy = _nhwc(n, cout, ho, wo, scale=0.1)
    shape = (cout, 3, 3, cin)
    for split in (1, 4):
        d1 = G.conv3x3_wgrad(x, dy, shape, None, split_k=split)
        d2 = G.conv3x3_wgrad(x, dy, shape, None, split_k=split)
        assert torch.equal(d1, d2), split
        fb.check_bf16(d1.view(cout, -1), *_wref(x, dy, shape, 2), n * ho * wo, split, what="wgrad3x3 s2")


def test_wgrad3x3_split_beyond_initial_partials_buffer():
    torch.manual_seed(0)
    n, cin, cout, h, w, split = 32, 512, 512, 7, 7, 8
    assert ops.native().conv3x3_wgrad_kblocks(n, h, w) >= split
    # the partial tiles of this split need more than the 64 MB the buffer starts with
    assert split * ops.native().conv3x3_wgrad_tiles(cin, cout) * 128 * 192 * 4 > 64 << 20
    x = _nhwc(n, cin, h, w)
    dy = _nhwc(n, cout, h, w, scale=0.1)
    got = G.conv3x3_wgrad(x, dy, (cout, 3, 3, cin), None, split_k=split)
    fb.check_bf16(got.view(cout, -1), *_wref(x, dy, (cout, 3, 3, cin)), n * h * w, split, what="wgrad3x3 split 8")


def test_split_without_enough_partials_raises():
    torch.manual_seed(0)
    x = _nhwc(8, 64, 28, 28)
    dy = _nhwc(8, 64, 28, 28, scale=0.1)
    dw = torch.full((64, 3, 3, 64), 7.0, device=DEV, dtype=torch.bfloat16)
    a = torch.randn(6272, 256, device=DEV).bfloat16()
    b = torch.randn(6272, 64, device=DEV).bfloat16()
    d = torch.full((256, 64), 7.0, device=DEV, dtype=torch.bfloat16)
    too_few = torch.empty(1024, device=DEV)
    for part in (None, too_few):
        with pytest.raises(RuntimeError, match="partial"):
            ops.native().conv3x3_wgrad(x, dy, dw, 4, False, part)
        with pytest.raises(RuntimeError, match="partial"):
            ops.native().gemm_wgrad_bf16(a, b, d, 4, False, part)
    torch.cuda.synchronize()
    assert bool((dw == 7.0).all()) and bool((d == 7.0).all())     # nothing was launched
