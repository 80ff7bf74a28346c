"""Weight-gradient delivery on the two weight-gradient streams for every convolution and linear path of ops/gemm.py:
the gradient lands in the sink exactly as a plain run computes it, ``ready`` runs once, ``param.grad`` stays unset and
each weight gradient takes one turn of the round-robin over the streams."""
import pytest
import torch

from edl_b200 import ops
from edl_b200.ops import gemm as G
from test_wgrad_delivery_cpu import _nhwc, check_delivery, conv1x1_case, conv_lib_case, linear_case

pytestmark = [pytest.mark.gpu]
DEV = "cuda"


@pytest.fixture
def streams():
    return [torch.cuda.Stream(), torch.cuda.Stream()]


def _conv_case(fn, n, cin, cout, hw, out_hw, **kw):
    x = _nhwc(n, cin, hw, hw, device=DEV).requires_grad_(True)
    w = (torch.randn(cout, 3, 3, cin, device=DEV) * 0.05).bfloat16().requires_grad_(True)
    dy = _nhwc(n, cout, out_hw, out_hw, device=DEV)
    return x, w, (lambda: fn(x, w, **kw).backward(dy)), [w]


@pytest.mark.parametrize("n,cin,cout,hw,split", [(8, 64, 64, 28, True), (2, 1024, 1024, 14, False)])
def test_conv1x1(streams, n, cin, cout, hw, split):
    torch.manual_seed(0)
    assert (G._split_k_for(cout, cin, n * hw * hw) > 1) == split
    run, params = conv1x1_case(n, cin, cout, hw, DEV)
    check_delivery(run, params, streams)


def test_linear_with_bias(streams):
    torch.manual_seed(1)
    check_delivery(*linear_case(256, 512, 1000, DEV), streams)


@pytest.mark.parametrize("cin,cout,hw,stride,groups", [(64, 128, 28, 2, 1), (128, 128, 14, 1, 4)])
def test_conv_lib(streams, cin, cout, hw, stride, groups):
    torch.manual_seed(2)
    check_delivery(*conv_lib_case(4, cin, cout, hw, stride, groups, DEV), streams)


@pytest.mark.parametrize("pair", [False, True])
def test_conv_lib_32_channels(monkeypatch, streams, pair):
    monkeypatch.setattr(G, "PAIR_WGRAD", pair)
    torch.manual_seed(3)
    x, w, run, params = _conv_case(lambda x, w: ops.conv_lib(x, w, 1, 1, 1), 2, 32, 32, 56, 56)
    assert G._pair_wgrad_ok(x, x, w, (1, 1, 1)) == pair
    check_delivery(run, params, streams)


@pytest.mark.parametrize("own", [False, True])
def test_conv3x3(monkeypatch, streams, own):
    monkeypatch.setattr(G, "OWN_WGRAD3", own)
    torch.manual_seed(4)
    x, w, run, params = _conv_case(ops.conv3x3, 4, 64, 128, 28, 28)
    assert ops.conv3x3_supported(x, w) and ops.conv3x3_wgrad_supported(x, w)
    check_delivery(run, params, streams)


@pytest.mark.parametrize("own", [False, True])
def test_conv3x3_s2(monkeypatch, streams, own):
    monkeypatch.setattr(G, "OWN_S2_BWD", own)
    torch.manual_seed(5)
    x, w, run, params = _conv_case(ops.conv3x3_s2, 4, 128, 128, 56, 28)
    assert ops.conv3x3_s2_supported(x, w) and G._s2_wgrad_supported(x, w) == own
    check_delivery(run, params, streams)


@pytest.mark.parametrize("h,w", [(64, 64), (33, 47)])
def test_stem_conv(streams, h, w):
    """Even input: the direct weight-gradient kernel; odd input: the library weight gradient."""
    torch.manual_seed(6)
    x = _nhwc(2, 3, h, w, device=DEV)
    wt = (torch.randn(32, 3, 3, 3, device=DEV) * 0.2).bfloat16().requires_grad_(True)
    dy = _nhwc(2, 32, (h - 1) // 2 + 1, (w - 1) // 2 + 1, device=DEV)
    assert ops.stem_conv_supported(x, wt)
    check_delivery(lambda: ops.stem_conv(x, wt).backward(dy), [wt], streams)


def test_conv3x3_pair(monkeypatch, streams):
    monkeypatch.setattr(G, "OWN_STEM23", True)
    torch.manual_seed(7)
    x, w, run, params = _conv_case(ops.conv3x3_pair, 2, 32, 32, 56, 56)
    assert ops.conv3x3_pair_supported(x, w)
    check_delivery(run, params, streams)
