"""Weight-gradient delivery into the flat gradient bucket (ops/gemm.py): a layer whose weight has a gradient sink adds
its weight gradient into the sink, reports it once through ``ready`` and leaves ``param.grad`` unset.  The CPU cases run
without side streams; tests/test_wgrad_delivery_gpu.py runs every path on the weight-gradient streams."""
import torch

from edl_b200 import ops
from edl_b200.ops import gemm as G

SINK_FILL = 0.125


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def check_delivery(run, params, streams=None):
    """``run()`` does one forward and backward through the layer that owns ``params``.  A plain run gives the
    reference gradients; a second run with every parameter's gradient sink prefilled with SINK_FILL and
    ``set_wgrad_stream(streams)`` must leave exactly those gradients in the sinks, each reported once, with one
    side-stream pick per weight gradient."""
    for p in params:
        p.grad = None
    run()
    want = [p.grad.float().clone() for p in params]
    sinks, calls = [], []
    for i, p in enumerate(params):
        p.grad = None
        sinks.append(torch.full((p.numel(),), SINK_FILL, device=p.device, dtype=p.dtype))
        p._edl_grad_sink = sinks[-1]
        p._edl_grad_ready = lambda i=i: calls.append(i)
    G.set_wgrad_stream(streams)
    try:
        run()
        for s in streams or ():
            torch.cuda.current_stream().wait_stream(s)
        G.release_wgrad_keepalive()
        picks = G._SIDE["next"]
    finally:
        G.set_wgrad_stream(None)
        for p in params:
            del p._edl_grad_sink, p._edl_grad_ready
    assert sorted(calls) == list(range(len(params))), calls
    assert all(p.grad is None for p in params)
    # the weight (params[0]) takes the side stream; a linear layer's bias is added on the current stream
    assert picks == (1 if streams else 0), picks
    for p, s, w in zip(params, sinks, want):
        assert _rel(s.float() - SINK_FILL, w.view(-1)) < 1e-2, _rel(s.float() - SINK_FILL, w.view(-1))


def _nhwc(*shape, device="cpu", scale=1.0):
    return (torch.randn(*shape, device=device) * scale).bfloat16().contiguous(memory_format=torch.channels_last)


def conv1x1_case(n, cin, cout, hw, device):
    x = _nhwc(n, cin, hw, hw, device=device).requires_grad_(True)
    w = (torch.randn(cout, cin, device=device) * 0.05).bfloat16().requires_grad_(True)
    dy = _nhwc(n, cout, hw, hw, device=device)
    return (lambda: ops.conv1x1(x, w).backward(dy)), [w]


def linear_case(m, k, n, device):
    x = torch.randn(m, k, device=device).bfloat16().requires_grad_(True)
    w = (torch.randn(n, k, device=device) * 0.05).bfloat16().requires_grad_(True)
    b = torch.randn(n, device=device).bfloat16().requires_grad_(True)
    dy = torch.randn(m, n, device=device).bfloat16()
    return (lambda: ops.linear_bf16(x, w, b).backward(dy)), [w, b]


def conv_lib_case(n, cin, cout, hw, stride, groups, device):
    x = _nhwc(n, cin, hw, hw, device=device).requires_grad_(True)
    w = (torch.randn(cout, 3, 3, cin // groups, device=device) * 0.05).bfloat16().requires_grad_(True)
    dy = _nhwc(n, cout, (hw - 1) // stride + 1, (hw - 1) // stride + 1, device=device)
    return (lambda: ops.conv_lib(x, w, stride, 1, groups).backward(dy)), [w]


def test_conv1x1_cpu():
    torch.manual_seed(0)
    check_delivery(*conv1x1_case(2, 64, 32, 6, "cpu"))


def test_linear_with_bias_cpu():
    torch.manual_seed(1)
    check_delivery(*linear_case(48, 64, 40, "cpu"))


def test_conv_lib_cpu():
    torch.manual_seed(2)
    check_delivery(*conv_lib_case(2, 16, 32, 9, 2, 1, "cpu"))
    check_delivery(*conv_lib_case(2, 32, 32, 8, 1, 4, "cpu"))
