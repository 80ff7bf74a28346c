"""Plain ResNet (models/resnet.py: 7x7 stem, 1x1 / stride-2 projections) in fp32 on the CPU against the same network
written with stock PyTorch ops: forward and backward agree, and CPU tensors never count a library fallback."""
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models.resnet import ResNet, _Bottleneck


def _ref_unit(u, x, residual=None):
    y = F.conv2d(x, u.weight.permute(0, 3, 1, 2), None, u.stride, (u.k - 1) // 2)
    y = F.batch_norm(y, None, None, u.bn.weight, u.bn.bias, True, 0.1, u.bn.eps)
    if residual is not None:
        y = y + residual
    return torch.relu(y) if u.bn.relu else y


def _ref_forward(m, x):
    x = F.max_pool2d(_ref_unit(m.stem, x), 3, 2, 1)
    for b in m.blocks:
        s = _ref_unit(b.short, x) if b.short is not None else x
        if isinstance(b, _Bottleneck):
            x = _ref_unit(b.c, _ref_unit(b.b, _ref_unit(b.a, x)), s)
        else:
            x = _ref_unit(b.b, _ref_unit(b.a, x), s)
    return F.linear(x.mean((2, 3)), m.fc.weight, m.fc.bias)


@pytest.mark.parametrize("layers,width", [(18, 0.25), (50, 0.125)])
def test_plain_resnet_cpu_matches_reference(layers, width):
    torch.manual_seed(layers)
    m = ResNet(layers, class_dim=10, width_mult=width).train()
    convs = [mod for mod in m.modules() if hasattr(mod, "k")]
    assert any(u.k == 7 for u in convs) and any(u.k == 1 and u.stride == 2 for u in convs)
    x = torch.randn(4, 3, 48, 48)
    t = torch.randint(0, 10, (4,))
    ops.reset_fallbacks()

    y = m(x)
    F.cross_entropy(y, t).backward()
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)

    ref = _ref_forward(m, x)
    F.cross_entropy(ref, t).backward()
    torch.testing.assert_close(y, ref, rtol=1e-4, atol=1e-4)
    for n, p in m.named_parameters():
        assert got[n] is not None and p.grad is not None, n
        # fp32 sums in a different order through up to 50 train-mode BatchNorms: compare as tensors, not elements
        rel = ((got[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30)).item()
        assert rel < 1e-3, (n, rel)
    assert ops.fallbacks() == {}, "CPU tensors count no library fallback"
