"""The step oracle (tests/step_oracle.py) on the CPU fp32 paths: it passes a real step of ResNet18_vd / ResNet50_vd, and
each small corruption of the recorded step -- one bf16 ulp on a weight gradient, one channel's dgamma off by 2^-10, two
layers' gradient windows swapped, the shortcut term missing from a block input's gradient, one zeroed window -- fails
with a message naming the layer.  Also: a recomputed (checkpointed) forward leaves the running statistics as one plain
step does."""
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.models import ResNetVd, to_train_dtype
from step_oracle import StepRecorder


def _step(layers, seed=0, recompute=False, n=2, size=32):
    torch.manual_seed(seed)
    m = to_train_dtype(ResNetVd(layers, class_dim=10, width_mult=0.125, recompute=recompute), torch.float32).train()
    x = torch.randn(n, 3, size, size)
    t = torch.softmax(torch.randn(n, 10), -1)
    return m, x, t


def _recorded(layers):
    m, x, t = _step(layers)
    with StepRecorder(m) as rec:
        ops.soft_cross_entropy(m(x), t).backward()
    return m, rec


@pytest.fixture(scope="module")
def r18():
    return _recorded(18)


@pytest.mark.parametrize("layers", [18, 50])
def test_oracle_passes_a_cpu_step(layers):
    m, rec = _recorded(layers)
    report = rec.check()
    assert not report["library"]                    # nothing counts as a library fallback on the CPU
    names = {r["name"] for r in rec.convs}
    assert len(names) == len(rec.convs) == len(m.conv_bn_units())
    assert {"bn y", "bn dx", "wgrad", "conv fprop", "bn dgamma / dbeta"} <= set(report["ratios"])


def _best_element(rec, unit):
    """The element of ``unit``'s weight gradient whose reference is largest relative to its rounding slack."""
    r = next(r for r in rec.convs if r["unit"] is unit)
    ref, mag = fb.wgrad_ref(r["x"], r["dy"].grad, tuple(r["w"].shape), unit.stride, (unit.k - 1) // 2)
    return int((ref.abs() / (mag + 1e-30)).flatten().argmax())


def _fails(rec, pattern):
    with pytest.raises(AssertionError, match=pattern):
        rec.check()


def test_one_ulp_on_one_weight_gradient_element_fails(r18):
    m, rec = r18
    u = m.blocks[1].b
    i = _best_element(rec, u)
    g = u.weight.grad.view(-1)
    old = g[i].item()
    try:
        g[i] = old + float(fb.ulp(torch.tensor(abs(old), dtype=torch.float64), 8))
        _fails(rec, r"blocks\.1\.b wgrad \(grad\)")
    finally:
        g[i] = old


def test_one_dgamma_channel_scaled_fails(r18):
    m, rec = r18
    bn = m.blocks[2].a.bn
    r = next(b for b in rec.bns if b["bn"] is bn)
    ref, mag, _ = fb.bn_dsums_ref(r["oact"].grad, r["x"], r["mean"], r["rstd"], r["gamma"], r["beta"], bn.relu,
                                  y=r["out"])
    c = bn.num_features
    ch = int((ref[c:].abs() / mag[c:]).argmax())
    old = bn.weight.grad[ch].item()
    try:
        bn.weight.grad[ch] = old * (1 + 2 ** -10)
        _fails(rec, r"blocks\.2\.a bn dgamma \(grad\)")
    finally:
        bn.weight.grad[ch] = old


def test_swapped_gradient_windows_fail(r18):
    m, rec = r18
    a, b = m.blocks[0].a.weight, m.blocks[0].b.weight
    assert a.shape == b.shape
    ga, gb = a.grad.clone(), b.grad.clone()
    try:
        a.grad.copy_(gb)
        b.grad.copy_(ga)
        _fails(rec, r"blocks\.0\.a wgrad")
    finally:
        a.grad.copy_(ga)
        b.grad.copy_(gb)


def test_dropped_shortcut_term_fails():
    """ResNet50_vd block 1's input feeds conv a and the identity shortcut (c's residual): without the shortcut's term the
    input gradient is that of conv a alone."""
    m, rec = _recorded(50)
    blk = m.blocks[1]
    r = next(r for r in rec.convs if r["unit"] is blk.a)
    act = next(a for a in rec.acts.values() if any(d == "blocks.1.c bn dres" for d, _ in a.terms))
    assert any(d == "blocks.1.a dgrad" for d, _ in act.terms) and r is not None
    res = next(b for b in rec.bns if b["bn"] is blk.c.bn)
    dres = rec._dres_term(res)[0]
    act.grad = (act.grad.double() - dres).to(act.grad.dtype)
    _fails(rec, r"blocks\.0\.c gradient \(blocks\.1\.a dgrad \+ blocks\.1\.c bn dres\)")


def test_zeroed_window_fails(r18):
    m, rec = r18
    p = m.stem[1].bn.bias
    old = p.grad.clone()
    try:
        p.grad.zero_()
        _fails(rec, r"stem\.1 bn dbeta")
    finally:
        p.grad.copy_(old)


def test_missing_gradient_fails(r18):
    m, rec = r18
    p = m.fc.weight
    old = p.grad
    try:
        p.grad = None
        _fails(rec, r"fc wgrad: no gradient")
    finally:
        p.grad = old


def test_recompute_updates_running_statistics_once():
    """The checkpointed blocks run their forward twice; the running statistics must see one momentum update per step,
    as without recompute."""
    a, x, t = _step(18, seed=1, n=3)
    b = to_train_dtype(ResNetVd(18, class_dim=10, width_mult=0.125, recompute=True), torch.float32).train()
    b.load_state_dict(a.state_dict())
    for m in (a, b):
        ops.soft_cross_entropy(m(x), t).backward()
    for (n, p), (_, q) in zip(a.named_buffers(), b.named_buffers()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-6), (n, p[:4], q[:4])
    for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.allclose(p.grad, q.grad, atol=1e-5, rtol=1e-4), n
