"""Plain ResNet (models/resnet.py) on the wgmma kernels: the 1x1 / stride-2 projection shortcuts and the 7x7 / stride-2
stem in training, held to the float64 element-wise bounds of tests/f64_bounds.py, then end to end in the model, the
trainer and its CUDA graph."""
import copy
import os
import subprocess
import sys
import textwrap

import pytest
import torch
import torch.nn.functional as F

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.models import to_train_dtype
from edl_b200.models.resnet import ResNet, _Bottleneck
from edl_b200.ops import gemm as G
from edl_b200.trainer import StudentTrainer

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = -3.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).bfloat16()


def _nhwc(n, c, h, w, scale=1.0):
    return _bf(n, c, h, w, scale=scale).contiguous(memory_format=torch.channels_last)


# ------------------------------------------------------------------------------------------- 1x1 / stride 2 convolution
# (cin, cout, input size): the ResNet50 and ResNet18 projections, then partial tiles (6 -> 3, 12 -> 6, 24 -> 12) and a
# 128-pixel-wide output
PROJ = [(256, 512, 56), (512, 1024, 28), (1024, 2048, 14), (64, 128, 56), (128, 256, 28), (256, 512, 14)]
EDGE = [(64, 128, 6, 6), (128, 64, 12, 12), (64, 192, 24, 24), (64, 64, 4, 256)]
FPROP = ([(n, ci, co, s, s) for ci, co, s in PROJ for n in (1, 3, 32)]
         + [(n, ci, co, h, w) for ci, co, h, w in EDGE for n in (1, 3)])


@pytest.mark.parametrize("n,cin,cout,h,w", FPROP)
def test_conv1x1_s2_fprop_stats_and_inference(n, cin, cout, h, w):
    torch.manual_seed(n * 7 + h + cin)
    x = _nhwc(n, cin, h, w)
    wt = _bf(cout, 1, 1, cin, scale=0.05)
    assert ops.conv1x1_s2_supported(x, wt)
    what = "conv1x1 s2 %s" % ((n, cin, cout, h, w),)
    ref, mag = fb.conv_ref(x, wt, 2, 0)
    y = ops.conv1x1_s2(x, wt)
    fb.check_bf16(y, ref, mag, cin, what=what)
    st = torch.zeros(2 * cout, device=DEV)
    y2 = ops.conv1x1_s2(x, wt, st)
    assert torch.equal(y, y2), what + ": statistics changed the output"
    fb.check_sums(st, *fb.stats_ref(y2), y2.numel() // cout, what=what + " stats")
    sc, sh = torch.rand(cout, device=DEV) + 0.5, torch.randn(cout, device=DEV) * 0.1
    yi = ops.conv1x1_s2_infer(x, wt, sc, sh, relu=True)
    fb.check_bf16(yi, *fb.conv_ref(x, wt, 2, 0, scale=sc.view(1, -1, 1, 1), shift=sh.view(1, -1, 1, 1), relu=True), cin,
                  what=what + " inference")


@pytest.mark.parametrize("n,cin,cout,h,w", [(3, 256, 512, 56, 56), (32, 1024, 2048, 14, 14), (2, 64, 128, 6, 6),
                                            (3, 128, 64, 12, 12), (1, 64, 64, 4, 256)])
def test_conv1x1_s2_dgrad_parities(n, cin, cout, h, w):
    C = ops.native()
    torch.manual_seed(h + cout)
    wt = _bf(cout, 1, 1, cin, scale=0.05)
    dy = _nhwc(n, cout, h // 2, w // 2)
    assert C.conv1x1_s2_supported(n, h // 2, w // 2, cin, cout, True)
    dx = fb.guarded((n, cin, h, w), 3, fill=SENT, values=_nhwc(n, cin, h, w))     # stale values under the zero fill
    C.conv1x1_s2(dy, wt, dx.t, True, None, None, None, False)
    what = "conv1x1 s2 dgrad %s" % ((n, cin, cout, h, w),)
    ref, mag = fb.dgrad_ref(dy, wt, (n, cin, h, w), 2, 0)
    fb.check_bf16(dx.t[:, :, ::2, ::2], ref[:, :, ::2, ::2], mag[:, :, ::2, ::2], cout, what=what)
    for sl in ((slice(None), slice(None), slice(1, None, 2)), (slice(None), slice(None), slice(None, None, 2), slice(1, None, 2))):
        assert (dx.t[sl] == 0).all() and not torch.signbit(dx.t[sl].float()).any(), what + ": skipped pixels not +0"
    dx.assert_untouched(what)


def test_conv1x1_s2_dgrad_through_forked_bottleneck():
    """x feeds conv a (1x1 / stride 1) and the stride-2 projection: its gradient is a's dgrad with the projection's
    (dense, zero-filled) input gradient added in a's epilogue."""
    torch.manual_seed(5)
    blk = to_train_dtype(_Bottleneck(256, 128, 2, "auto"), torch.bfloat16, DEV).train()
    x = _nhwc(4, 256, 28, 28).requires_grad_(True)
    assert blk.a.can_fork(x) and ops.conv1x1_s2_supported(x, blk.short.weight)
    grads = {}

    def capture(unit, key):
        conv = unit.conv

        def wrapped(inp, want_stats, fork=False):
            y, stats = conv(inp, want_stats, fork)
            t = y[0] if fork else y
            t.register_hook(lambda g: grads.__setitem__(key, g.detach().contiguous(memory_format=torch.channels_last)))
            return y, stats
        unit.conv = wrapped

    capture(blk.a, "a")
    capture(blk.short, "short")
    out = blk(x)
    out.backward(_nhwc(*out.shape))
    wa, ws = blk.a.weight.detach(), blk.short.weight.detach()
    ta = fb.dgrad_ref(grads["a"], wa, x.shape, 1, 0)
    ts = fb.dgrad_ref(grads["short"], ws, x.shape, 2, 0)
    ref, mag = ta[0] + ts[0], ta[1] + ts[1]
    fb.check_bf16(x.grad, ref, mag, wa.shape[0] + ws.shape[0], what="bottleneck fork dgrad", terms=[ta, ts])


WGRAD = [(32, 256, 512, 56, 56), (32, 1024, 2048, 14, 14), (8, 64, 128, 56, 56), (16, 128, 64, 6, 6),
         (4, 64, 192, 24, 24)]


@pytest.mark.parametrize("n,cin,cout,h,w", WGRAD)
def test_conv1x1_s2_wgrad_fresh_sink_split(n, cin, cout, h, w):
    C = ops.native()
    torch.manual_seed(n + h + cin)
    x = _nhwc(n, cin, h, w)
    dy = _nhwc(n, cout, h // 2, w // 2, scale=0.1)
    shape = (cout, 1, 1, cin)
    assert C.conv3x3_wgrad_s2_supported(n, h // 2, w // 2, cin, cout)
    ref, mag = [t.reshape(cout, cin) for t in fb.wgrad_ref(x, dy, shape, 2, 0)]
    k = n * (h // 2) * (w // 2)
    kblocks = C.conv3x3_wgrad_s2_kblocks(n, h // 2, w // 2)
    for split in (1, max(2, kblocks // 2), None):
        eff = split if split is not None else G.conv1x1_s2_wgrad_split(n, h // 2, w // 2, cin, cout)
        what = "conv1x1 s2 wgrad %s split %s" % ((n, cin, cout, h, w), eff)
        got = G.conv1x1_s2_wgrad(x, dy, shape, None, split_k=split)
        fb.check_bf16(got.reshape(cout, cin), ref, mag, k, eff, what=what)
        again = G.conv1x1_s2_wgrad(x, dy, shape, None, split_k=split)
        assert torch.equal(got.view(torch.int16), again.view(torch.int16)), what + ": not reproducible"
        prior = _bf(cout * cin)
        sink = fb.guarded(prior.shape, 64, fill=SENT, values=prior)
        assert G.conv1x1_s2_wgrad(x, dy, shape, sink.t, split_k=split) is None
        fb.check_bf16(sink.t.view(cout, cin), *fb.epilogue(ref, mag, add=prior.view(cout, cin)), k, eff,
                      what=what + " sink")
        sink.assert_untouched(what + " sink")


# ------------------------------------------------------------------------------------------------------ 7x7 stem
@pytest.mark.parametrize("n,h,w", [(2, 224, 224), (3, 34, 46), (1, 17, 33)])
def test_stem7_fprop_and_stats(n, h, w):
    torch.manual_seed(h + w)
    x = _nhwc(n, 3, h, w)
    wt = _bf(64, 7, 7, 3, scale=0.05)
    st = torch.zeros(128, device=DEV)
    y = ops.stem7(x, wt, st)
    what = "stem7 %s" % ((n, h, w),)
    fb.check_bf16(y, *fb.conv_ref(x, wt, 2, 3), 160, what=what)
    fb.check_sums(st, *fb.stats_ref(y), y.numel() // 64, what=what + " stats")


@pytest.mark.parametrize("n,h,w,split", [(1, 17, 33, 1), (2, 224, 224, 66)])
def test_stem7_wgrad_guarded_sink(n, h, w, split):
    C = ops.native()
    torch.manual_seed(w)
    x = _nhwc(n, 3, h, w)
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    dy = _nhwc(n, 64, ho, wo, scale=0.1)
    shape = (64, 7, 7, 3)
    assert G._split_k_for(64, 160, n * ho * wo) == split, "the shape no longer takes the path this case is for"
    a = torch.empty((n * ho * wo, 160), device=DEV, dtype=torch.bfloat16)
    C.stem7_im2col(x, a)
    ref, mag = [t.reshape(64, 147) for t in fb.wgrad_ref(x, dy, shape, 2, 3)]
    k = n * ho * wo
    what = "stem7 wgrad %s split %d" % ((n, h, w), split)
    got = G.stem7_wgrad(dy, a, shape)
    fb.check_bf16(got.reshape(64, 147), ref, mag, k, split, what=what)
    prior = _bf(64 * 147)
    sink = fb.guarded(prior.shape, 64, fill=SENT, values=prior)
    assert G.stem7_wgrad(dy, a, shape, sink.t) is None
    fb.check_bf16(sink.t.view(64, 147), *fb.epilogue(ref, mag, add=prior.view(64, 147)), k, split, what=what + " sink")
    sink.assert_untouched(what + " sink")


# ----------------------------------------------------------------------------------------------------- model level
def _ref_unit(u, x, residual=None):
    """Same rounding points as the fused path (bf16 conv output, fp32 BN math, bf16 activation) in stock PyTorch ops."""
    y = F.conv2d(x, u.weight.detach().permute(0, 3, 1, 2), None, u.stride, (u.k - 1) // 2).float()
    y = F.batch_norm(y, None, None, u.bn.weight.detach().float(), u.bn.bias.detach().float(), True, 0.1, u.bn.eps)
    if residual is not None:
        y = y + residual.float()
    return (torch.relu(y) if u.bn.relu else y).bfloat16()


def _ref_forward(m, x):
    x = F.max_pool2d(_ref_unit(m.stem, x), 3, 2, 1)
    for b in m.blocks:
        s = _ref_unit(b.short, x) if b.short is not None else x
        if isinstance(b, _Bottleneck):
            x = _ref_unit(b.c, _ref_unit(b.b, _ref_unit(b.a, x)), s)
        else:
            x = _ref_unit(b.b, _ref_unit(b.a, x), s)
    x = x.float().mean((2, 3)).bfloat16()
    return F.linear(x.float(), m.fc.weight.detach().float(), m.fc.bias.detach().float())


def _images(n, s):
    return torch.randn(n, 3, s, s, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)


def _own_layer_fallbacks():
    return [k for k in ops.fallbacks() if "7x7" in k or ("1x1 stride 2" in k)]


def test_resnet50_matches_fp32_reference_and_trains_on_own_kernels():
    torch.manual_seed(0)
    m = to_train_dtype(ResNet(50, class_dim=104, width_mult=0.5), torch.bfloat16, DEV).train()
    x = _images(16, 96)
    ops.reset_fallbacks()
    y = m(x)
    ref = _ref_forward(m, x)
    rel = ((y.float() - ref).norm() / ref.norm()).item()
    assert rel < 0.15, rel
    t = torch.softmax(torch.randn(16, 104, device=DEV), -1).bfloat16()
    ops.soft_cross_entropy(y, t).backward()
    units = [m.stem] + [b.short for b in m.blocks if b.short is not None and b.short.stride == 2]
    assert len(units) == 4
    for u in units:
        g = u.weight.grad
        assert g is not None and torch.isfinite(g.float()).all() and g.float().abs().sum() > 0, u
    assert not _own_layer_fallbacks(), ops.fallbacks()

    tr = StudentTrainer(m, batch_size=16, image_shape=(3, 96, 96), num_classes=104, lr=0.05, use_graph=False)
    ops.reset_fallbacks()
    tr.step(x.cpu().pin_memory(), t.cpu().pin_memory(), sync=True)
    torch.cuda.synchronize()
    assert not _own_layer_fallbacks(), ops.fallbacks()


def test_stem7_captured_forward_reads_updated_weight():
    """The stem's padded GEMM weight is rebuilt inside a captured graph: a replay after an in-place weight update (what a
    replayed optimizer step does, without touching ``weight._version``) computes with the new weight."""
    torch.manual_seed(3)
    x = _nhwc(2, 3, 64, 64)
    w = _bf(64, 7, 7, 3, scale=0.05)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.stem7(x, w)                                     # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = ops.stem7(x, w)
    for scale in (0.5, -2.0):
        with torch.no_grad():
            w.copy_((w.float() * scale).bfloat16())
        g.replay()
        torch.cuda.synchronize()
        fb.check_bf16(y, *fb.conv_ref(x, w, 2, 3), 160, what="stem7 replay after update x%g" % scale)


def _train(base, graph, x, t, steps=4):
    """``steps`` optimizer steps from ``base``'s state; with a graph, one eager warm-up step and ``steps - 1`` replays."""
    m = to_train_dtype(copy.deepcopy(base), torch.bfloat16, DEV).train()
    tr = StudentTrainer(m, batch_size=x.shape[0], image_shape=tuple(x.shape[1:]), num_classes=t.shape[1], lr=0.1,
                        use_graph=graph)
    if graph:
        tr.static_x.copy_(x)
        tr.static_t.copy_(t)
        tr.capture(warmup=1)
        steps -= 1
    losses = [float(tr.step(x, t, sync=True).item()) for _ in range(steps)]
    torch.cuda.synchronize()
    return losses[-1], {k: v.detach().float().clone() for k, v in m.named_parameters()}


def test_graph_replay_matches_eager_steps():
    """Four optimizer steps through the captured graph (one eager warm-up step, three replays) against four eager steps
    from the same state.  Training in bf16 with atomically reduced BatchNorm statistics is not bit-reproducible and the
    differences grow step by step, so the yardstick is the spread of two eager runs: the graph run may not stray from an
    eager one by more than that."""
    torch.manual_seed(1)
    base = ResNet(18, class_dim=16)
    x = torch.randn(8, 3, 64, 64).bfloat16().contiguous(memory_format=torch.channels_last).pin_memory()
    t = torch.softmax(torch.randn(8, 16), -1).bfloat16().pin_memory()
    lg, pg = _train(base, True, x, t)
    le, pe = _train(base, False, x, t)
    le2, pe2 = _train(base, False, x, t)
    weights = [k for k in pe if k.endswith("weight") and pe[k].dim() > 1]

    def spread(p, q):
        return sum(((p[k] - q[k]).norm() / q[k].norm()).item() for k in weights) / len(weights)

    d_ge, d_ee = spread(pg, pe), spread(pe2, pe)
    assert d_ge <= 2.0 * d_ee + 2e-3, (d_ge, d_ee)
    assert abs(lg - le) <= 2.0 * abs(le2 - le) + 0.02 * abs(le), (lg, le, le2)


_STRICT = textwrap.dedent("""
    import sys
    import torch
    sys.path.insert(0, {root!r})
    from edl_b200 import ops
    from edl_b200.models import to_train_dtype
    from edl_b200.models.resnet import ResNet
    from edl_b200.trainer import StudentTrainer
    torch.manual_seed(0)
    m = to_train_dtype(ResNet({layers}, class_dim=16, width_mult={width}), torch.bfloat16, 'cuda').train()
    tr = StudentTrainer(m, batch_size=8, image_shape=(3, 64, 64), num_classes=16, lr=0.05, use_graph=True)
    x = torch.randn(8, 3, 64, 64).bfloat16().contiguous(memory_format=torch.channels_last).pin_memory()
    t = torch.softmax(torch.randn(8, 16), -1).bfloat16().pin_memory()
    loss = float(tr.step(x, t, sync=True).item())
    torch.cuda.synchronize()
    assert loss == loss, loss
    assert not ops.fallbacks(), ops.fallbacks()
    print('strict ok', loss)
""")


@pytest.mark.parametrize("layers,width", [(50, 0.5), (18, 1.0)])
def test_strict_native_captured_step(layers, width):
    """One captured training step with every library convolution an error (the switches are read at import, hence a
    subprocess).  The half-width ResNet50's 32-channel 3x3 convolutions of stage 1 need the pixel-pair form
    (EDL_OWN_STEM23=1)."""
    env = dict(os.environ, EDL_OWN_S2_BWD="1", EDL_OWN_WGRAD3="1", EDL_STRICT_NATIVE="1", EDL_OWN_STEM23="1")
    r = subprocess.run([sys.executable, "-c", _STRICT.format(root=ROOT, layers=layers, width=width)], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "strict ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_plain_resnet18_learns_with_graph():
    torch.manual_seed(0)
    m = to_train_dtype(ResNet(18, class_dim=16), torch.bfloat16, DEV).train()
    tr = StudentTrainer(m, batch_size=16, image_shape=(3, 32, 32), num_classes=16, lr=0.05, use_graph=True)
    x = torch.randn(16, 3, 32, 32).bfloat16().contiguous(memory_format=torch.channels_last).pin_memory()
    t = torch.zeros(16, 16)
    t[torch.arange(16), torch.arange(16)] = 1.0
    t = t.bfloat16().pin_memory()
    losses = [float(tr.step(x, t).item()) for _ in range(30)]
    assert losses[-1] < 0.5 * losses[0], losses
