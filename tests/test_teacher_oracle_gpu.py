"""The ResNeXt teacher's inference forward on the GPU kernels, layer by layer against float64 (tests/teacher_oracle.py),
with a random folded BatchNorm in every layer and a nonzero classifier bias: ResNeXt101_32x16d (bf16 with the residual
fused and unfused, FP8 block, FP8 per-tensor run on a batch twice the calibration batch so that the saturation is live),
ResNeXt50_32x4d (bf16 and FP8 block, its 4-channel groups widened 16-way, and one CUDA-graph replay), ResNeXt_tiny at
odd sizes and with the stride-2 kernel off, and negative controls that the oracle must name."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import teacher_oracle as T  # noqa: E402
from edl_b200 import ops  # noqa: E402
from edl_b200.models import resnext, teacher_zoo  # noqa: E402

DEV = torch.device("cuda", 0)


def _model(ctor, seed=0, **kw):
    torch.manual_seed(seed)
    m = resnext.to_inference_dtype(ctor(**kw), torch.bfloat16, DEV).eval()
    T.random_bn(m, seed + 1)
    return m


def _image(n, h, w, seed=3, scale=1.0):
    x = torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(seed)) * scale
    return x.to(DEV).bfloat16().contiguous(memory_format=torch.channels_last)


def _run(model, x, what, probs=False, library=False):
    """One recorded forward, judged; returns (recorder, worst ratios per category).  ``library``: grouped 3x3 layers the
    kernels do not take (ResNeXt_tiny's 2- and 4-channel groups) may run on the library, and only those."""
    top = teacher_zoo._Probs(model) if probs else model
    ops.reset_fallbacks()
    with T.TeacherRecorder(top) as rec:
        top(x)
    torch.cuda.synchronize()
    lib = [n for n, p in rec.paths().items() if p == "library"]
    if library:
        assert all(r.startswith("teacher conv on cuDNN: 3x3") for r in ops.fallbacks()), ops.fallbacks()
        assert sum(ops.fallbacks().values()) == len(lib), (ops.fallbacks(), lib)
    else:
        assert ops.fallbacks() == {} and not lib, (ops.fallbacks(), lib)
    worst = rec.check(log=print)                     # the worst criterion-1 ratio of every FP8 layer
    for cat, (c1, c2) in sorted(worst.items()):
        print("%s %s: worst c1 %.3f, c2 %.2f" % (what, cat, c1, c2))
    return rec, worst


def _paths(rec):
    return rec.paths()


def _assert_stage_rms(rec, model, what):
    rms = T.stage_rms(rec, model)
    print(what, "stage RMS", {k: round(v, 3) for k, v in rms.items()})
    assert all(2.0 ** -8 < v < 2.0 ** 8 for v in rms.values()), rms


def _by_stage(model):
    """[(stage index, block)] for the blocks of ``model``."""
    out, st = [], 0
    for i, b in enumerate(model.blocks):
        if i > 0 and b.ds is not None:
            st += 1
        out.append((st, b))
    return out


def test_resnext101_32x16d_bf16_fp8_block_and_tensor(monkeypatch):
    model = _model(resnext.ResNeXt101_32x16d)
    x = _image(2, 224, 224)
    for fuse in (True, False):
        monkeypatch.setattr(resnext, "FUSE_RESIDUAL", fuse)
        rec, _ = _run(model, x, "resnext101 bf16 fuse=%d" % fuse, probs=True)
        p = _paths(rec)
        assert p["stem"] == "stem7"
        for st, b in _by_stage(model):
            name = rec.convs[b.c2].name
            first = b.ds is not None and st > 0
            want = ("widened, " if st < 2 else "") + ("s2" if first else "s1")
            assert p[name] == want, (name, p[name], want)
            assert p[rec.convs[b.c3].name] == ("fused residual" if fuse else "two-kernel residual")
            assert p[rec.convs[b.c1].name] == "1x1"
        if fuse:
            _assert_stage_rms(rec, model, "resnext101")
    monkeypatch.setattr(resnext, "FUSE_RESIDUAL", True)

    assert model.enable_fp8(scaling="block") == 70          # every 1x1 convolution: 33 blocks x 2 + 4 projections
    rec, _ = _run(model, x, "resnext101 fp8 block")
    paths = set(_paths(rec).values())
    assert {"fp8 block", "fp8 block, residual"} <= paths and "1x1" not in paths and "fused residual" not in paths

    calib = _image(2, 224, 224, seed=4)
    assert model.enable_fp8(calib, scaling="tensor") == 70
    rec, _ = _run(model, x * 2, "resnext101 fp8 tensor (input x2)")
    paths = set(_paths(rec).values())
    assert {"fp8 tensor", "fp8 tensor, residual"} <= paths
    # the doubled input saturates: some quantised operands hold +-448
    sat = sum(int(((r.x8 & 0x7F) == 0x7E).sum()) for r in rec.convs.values() if r.path.startswith("fp8 tensor"))
    assert sat > 0


def test_resnext50_32x4d_bf16_and_fp8_block():
    model = _model(resnext.ResNeXt50_32x4d)
    x = _image(4, 224, 224)
    rec, _ = _run(model, x, "resnext50 bf16", probs=True)
    p = _paths(rec)
    for st, b in _by_stage(model):                   # 4, 8, 16, 32 channels per group: every stage is widened
        first = b.ds is not None and st > 0
        assert p[rec.convs[b.c2].name] == "widened, " + ("s2" if first else "s1")
    assert model.blocks[0].c2.weight.shape[3] == 4                          # 4-channel groups, widened 16-way
    assert model.enable_fp8(scaling="block") == 36
    _run(model, x, "resnext50 fp8 block")


@pytest.mark.parametrize("h,w", [(61, 83), (33, 47)])
def test_resnext_tiny_odd_sizes(h, w):
    model = _model(resnext.ResNeXt_tiny)
    rec, _ = _run(model, _image(2, h, w), "resnext_tiny %dx%d" % (h, w), probs=True, library=True)
    p = _paths(rec)
    print(p)
    firsts = [b.c2 for st, b in _by_stage(model) if b.ds is not None and st > 0]
    assert any(p[rec.convs[c].name].endswith("subsample") for c in firsts), p


def test_resnext_tiny_without_the_stride2_kernel(monkeypatch):
    monkeypatch.setattr(ops.gemm, "CONV3_S2", False)
    model = _model(resnext.ResNeXt_tiny)
    rec, _ = _run(model, _image(2, 64, 64), "resnext_tiny 64x64 no CONV3_S2", library=True)
    p = _paths(rec)
    print(p)
    assert not any(v.endswith("s2") for v in p.values()), p           # no layer takes the stride-2 kernel
    for st, b in _by_stage(model):
        if b.ds is not None and st > 0:
            assert p[rec.convs[b.c2].name].endswith("subsample") or p[rec.convs[b.c2].name] == "library", p
    assert "widened, subsample" in p.values(), p


def test_resnext50_fp8_block_graph_replay():
    model = _model(resnext.ResNeXt50_32x4d)
    model.enable_fp8(scaling="block")
    static = _image(2, 128, 128)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model(static)
    torch.cuda.current_stream().wait_stream(s)
    rec = T.TeacherRecorder(model)
    g = torch.cuda.CUDAGraph()
    with rec:
        with torch.cuda.graph(g):
            model(static)
    static.copy_(_image(2, 128, 128, seed=9))
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(rec.convs[model.stem].x, static)
    worst = rec.check(log=print)
    print("resnext50 fp8 block graph replay", worst)


def test_oracle_negative_controls(monkeypatch):
    model = _model(resnext.ResNeXt50_32x4d)
    x = _image(2, 64, 64)
    orig = resnext.FoldedConv._widened_groups

    def swapped(self):
        r = orig(self)
        if r is None:
            return r
        w64, g = r
        c = self.weight.shape[3]
        w = w64.clone()
        w[..., :c], w[..., c:2 * c] = w64[..., c:2 * c], w64[..., :c]      # two sub-groups trade input channels
        return w, g

    monkeypatch.setattr(resnext.FoldedConv, "_widened_groups", swapped)
    with T.TeacherRecorder(model) as rec:
        model(x)
    with pytest.raises(AssertionError, match=r"blocks\.0\.c2 \(widened, s1\)"):
        rec.check(log=lambda s: None)
    monkeypatch.setattr(resnext.FoldedConv, "_widened_groups", orig)

    with T.TeacherRecorder(model) as rec:
        model(x)
    rec.check(log=lambda s: None)
    r = rec.convs[model.blocks[4].c1]
    ch = int(r.out.amax((0, 2, 3)).argmax())
    r.shift[ch] += 0.02
    with pytest.raises(AssertionError, match=r"blocks\.4\.c1 \(1x1\)"):
        rec.check(log=lambda s: None)


def _same_act_scales(dst, src):
    """Give ``dst``'s per-tensor FP8 layers the calibrated activation scales of ``src``'s."""
    for a, b in zip(src.modules(), dst.modules()):
        if isinstance(a, resnext.FoldedConv) and a._fp8 == "tensor":
            b.act_scale = a.act_scale.to(DEV).clone()


@pytest.mark.parametrize("scaling", ["block", "tensor"])
def test_fp8_teacher_after_a_load_and_a_move(scaling):
    """The FP8 weights follow a ``load_state_dict`` + ``load_bn`` and a move from the CPU: the logits equal those of a
    model enabled directly on the loaded weights on the GPU (with the same calibrated activation scales)."""
    x, calib = _image(2, 64, 64), _image(2, 64, 64, seed=5)
    model = _model(resnext.ResNeXt50_32x4d, seed=0)
    model.enable_fp8(calib, scaling=scaling)
    model(x)                                             # quantised weights of the first state are in use
    other = _model(resnext.ResNeXt50_32x4d, seed=10)
    model.load_state_dict(other.state_dict())
    T.random_bn(model, 20)
    T.random_bn(other, 20)
    other.enable_fp8(calib, scaling=scaling)
    _same_act_scales(other, model)
    ops.reset_fallbacks()
    got = model(x)
    assert ops.fallbacks() == {}, ops.fallbacks()
    assert torch.equal(got, other(x)), "stale FP8 weights after load_state_dict / load_bn"

    torch.manual_seed(10)
    cpu = resnext.to_inference_dtype(resnext.ResNeXt50_32x4d(), torch.bfloat16, "cpu")
    T.random_bn(cpu, 11)
    cpu.enable_fp8(calib.cpu(), scaling=scaling)          # quantised (and calibrated) on the CPU
    moved = resnext.to_inference_dtype(cpu, torch.bfloat16, DEV)
    ref = _model(resnext.ResNeXt50_32x4d, seed=10)
    ref.load_state_dict(moved.state_dict())              # the BatchNorm as folded on the CPU, bit for bit
    ref.enable_fp8(calib, scaling=scaling)
    _same_act_scales(ref, moved)
    got = moved(x)
    for c in moved.modules():
        if isinstance(c, resnext.FoldedConv) and c._fp8 is not None:
            assert c._fp8_weights()[0].is_cuda and (c._fp8 != "tensor" or c.act_scale.is_cuda)
    assert torch.equal(got, ref(x)), "FP8 weights not re-quantised on the new device"
