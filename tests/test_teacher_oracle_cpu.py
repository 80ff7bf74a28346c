"""The ResNeXt teacher oracle (tests/teacher_oracle.py) on the CPU: the recorder on an fp32 ResNeXt_tiny (library
path), its path classification and how it reports a wrong layer; and the FP8 weights re-quantised after a load."""
import copy

import pytest
import torch

import teacher_oracle as T
from edl_b200.models import resnext, teacher_zoo
from edl_b200.ops import fp8


def _tiny(seed=0):
    torch.manual_seed(seed)
    m = resnext.ResNeXt_tiny().eval()
    T.random_bn(m, seed + 1)
    return m


def _image(n, h, w, seed=2):
    return torch.randn(n, 3, h, w, generator=torch.Generator().manual_seed(seed)).contiguous(memory_format=torch.channels_last)


def test_recorder_on_cpu_resnext_tiny():
    model = teacher_zoo._Probs(_tiny())
    with T.TeacherRecorder(model) as rec:
        probs = model(_image(2, 61, 83))
    assert set(rec.paths().values()) == {"library"}
    assert all(r.runs == 1 for r in rec.convs.values())
    assert torch.equal(rec.probs, probs)
    worst = rec.check()
    assert set(worst) >= {"library", "pools", "classifier", "softmax"}
    rms = T.stage_rms(rec, model.net)
    assert list(rms) == ["stem", "stage 1", "stage 2", "stage 3", "stage 4"]
    assert all(2.0 ** -8 < v < 2.0 ** 8 for v in rms.values()), rms
    assert float(model.net.fc_bias.abs().max()) > 0


def test_recorder_counts_runs_and_restores_ops():
    from edl_b200 import ops

    model = _tiny()
    orig = ops.gemm_bf16
    with T.TeacherRecorder(model) as rec:
        x = _image(1, 32, 32)
        model(x)
        model(x)
    assert ops.gemm_bf16 is orig and fp8.gemm_fp8.__name__ == "gemm_fp8"
    with pytest.raises(AssertionError, match="exactly once"):
        rec.check()


def test_path_classification():
    c3 = resnext.FoldedConv(64, 64, 3, stride=2, groups=4)
    c1 = resnext.FoldedConv(64, 64, 1)
    cases = [
        ([("conv3x3_s2_infer", {"widened": True})], c3, "widened, s2"),
        ([("conv3x3_s2_infer", {"widened": False})], c3, "s2"),
        ([("conv3x3_infer", {"widened": False})], c3, "subsample"),
        ([("conv3x3_infer", {"widened": True})], resnext.FoldedConv(64, 64, 3, groups=16), "widened, s1"),
        ([("stem7_infer", {})], c3, "stem7"),
        ([("gemm_bf16", {"add": True})], c1, "fused residual"),
        ([("gemm_bf16", {"add": False}), ("scale_shift_act", {})], c1, "two-kernel residual"),
        ([("gemm_bf16", {"add": False})], c1, "1x1"),
        ([("quantize_e4m3_blocks", {}), ("gemm_fp8_blockscaled", {})], c1, "fp8 block"),
        ([("quantize_e4m3", {}), ("gemm_fp8", {}), ("scale_shift_act", {})], c1, "fp8 tensor, residual"),
        ([("scale_shift_act", {})], c3, "library"),
    ]
    for calls, conv, want in cases:
        assert T.classify(calls, conv) == want, (calls, want)


def test_negative_control_names_the_layer():
    model = _tiny()
    with T.TeacherRecorder(model) as rec:
        model(_image(2, 33, 47))
    rec.check()
    target = model.blocks[2].c2
    r = rec.convs[target]
    ch = int(r.out.amax((0, 2, 3)).argmax())            # a channel the ReLU leaves alive
    r.shift[ch] += 0.25                                  # one channel of the recorded shift
    with pytest.raises(AssertionError, match=r"blocks\.2\.c2 \(library\)"):
        rec.check()


# ------------------------------------------------------------------------------------------ FP8 weights after a load
def _loaded_copy(model, seed):
    """The state of a differently initialised model, and new BatchNorm statistics for every layer."""
    other = _tiny(seed)
    bn = {}
    gen = torch.Generator().manual_seed(seed)
    for name, m in other.named_modules():
        if isinstance(m, resnext.FoldedConv):
            c = m.cout
            bn[name] = (torch.rand(c, generator=gen) + 0.5, torch.randn(c, generator=gen) * 0.1,
                        torch.randn(c, generator=gen) * 0.1, torch.rand(c, generator=gen) + 0.5)
    return other.state_dict(), bn


def _load(model, state, bn):
    model.load_state_dict(state)
    for name, m in model.named_modules():
        if name in bn:
            m.load_bn(*bn[name])


@pytest.mark.parametrize("scaling", ["block", "tensor"])
def test_fp8_weights_requantised_after_load(scaling):
    model = _tiny()
    calib = _image(2, 32, 32)
    n = model.enable_fp8(calib, scaling=scaling)
    assert n > 0
    convs = {name: m for name, m in model.named_modules() if isinstance(m, resnext.FoldedConv) and m.fp8_eligible()}
    before = {name: m._fp8_weights()[0].clone() for name, m in convs.items()}
    act = {name: getattr(m, "act_scale", None) for name, m in convs.items()}
    state, bn = _loaded_copy(model, 7)
    _load(model, state, bn)

    fresh = _tiny(7)
    _load(fresh, state, bn)
    fresh.enable_fp8(calib, scaling=scaling)
    fresh_convs = dict(fresh.named_modules())
    changed = 0
    for name, m in convs.items():
        f = fresh_convs[name]
        if scaling == "block":
            assert torch.equal(m.w8_blocks, f.w8_blocks), name
            assert torch.equal(m.w_block_scales, f.w_block_scales), name
            assert m.w8 is None
        else:
            assert torch.equal(m.w8, f.w8), name
            assert m.act_scale is act[name] or torch.equal(m.act_scale, act[name])     # the calibration is kept
            q, ws = fp8.quantize_weight_rows(m.weight.view(m.cout, m.cin))
            assert torch.equal(m.deq_scale, (act[name] * ws * m.scale).contiguous()), name
            assert m.w8_blocks is None
        changed += int(not torch.equal(m._fp8_weights()[0], before[name]))
    assert changed == len(convs)

    # load_bn alone changes the per-tensor dequantisation scale (it carries the folded-BN scale)
    if scaling == "tensor":
        m = next(iter(convs.values()))
        old = m.deq_scale.clone()
        m.load_bn(torch.full((m.cout,), 2.0), torch.zeros(m.cout), torch.zeros(m.cout), torch.ones(m.cout))
        _, ws = fp8.quantize_weight_rows(m.weight.view(m.cout, m.cin))
        assert not torch.equal(m.deq_scale, old)
        assert torch.equal(m.deq_scale, (m.act_scale * ws * m.scale).contiguous())


def test_fp8_mode_switch_and_deepcopy():
    model = _tiny()
    model.enable_fp8(scaling="block")
    conv = model.blocks[0].c1
    assert conv.w8_blocks is not None and conv.w8 is None
    model.enable_fp8(_image(1, 32, 32), scaling="tensor")
    assert conv.w8 is not None and conv.w8_blocks is None
    twin = copy.deepcopy(model)
    assert torch.equal(twin.blocks[0].c1.w8, conv.w8)


@pytest.mark.parametrize("how", ["batch", "margin", "act_scale"])
def test_fp8_tensor_recalibration_rebuilds_the_dequantisation_scale(how):
    model = _tiny()
    x = _image(2, 32, 32)
    model.enable_fp8(x)
    convs = [m for m in model.modules() if isinstance(m, resnext.FoldedConv) and m.w8 is not None]
    old = {m: (m.act_scale.clone(), m.deq_scale.clone()) for m in convs}
    if how == "batch":
        model.enable_fp8(4 * x)
    elif how == "margin":
        model.enable_fp8(x, margin=0.5)
    else:
        for m in convs:
            m.act_scale.mul_(3)                          # an in-place change of the activation scale
    for m in convs:
        _, ws = fp8.quantize_weight_rows(m.weight.view(m.cout, m.cin))
        assert not torch.equal(m.act_scale, old[m][0])
        assert torch.equal(m.deq_scale, (m.act_scale * ws * m.scale).contiguous()), m
        assert not torch.equal(m.deq_scale, old[m][1])
