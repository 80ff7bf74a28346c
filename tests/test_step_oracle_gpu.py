"""Whole training steps held layer by layer to the float64 oracle of tests/step_oracle.py: every activation, gradient
and update of ResNet50_vd, ResNet18_vd and plain ResNet50, in eager autograd steps under each BatchNorm mode, in the
trainer (side-stream weight gradients into the flat buckets, per-bucket optimizer) and replayed from its CUDA graph.

"No library" sets ``OWN_WGRAD3 = OWN_S2_BWD = OWN_STEM23 = True`` (all read at call time): the 3x3 and stride-2 weight
gradients, the stride-2 dgrads and the 32-channel stem convolutions then run on our kernels.  Worst ratios go to
``EDL_F64_BOUNDS_LOG`` like the other bounds tests."""
import copy

import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.models import ResNet, ResNet18_vd, ResNet50_vd, to_train_dtype
from edl_b200.ops import gemm as G
from edl_b200.trainer import StudentTrainer
from step_oracle import StepRecorder, bn_tau, check_sgd_step

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF16 = torch.bfloat16


def _no_library(monkeypatch):
    for flag in ("OWN_WGRAD3", "OWN_S2_BWD", "OWN_STEM23"):
        monkeypatch.setattr(G, flag, True)


def _model(ctor, seed=0, **kw):
    torch.manual_seed(seed)
    return to_train_dtype(ctor(**kw), BF16, DEV).train()


def _batch(n, size, classes, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, size, size, generator=g).to(BF16).contiguous(memory_format=torch.channels_last)
    t = torch.softmax(torch.randn(n, classes, generator=g) * 2, -1).to(BF16)
    return x.to(DEV), t.to(DEV)


def _eager_step(m, n, size, classes):
    """One forward / backward with the recorder attached; returns (recorder, report)."""
    x, t = _batch(n, size, classes)
    ops.reset_fallbacks()
    with StepRecorder(m) as rec:
        ops.soft_cross_entropy(m(x), t).backward()
    torch.cuda.synchronize()
    return rec, rec.check()


def _odd_stride2(rec):
    """Layers with no own kernel at any flag: the stride-2 3x3 convolution of an odd-sized input (7 x 7 at 112 x 112)."""
    return {r["name"] for r in rec.convs if r["unit"].stride == 2 and r["x"].shape[2] % 2}


def _assert_no_library(rec, report):
    """Nothing on the library but the stride-2 3x3 convolutions of odd-sized inputs, which no own kernel takes."""
    lib = {s.split(" (")[0] for s in report["library"]}
    assert lib <= _odd_stride2(rec), report["library"]
    assert all(k.startswith("conv ") and "3x3 stride 2" in k for k in ops.fallbacks()), ops.fallbacks()
    assert bool(lib) == bool(ops.fallbacks()), (report["library"], ops.fallbacks())


@pytest.mark.parametrize("no_lib", [False, True], ids=["default", "no-library"])
def test_resnet50_vd_224(monkeypatch, no_lib):
    if no_lib:
        _no_library(monkeypatch)
    rec, report = _eager_step(_model(ResNet50_vd, class_dim=1000), 4, 224, 1000)
    if no_lib:
        _assert_no_library(rec, report)
    else:
        assert report["library"], "the default flags leave the 3x3 weight gradients on the library"


BN_MODES = {"hooks-mask-bits": {}, "no-mask-bits": {"_RELU_MASK": False}, "no-fused-reduction": {"FUSE_BN_BWD": False},
            "sm-resident": {"_FUSED": True}}


@pytest.mark.parametrize("mode", list(BN_MODES))
def test_resnet50_vd_112_bn_modes(monkeypatch, mode):
    """7 -> 4 ceil-mode shortcuts, a stride-2 3x3 on 7 x 7 and partial tiles, in each BatchNorm mode."""
    _no_library(monkeypatch)
    for k, v in BN_MODES[mode].items():
        monkeypatch.setattr(G if k == "FUSE_BN_BWD" else ops.bn, k, v)
    rec, report = _eager_step(_model(ResNet50_vd, class_dim=104), 8, 112, 104)
    _assert_no_library(rec, report)
    hooks = [b for b in rec.bns if getattr(b["ctx"], "hook", None) is not None and b["ctx"].hook.done]
    if mode == "hooks-mask-bits":
        assert hooks and any(b["saved_y"] is not None and b["saved_y"].dtype == torch.uint8 for b in rec.bns)
    if mode in ("no-fused-reduction", "sm-resident"):
        assert not hooks, [b["name"] for b in hooks]


@pytest.mark.parametrize("no_lib", [False, True], ids=["default", "no-library"])
def test_resnet18_vd_basic_blocks(monkeypatch, no_lib):
    if no_lib:
        _no_library(monkeypatch)
    rec, report = _eager_step(_model(ResNet18_vd, class_dim=104), 8, 64, 104)
    if no_lib:
        _assert_no_library(rec, report)


def test_plain_resnet50_stem7_and_projections(monkeypatch):
    _no_library(monkeypatch)
    rec, report = _eager_step(_model(ResNet, layers=50, class_dim=1000), 4, 224, 1000)
    _assert_no_library(rec, report)
    kinds = {r["kind"] for r in rec.convs}
    assert {"_Stem7FnBackward", "_Conv1x1S2FnBackward"} <= kinds, kinds


def test_negative_control_missing_drop_bn_hook(monkeypatch):
    """Without ``drop_bn_hook`` the 3x3 conv a of a BasicBlock computes the BatchNorm-backward sums of its input from its
    own gradient only, not from the shortcut's as well: the oracle must name that BatchNorm.  (Without mask bits the 3x3
    dgrad takes the hook; with them it never does.)"""
    monkeypatch.setattr(ops, "drop_bn_hook", lambda t: t)
    monkeypatch.setattr(ops.bn, "_RELU_MASK", False)
    with pytest.raises(AssertionError, match=r"blocks\.\d+\.b bn (dgamma|dbeta|dx)"):
        _eager_step(_model(ResNet18_vd, class_dim=104), 8, 64, 104)


# ---------------------------------------------------------------------------------------------------------- trainer
def _snapshot(tr):
    return {dt: ((g.master if g.master is not None else g.param).clone(), tr.opt.state[dt]["mom"].clone())
            for dt, g in tr.dp.flat.groups.items()}


def _check_trainer_step(tr, rec, snap, what):
    torch.cuda.synchronize()
    report = rec.check()
    _assert_no_library(rec, report)
    assert any(getattr(p, "_edl_grad_sink", None) is not None for p in tr.model.parameters())
    check_sgd_step(tr.dp.flat, tr.opt, snap, tr.opt.lr_t.item(), fb.f32(0.9), fb.f32(1e-4), what=what)
    return report


def test_trainer_eager_and_graph_replays(monkeypatch):
    """StudentTrainer with the per-bucket optimizer on the side stream: one eager step, then a graph captured with the
    recorder attached, checked after replays 1 and 3.  Every bucket window must hold the gradient the oracle accepts and
    every master weight, parameter and momentum must follow the float64 SGD rule applied to that gradient: an optimizer
    that read a bucket before its last side-stream weight gradient landed fails."""
    _no_library(monkeypatch)
    m = _model(ResNet50_vd, class_dim=104)
    tr = StudentTrainer(m, batch_size=8, image_shape=(3, 112, 112), num_classes=104, lr=0.05, weight_decay=1e-4,
                        use_graph=True)
    assert tr.dp.bucket_opt
    rec = StepRecorder(m).attach()
    body = tr._step_body

    def recorded_body():
        rec.reset()
        body()
    tr._step_body = recorded_body
    try:
        x, t = _batch(8, 112, 104)
        tr.use_graph = False
        ops.reset_fallbacks()
        snap = _snapshot(tr)
        tr.step(x, t, sync=True)
        _check_trainer_step(tr, rec, snap, "eager step")
        tr.use_graph = True
        ops.reset_fallbacks()
        tr.capture(warmup=1)
        for i in (1, 2, 3):
            x, t = _batch(8, 112, 104, seed=10 + i)
            tr.static_x.copy_(x)
            tr.static_t.copy_(t)
            torch.cuda.synchronize()
            snap = _snapshot(tr)
            tr.graph.replay()
            if i != 2:
                _check_trainer_step(tr, rec, snap, "replay %d" % i)
    finally:
        tr._step_body = body
        rec.detach()


# -------------------------------------------------------------------------------------------------------- recompute
def test_recompute_updates_running_statistics_once():
    """``recompute=True`` runs every block's forward again during backward.  The running statistics after one step must
    be one momentum update from the first forward's batch statistics.  The recorder cannot read the first forward's
    saved tensors (checkpointing drops them), so the parameter gradients are held to twice the run-to-run spread of two
    plain steps instead of the layer-by-layer oracle."""
    torch.manual_seed(0)
    base = ResNet50_vd(class_dim=104)
    x, t = _batch(8, 112, 104)

    def run(recompute):
        m = to_train_dtype(copy.deepcopy(base), BF16, DEV).train()
        m.recompute = recompute
        seen = []

        def pre(bn, args):
            if not ops.bn._RECOMPUTING:
                seen.append([bn, bn.running_mean.clone(), bn.running_var.clone()])

        def post(bn, args, out):
            if not ops.bn._RECOMPUTING:
                seen[-1].append(args[0].detach().clone())
        hs = [h for u in m.conv_bn_units() for h in (u.bn.register_forward_pre_hook(pre), u.bn.register_forward_hook(post))]
        ops.soft_cross_entropy(m(x), t).backward()
        torch.cuda.synchronize()
        for h in hs:
            h.remove()
        return m, seen

    mr, seen = run(True)
    assert len(seen) == len(mr.conv_bn_units())
    names = {bn: n for n, bn in mr.named_modules()}
    for bn, rm0, rv0, xin in seen:
        c = bn.num_features
        m = xin.numel() // c
        fb.check_bn_running_e2e(xin, rm0, rv0, bn.running_mean, bn.running_var, bn.momentum, bn_tau(m, c),
                                what=names[bn])
    (m1, _), (m2, _) = run(False), run(False)
    grads = {n: [p.grad.float() for p in (dict(mm.named_parameters())[n] for mm in (mr, m1, m2))]
             for n, _ in mr.named_parameters()}

    def rel(a, b):
        return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()
    d_rc = sum(rel(g[0], g[1]) for g in grads.values()) / len(grads)
    d_pp = sum(rel(g[2], g[1]) for g in grads.values()) / len(grads)
    assert d_rc <= 2.0 * d_pp + 1e-3, (d_rc, d_pp)
