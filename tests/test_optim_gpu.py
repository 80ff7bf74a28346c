"""Optimizer kernels (csrc/optim.cu: sgd_momentum, adam_step, grad_sqnorm, clip_scale) and the one-GPU training step
that uses them, against float64 references.

Each reference step starts from the kernel's own previous state, so error does not accumulate and the bounds stay
tight.  Constants are rounded to float32 first, as the kernels receive them.  |upd| and |m| in the bounds stand for the
sum of the magnitudes of their terms, so a cancellation inside a term does not shrink the bound below the rounding
error of its parts.  The CPU tests check the same references against the CPU branches of ``FlatSGDMomentum`` /
``FlatAdam`` and against ``ElasticDataParallel._clip_cpu``, and run without a GPU."""
import itertools
import math
from types import SimpleNamespace

import pytest
import torch

from edl_b200 import ops
from edl_b200.parallel import FlatParams
from edl_b200.parallel.ddp import ElasticDataParallel

gpu = pytest.mark.gpu
DEV = "cuda"
BF16, F32 = torch.bfloat16, torch.float32


def f32(x):
    return torch.tensor(x, dtype=F32).item()


def ulp32(x):
    _, e = torch.frexp(x)
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 24))


# ---------------------------------------------------------------------------------------------------- references
def ref_sgd(w, v, g, lr, mu, wd, nesterov=False, gs=1.0, mask=None):
    """One SGD-momentum step in float64.  Returns (w, v) and their bounds:
    |dw| <= 1e-6 (|w| + lr |upd|), |dv| <= 1e-6 (mu |v| + |g s| + wd |w|)."""
    w, v, g = w.double(), v.double(), g.double()
    wdv = wd * mask.double() if mask is not None else wd
    gg = g * gs + wdv * w
    v1 = mu * v + gg
    upd = mu * v1 + gg if nesterov else v1
    mag_v = mu * v.abs() + (g * gs).abs() + (wdv * w).abs()
    mag_upd = mag_v * (1 + mu) if nesterov else mag_v
    return w - lr * upd, v1, 1e-6 * (w.abs() + lr * mag_upd), 1e-6 * mag_v


def ref_adam(w, m, v, g, t, lr, b1, b2, eps, wd, decoupled, gs=1.0):
    """One Adam step at step count t in float64.  Returns (w, m, v) and their bounds:
    |dw| <= 1e-5 lr |mhat| / (sqrt(vhat) + eps) + 2 ulp(w), |dm| <= 1e-6 |m|, |dv| <= 1e-6 v."""
    w, m, v, g = w.double(), m.double(), v.double(), g.double()
    mag_g = (g * gs).abs()
    g = g * gs
    if not decoupled:
        mag_g = mag_g + wd * w.abs()
        g = g + wd * w
    m1 = b1 * m + (1 - b1) * g
    mag_m = b1 * m.abs() + (1 - b1) * mag_g
    v1 = b2 * v + (1 - b2) * g * g
    den = (v1 / (1 - b2 ** t)).sqrt() + eps
    w1 = (w - lr * wd * w if decoupled else w) - lr * (m1 / (1 - b1 ** t)) / den
    tol_w = 1e-5 * lr * (mag_m / (1 - b1 ** t)) / den + 2 * ulp32(torch.maximum(w.abs(), w1.abs()))
    return w1, m1, v1, tol_w, 1e-6 * mag_m, 1e-6 * v1


def ref_clip_scale(norm, max_norm):
    """The global-norm clip factor: applied only to a finite norm above max_norm (a non-finite one is left to the
    found_inf machinery)."""
    return max_norm / (norm + 1e-6) if math.isfinite(norm) and norm > max_norm else 1.0


def assert_close(got, ref, tol, what):
    bad = ~((got.double() - ref.to(got.device)).abs() <= tol.to(got.device))
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d of %d elements out of bounds, first at %d: got %r, ref %r, tol %r" % (
            what, int(bad.sum()), bad.numel(), i, got[i].item(), ref[i].item(), tol[i].item()))


def _bits(*ts):
    return [t.clone().view(torch.int16 if t.element_size() == 2 else torch.int32) for t in ts]


def _same_bits(before, ts):
    return all(torch.equal(a, b) for a, b in zip(before, _bits(*ts)))


def _mixed_model(dev):
    """A bf16 group (with an fp32 master) and an fp32 group (updated in place)."""
    torch.manual_seed(0)
    m = torch.nn.Sequential(torch.nn.Linear(37, 61), torch.nn.Linear(61, 9)).to(dev)
    for lin in m:
        lin.weight.data = lin.weight.data.to(BF16)
    return m


def _fill_grads(flat, gen):
    for g in flat.groups.values():
        g.grad.copy_(torch.randn(g.numel, generator=gen).to(g.grad.device).to(g.dtype))


# ---------------------------------------------------------------------------------------------------- CPU: the yardsticks
@pytest.mark.parametrize("nesterov,masked,scaled", [(False, False, False), (True, True, True), (True, False, True),
                                                    (False, True, False)])
def test_ref_sgd_matches_cpu_step(nesterov, masked, scaled):
    flat = FlatParams(_mixed_model("cpu"))
    opt = ops.FlatSGDMomentum(flat, lr=0.1, momentum=0.9, weight_decay=0.05, nesterov=nesterov,
                              decay_filter=(lambda name, p: p.dim() > 1) if masked else None)
    gs = 0.25 if scaled else 1.0
    if scaled:
        opt.set_grad_scale(torch.full((1,), gs))
    gen = torch.Generator().manual_seed(1)
    for _ in range(3):
        _fill_grads(flat, gen)
        snap = {dt: ((g.master if g.master is not None else g.param).clone(), opt.state[dt]["mom"].clone())
                for dt, g in flat.groups.items()}
        opt.step()
        for dt, g in flat.groups.items():
            master = g.master if g.master is not None else g.param
            w, v, tw, tv = ref_sgd(*snap[dt], g.grad, 0.1, 0.9, 0.05, nesterov, gs, opt.state[dt]["wd_mask"])
            assert_close(master, w, tw, "master %s" % dt)
            assert_close(opt.state[dt]["mom"], v, tv, "momentum %s" % dt)
    opt.set_found_inf(torch.ones(1, dtype=torch.int32))
    before = _bits(*[t for g in flat.groups.values() for t in (g.param, g.master) if t is not None])
    opt.step()
    assert _same_bits(before, [t for g in flat.groups.values() for t in (g.param, g.master) if t is not None])


@pytest.mark.parametrize("decoupled", [True, False])
@pytest.mark.parametrize("scaled", [False, True])
def test_ref_adam_matches_cpu_step(decoupled, scaled):
    flat = FlatParams(_mixed_model("cpu"))
    opt = ops.FlatAdam(flat, lr=1e-2, weight_decay=0.05, decoupled=decoupled)
    gs = 0.5 if scaled else 1.0
    if scaled:
        opt.set_grad_scale(torch.full((1,), gs))
    gen = torch.Generator().manual_seed(2)
    for it in range(3):
        _fill_grads(flat, gen)
        snap = {dt: ((g.master if g.master is not None else g.param).clone(), opt.state[dt]["m"].clone(),
                     opt.state[dt]["v"].clone()) for dt, g in flat.groups.items()}
        opt.step()
        assert opt.step_t.item() == it + 1
        for dt, g in flat.groups.items():
            master = g.master if g.master is not None else g.param
            w, m, v, tw, tm, tv = ref_adam(*snap[dt], g.grad, it + 1, 1e-2, 0.9, 0.999, 1e-8, 0.05, decoupled, gs)
            assert_close(master, w, tw, "master %s" % dt)
            assert_close(opt.state[dt]["m"], m, tm, "m %s" % dt)
            assert_close(opt.state[dt]["v"], v, tv, "v %s" % dt)


def _clip_cpu(grads, max_norm):
    dp = SimpleNamespace(flat=SimpleNamespace(groups={i: SimpleNamespace(grad=g) for i, g in enumerate(grads)}),
                         clip_norm=max_norm)
    ElasticDataParallel._clip_cpu(dp)
    return dp.last_grad_norm


@pytest.mark.parametrize("case", ["below", "above", "nan", "inf"])
def test_ref_clip_matches_cpu_clip(case):
    gen = torch.Generator().manual_seed(3)
    grads = [torch.randn(100, generator=gen) * 0.05, torch.randn(37, generator=gen).to(BF16) * 0.05]
    if case == "above":
        grads[1] *= 100
    if case in ("nan", "inf"):
        grads[0][5] = float(case)
    before = [g.clone() for g in grads]
    norm = _clip_cpu(grads, 1.0)
    norm64 = math.sqrt(sum((g.double() ** 2).sum().item() for g in before))
    if math.isfinite(norm64):
        assert abs(norm - norm64) <= 1e-5 * norm64
    else:
        assert math.isnan(norm) == math.isnan(norm64) and math.isinf(norm) == math.isinf(norm64)
    scale = ref_clip_scale(norm, 1.0)
    assert (scale < 1.0) == (case == "above")
    for g, b in zip(grads, before):
        if scale == 1.0:
            assert torch.equal(g.view(torch.int16 if g.dtype == BF16 else torch.int32),
                               b.view(torch.int16 if b.dtype == BF16 else torch.int32))
        else:
            assert torch.equal(g, b * scale) or torch.equal(g, (b.float() * scale).to(b.dtype))


# ---------------------------------------------------------------------------------------------------- C. kernels
def _sgd_cases():
    ns = [1, 7, 8, 4096 + 3, 3 * 2 ** 20 + 5]
    combos = itertools.product([BF16, F32], [True, False], [True, False], [False, True], [None, 0.25])
    out = []
    for i, (gdt, lp, mask, nest, gs) in enumerate(combos):
        n = ns[i % 5]
        out.append(pytest.param(gdt, lp, mask, nest, gs, n, id="%s-n%d%s%s%s%s" % (
            "bf16" if gdt == BF16 else "fp32", n, "-lp" if lp else "", "-mask" if mask else "",
            "-nesterov" if nest else "", "-gs" if gs else "")))
    return out


@gpu
@pytest.mark.parametrize("gdt,with_lp,with_mask,nesterov,gs,n", _sgd_cases())
def test_sgd_momentum_kernel(gdt, with_lp, with_mask, nesterov, gs, n):
    """Three steps through the vector body, the scalar tail and (for 3 * 2^20 + 5) the grid-stride loop beyond the
    grid cap; then a step with found_inf raised leaves every buffer bit-identical."""
    C = ops.native()
    gen = torch.Generator(device=DEV).manual_seed(n)
    master = torch.randn(n, device=DEV, generator=gen)
    mom = torch.randn(n, device=DEV, generator=gen) * 0.1
    lp = master.to(BF16) if with_lp else None
    mask = (torch.rand(n, device=DEV, generator=gen) < 0.5).float() if with_mask else None
    lr_t = torch.full((1,), 0.1, device=DEV)
    gs_t = torch.full((1,), gs, device=DEV) if gs else None
    mu, wd = 0.9, 0.05
    for _ in range(3):
        grad = torch.randn(n, device=DEV, generator=gen).to(gdt)
        w0, v0 = master.clone(), mom.clone()
        C.sgd_momentum(lp, master, mom, grad, mask, lr_t, gs_t, None, mu, wd, nesterov)
        w, v, tw, tv = ref_sgd(w0, v0, grad, lr_t.item(), f32(mu), f32(wd), nesterov, gs or 1.0, mask)
        assert_close(master, w, tw, "master")
        assert_close(mom, v, tv, "momentum")
        if lp is not None:
            assert torch.equal(lp, master.to(BF16))
    inf_t = torch.ones(1, dtype=torch.int32, device=DEV)
    keep = [master, mom] + ([lp] if lp is not None else [])
    before = _bits(*keep)
    C.sgd_momentum(lp, master, mom, torch.randn(n, device=DEV).to(gdt), mask, lr_t, gs_t, inf_t, mu, wd, nesterov)
    assert _same_bits(before, keep)


@gpu
@pytest.mark.parametrize("decoupled", [True, False])
@pytest.mark.parametrize("gs", [None, 0.5])
@pytest.mark.parametrize("t0", [0, 1, 1000])
def test_flat_adam_kernel(decoupled, gs, t0):
    """FlatAdam on device from step count t0 (0: a fresh optimizer), a bf16 group with master and an fp32 group."""
    flat = FlatParams(_mixed_model(DEV))
    opt = ops.FlatAdam(flat, lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.05, decoupled=decoupled)
    if gs:
        opt.set_grad_scale(torch.full((1,), gs, device=DEV))
    gen = torch.Generator().manual_seed(t0)
    opt.step_t.fill_(t0)
    if t0:
        for st in opt.state.values():
            st["m"].copy_(torch.randn(st["m"].numel(), generator=gen) * 0.1)
            st["v"].copy_(torch.rand(st["v"].numel(), generator=gen) * 0.01)
    lr, b1, b2, eps, wd = f32(1e-2), f32(0.9), f32(0.999), f32(1e-8), f32(0.05)
    for it in range(2):
        _fill_grads(flat, gen)
        snap = {dt: ((g.master if g.master is not None else g.param).clone(), opt.state[dt]["m"].clone(),
                     opt.state[dt]["v"].clone()) for dt, g in flat.groups.items()}
        opt.step()
        t = t0 + it + 1
        assert opt.step_t.item() == t
        for dt, g in flat.groups.items():
            master = g.master if g.master is not None else g.param
            w, m, v, tw, tm, tv = ref_adam(*snap[dt], g.grad, t, lr, b1, b2, eps, wd, decoupled, gs or 1.0)
            assert_close(master, w, tw, "master %s" % dt)
            assert_close(opt.state[dt]["m"], m, tm, "m %s" % dt)
            assert_close(opt.state[dt]["v"], v, tv, "v %s" % dt)
            if g.master is not None:
                assert torch.equal(g.param, g.master.to(BF16))
    # a skipped step changes nothing, the step count included; the next applied step counts exactly one
    inf_t = torch.ones(1, dtype=torch.int32, device=DEV)
    opt.set_found_inf(inf_t)
    keep = [opt.step_t] + [t for dt, g in flat.groups.items()
                           for t in (g.param, g.master, opt.state[dt]["m"], opt.state[dt]["v"]) if t is not None]
    before = _bits(*keep)
    _fill_grads(flat, gen)
    opt.step()
    assert _same_bits(before, keep)
    inf_t.zero_()
    opt.step()
    assert opt.step_t.item() == t0 + 3


@gpu
@pytest.mark.parametrize("dtype", [BF16, F32])
@pytest.mark.parametrize("n", [1, 7, 4099, 10 ** 7 + 3])
def test_grad_sqnorm_kernel(dtype, n):
    g = torch.randn(n, device=DEV, generator=torch.Generator(device=DEV).manual_seed(n)).to(dtype)
    out = torch.full((1,), 3.0, device=DEV)          # the kernel adds into out
    ops.native().grad_sqnorm(g, out)
    ref = 3.0 + (g.double() ** 2).sum().item()
    assert abs(out.item() - ref) <= 1e-5 * ref, (out.item(), ref)


@gpu
@pytest.mark.parametrize("case", ["below", "above", "nan", "inf"])
def test_clip_scale_kernel(case):
    """Five partials at stride 2: the odd entries (1e30) must not be read."""
    parts = torch.full((10,), 1e30)
    parts[0::2] = torch.tensor({"below": [0.01, 0.02, 0.03, 0.04, 0.05]}.get(case, [1.0, 2.0, 3.0, 4.0, 5.5]))
    if case in ("nan", "inf"):
        parts[4] = float(case)
    parts = parts.to(DEV)
    scale = torch.full((1,), -1.0, device=DEV)
    norm = torch.full((1,), -1.0, device=DEV)
    ops.native().clip_scale(parts, 5, 2, 1.0, scale, norm)
    norm64 = math.sqrt(parts[0::2].double().sum().item())
    want = ref_clip_scale(norm64, 1.0)
    if case == "below":
        assert scale.item() == 1.0 and abs(norm.item() - norm64) <= 1e-6 * norm64
    elif case == "above":
        assert abs(norm.item() - norm64) <= 1e-6 * norm64
        assert want < 1.0 and abs(scale.item() - want) <= 1e-6 * want
    else:
        assert scale.item() == 1.0 == want
        assert math.isnan(norm.item()) if case == "nan" else norm.item() == math.inf


# ---------------------------------------------------------------------------------------------------- the training step
def _trainer(fused, graph, clip=None, stall=None):
    """``stall["cycles"]``: while non-zero, backward spins that many GPU cycles on the step's stream as soon as the
    logits' gradient is computed, so every gradient of the step is produced late while the host keeps launching."""
    from edl_b200.models import ResNetVd, to_train_dtype
    from edl_b200.trainer import StudentTrainer

    def loss_fn(logits, target):
        if stall is not None and logits.requires_grad:
            logits.register_hook(lambda g: (torch.cuda._sleep(stall["cycles"]) if stall["cycles"] else None, g)[1])
        return ops.soft_cross_entropy(logits, target)

    torch.manual_seed(0)
    m = to_train_dtype(ResNetVd(18, class_dim=16, width_mult=0.25), BF16, DEV).train()
    return StudentTrainer(m, batch_size=8, image_shape=(3, 32, 32), num_classes=16, lr=0.05, use_graph=graph,
                          bucket_cap_mb=0.25, fused_optimizer=fused, clip_norm=clip, loss_fn=loss_fn)


def _batch(gen):
    x = torch.randn(8, 3, 32, 32, generator=gen).to(BF16).contiguous(memory_format=torch.channels_last)
    return x.to(DEV), torch.softmax(torch.randn(8, 16, generator=gen), -1).to(BF16).to(DEV)


@gpu
@pytest.mark.parametrize("fused,graph,clip", [(True, False, None), (False, False, None), (True, True, None),
                                              (False, True, None), (None, False, 0.05)],
                         ids=["bucket-opt-eager", "whole-opt-eager", "bucket-opt-graph", "whole-opt-graph",
                              "clip-eager"])
def test_training_step_matches_sgd_reference(fused, graph, clip):
    """One StudentTrainer step on one GPU updates every element of every group exactly once, from the gradient the
    step leaves behind: a bucket that is skipped, updated twice or updated from another gradient disagrees.

    In the eager steps backward stalls for ~0.1 s on the GPU right after the loss, so the host has launched every
    per-bucket optimizer long before the bucket's gradient exists: an optimizer launch that is not ordered behind the
    gradient's producers reads the previous step's gradient and fails the comparison."""
    stall = {"cycles": 0}
    tr = _trainer(fused, graph, clip, stall)
    dp, opt = tr.dp, tr.opt
    assert dp.bucket_opt == bool(fused and clip is None)
    fused_buckets = sorted(b.numel * dp.flat.groups[b.dtype].grad.element_size() for b in dp.buckets if b.fused_opt)
    if fused:
        assert len(fused_buckets) > 4
    gen = torch.Generator().manual_seed(5)
    tr.step(*_batch(gen), sync=True)            # with graphs: warm-up steps, capture and one replay
    torch.cuda.synchronize()
    snap = {dt: ((g.master if g.master is not None else g.param).clone(), opt.state[dt]["mom"].clone())
            for dt, g in dp.flat.groups.items()}
    stall["cycles"] = 0 if graph else 200_000_000
    tr.step(*_batch(gen), sync=True)
    torch.cuda.synchronize()
    stall["cycles"] = 0
    # one per-bucket optimizer launch per fused bucket, none for the others (with graphs: those of the capture)
    assert sorted(nbytes for algo, nbytes, _ in dp.last_algos if algo == "local_sgd") == fused_buckets
    gs = 1.0
    if clip is not None:
        norm64 = math.sqrt(sum((g.grad.double() ** 2).sum().item() for g in dp.flat.groups.values()))
        norm = dp.grad_norm_t.item()
        assert abs(norm - norm64) <= 1e-5 * norm64, (norm, norm64)
        gs = dp.clip_scale_t.item()
        want = min(1.0, clip / (norm + 1e-6))
        assert want < 1.0 and abs(gs - want) <= 1e-6 * want, (gs, want)
    for dt, g in dp.flat.groups.items():
        master = g.master if g.master is not None else g.param
        w, v, tw, tv = ref_sgd(*snap[dt], g.grad, opt.lr_t.item(), f32(0.9), f32(1e-4), False, gs)
        assert_close(master, w, tw, "master %s" % dt)
        assert_close(opt.state[dt]["mom"], v, tv, "momentum %s" % dt)
        if g.master is not None:
            assert torch.equal(g.param, g.master.to(BF16))
