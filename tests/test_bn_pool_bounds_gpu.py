"""Float64 element-wise bounds for the BatchNorm kernels (csrc/bn.cu register kernels, bn_stream.cu streaming kernels,
bn_fused.cu SM-resident kernels) and the pooling kernels (csrc/pool.cu), through their native entry points.

Every case first asserts which path runs (``bn_set_stream_kernels(False)`` for the register kernels,
``bn_stream_supported`` for the streaming ones, ``bn_fused_fits`` for the SM-resident ones), then checks each stage
against a float64 reference built from the kernel's own fp32 intermediates (tests/f64_bounds.py: the reduction sums
against ``bn_reduce_tau``, saved and running statistics against their formulas, ``y``/``dx`` criterion 1) and end to end
against the exact statistics of the bf16 input (criterion 2, and the propagated statistics bound).  Operands sit in
NaN-filled windows and outputs in sentinel-filled ones: a read past ``M C`` poisons the result, a stray store is found.

Inputs have per-channel |mean| / std of 0, 4 and 16, a constant channel (var = 0, rstd = eps^-1/2), a channel with
gamma = 0 and one with gamma < 0.  NaN propagation through max-pool is out of scope: the kernel's ``>`` drops NaN while
torch propagates it."""
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS, MOM = 1e-5, 0.1
PAD = 4                      # sentinel rows around every [M, C] window (whole rows keep 16-byte alignment)
SENT = -7.0                  # finite sentinel around outputs


def nat():
    return ops.native()


@pytest.fixture(autouse=True)
def _default_paths():
    yield
    nat().bn_set_stream_kernels(True)
    ops.set_fused_bn(False)


def _vec(c, values=None, fill=SENT):
    return fb.guarded((c,), 8, fill=fill, dtype=torch.float32, values=values)


def _mat(m, c, values=None, fill=float("nan"), dtype=torch.bfloat16):
    return fb.guarded((m, c), PAD, fill=fill, dtype=dtype, values=values)


def _inputs(m, c, seed, res):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ch = torch.arange(c, device=DEV)
    offs = torch.tensor([0.0, 4.0, -16.0, 16.0, -4.0, 0.0], device=DEV)[ch % 6]
    std = torch.rand(c, generator=g, device=DEV) * 1.5 + 0.5
    x = (torch.randn(m, c, generator=g, device=DEV) + offs) * std
    x[:, 1] = 1.0                                              # constant channel
    gamma = torch.rand(c, generator=g, device=DEV) + 0.5
    gamma[2] = 0.0
    gamma[3] = -gamma[3]
    beta = torch.randn(c, generator=g, device=DEV) * 0.2
    r = torch.randn(m, c, generator=g, device=DEV).bfloat16() if res else None
    dy = torch.randn(m, c, generator=g, device=DEV).bfloat16()
    return x.bfloat16(), r, gamma, beta, dy


def _set_path(path, m, c, nt):
    """Select and assert the kernels that will run for [m, c] with ``nt`` staged operands."""
    n = nat()
    n.bn_set_stream_kernels(path != "regs")
    if path == "fused":
        assert n.bn_fused_fits(m, c, nt), (m, c, nt)
    elif path == "stream":
        assert n.bn_stream_supported(m, c), (m, c)
    else:
        assert path == "regs"


def _e2e_cols(x):
    """Channels judged end to end: all but the constant ones, whose rstd is set by eps and the rounding of a zero
    variance (the propagated statistics bound judges those)."""
    return fb.bn_exact_stats(x)[1] > 0


def _forward(path, x, res, gamma, beta, relu, bits=False, what=""):
    m, c = x.shape
    n = nat()
    _set_path(path, m, c, 2 if res is not None else 1)
    X, R = _mat(m, c, x), (_mat(m, c, res) if res is not None else None)
    G, B = _vec(c, gamma, fill=float("nan")), _vec(c, beta, fill=float("nan"))
    Y = _mat(m, c, fill=SENT)
    sums, mean, rstd = _vec(2 * c, torch.zeros(2 * c, device=DEV)), _vec(c), _vec(c)
    rm0, rv0 = torch.randn(c, device=DEV) * 0.1, torch.rand(c, device=DEV) + 0.5
    RM, RV = _vec(c, rm0), _vec(c, rv0)
    Mb = None
    if bits:
        assert path == "stream" and res is not None and relu and n.bn_relu_mask_supported(m, c)
        Mb = _mat(m, c // 8, fill=0xA5, dtype=torch.uint8)
    rt = R.t if R is not None else None
    if path == "fused":
        n.bn_fwd_fused(X.t, rt, Y.t, sums.t, G.t, B.t, RM.t, RV.t, mean.t, rstd.t, EPS, MOM, relu,
                       torch.zeros(1, device=DEV, dtype=torch.int32))
    else:
        n.bn_stats(X.t, sums.t)
        n.bn_apply(X.t, rt, Y.t, sums.t, G.t, B.t, RM.t, RV.t, mean.t, rstd.t, EPS, MOM, relu,
                   Mb.t if Mb is not None else None)
    for o, name in ((Y, "y"), (sums, "sums"), (mean, "mean"), (rstd, "rstd"), (RM, "running mean"),
                    (RV, "running var")) + (((Mb, "mask bits"),) if Mb is not None else ()):
        o.assert_untouched(what + " " + name)
    tau_s = fb.bn_reduce_tau(path, m, c)
    fb.check_sums(sums.t, *fb.stats_ref(x), m, what=what + " sums", tau_s=tau_s)
    fb.check_bn_saved_stats(sums.t, mean.t, rstd.t, m, EPS, what=what, running=(rm0, rv0, RM.t, RV.t, MOM))
    fb.check_bn_stats_e2e(x, mean.t, rstd.t, EPS, tau_s, what=what)
    y = Y.t
    fb.check_bf16(y, *fb.bn_y_ref(x, mean.t, rstd.t, gamma, beta, res, relu), tau=fb.BN_Y_TAU, criteria=(1,),
                  what=what + " y")
    if m >= fb.E2E_MIN_ROWS:
        cols = _e2e_cols(x)
        ey = fb.bn_exact(x, gamma, beta, EPS, res, relu)["y"]
        fb.check_bf16(y, *ey, tau=fb.BN_Y_TAU, criteria=(2,), columns=cols, what=what + " y e2e")
    if Mb is not None:
        fb.check_exact(Mb.t, fb.mask_bits(y > 0), what=what + " mask bits vs (stored y > 0)")
    return y.clone(), mean.t.clone(), rstd.t.clone(), (Mb.t.clone() if Mb is not None else None)


def _backward(path, x, res, gamma, beta, relu, y, mean, rstd, dy, ysrc, acc, bits=None, what=""):
    """``ysrc``: where the ReLU mask comes from: "x" (recomputed), "y" (the stored output), "bits" (the forward's mask
    bits), "premasked" (``dy`` stored already masked, the backward runs without ReLU and ``dres`` aliases ``dy``)."""
    m, c = x.shape
    n = nat()
    keep = (y > 0) if relu else None
    d = dy
    if ysrc == "premasked":
        assert relu and res is not None
        d, relu_k, keep = torch.where(keep, dy, torch.zeros_like(dy)), False, None
    else:
        relu_k = relu
    yk = {"x": None, "y": y, "bits": bits, "premasked": None}[ysrc] if relu_k else None
    nt = 2 + (1 if (yk is not None and path == "fused") else 0)
    _set_path(path, m, c, nt)
    D, X = _mat(m, c, d), _mat(m, c, x)
    G, B = _vec(c, gamma, fill=float("nan")), _vec(c, beta, fill=float("nan"))
    Mn, Rs = _vec(c, mean, fill=float("nan")), _vec(c, rstd, fill=float("nan"))
    YK = None
    if yk is not None:
        YK = _mat(m, c // 8, yk, fill=0xA5, dtype=torch.uint8) if yk.dtype == torch.uint8 else _mat(m, c, yk)
    DX = _mat(m, c, fill=SENT)
    has_dres = res is not None and ysrc != "premasked"
    DR = _mat(m, c, fill=SENT) if has_dres else None
    dsums = _vec(2 * c, torch.zeros(2 * c, device=DEV))
    g0, b0 = (torch.randn(c, device=DEV), torch.randn(c, device=DEV)) if acc else (torch.zeros(c, device=DEV),) * 2
    DG, DB = _vec(c, g0), _vec(c, b0)
    ykt, drt = (YK.t if YK is not None else None), (DR.t if DR is not None else None)
    if path == "fused":
        n.bn_bwd_fused(D.t, X.t, ykt, G.t, B.t, Mn.t, Rs.t, dsums.t, DX.t, drt, DG.t, DB.t, relu_k, acc,
                       torch.zeros(1, device=DEV, dtype=torch.int32))
    else:
        n.bn_bwd_reduce(D.t, X.t, ykt, G.t, B.t, Mn.t, Rs.t, dsums.t, relu_k)
        n.bn_bwd_apply(D.t, X.t, ykt, G.t, B.t, Mn.t, Rs.t, dsums.t, DX.t, drt, DG.t, DB.t, relu_k, acc)
    for o, name in ((DX, "dx"), (dsums, "dsums"), (DG, "dgamma"), (DB, "dbeta")) + (((DR, "dres"),) if DR else ()):
        o.assert_untouched(what + " " + name)
    ds = dsums.t
    ref, mag, extra = fb.bn_dsums_ref(d, x, mean, rstd, gamma, beta, relu_k, y=y if relu_k else None)
    fb.check_sums(ds, ref, mag, m, what=what + " dsums", extra=extra, tau_s=fb.bn_reduce_tau(path, m, c))
    want_g, want_b = (g0 + ds[c:], b0 + ds[:c]) if acc else (ds[c:], ds[:c])
    fb.check_exact(DG.t, want_g, what=what + " dgamma")
    fb.check_exact(DB.t, want_b, what=what + " dbeta")
    dx = DX.t
    fb.check_bf16(dx, *fb.bn_dx_ref(d, x, mean, rstd, gamma, ds, m, keep), tau=fb.BN_DX_TAU, criteria=(1,),
                  what=what + " dx")
    if m >= fb.E2E_MIN_ROWS:
        cols = _e2e_cols(x)
        ex = fb.bn_exact(x, gamma, beta, EPS, res, relu, y=y, dy=dy)
        fb.check_bf16(dx, *ex["dx"], tau=fb.BN_DX_TAU, criteria=(2,), columns=cols, what=what + " dx e2e")
    if has_dres:
        fb.check_exact(DR.t, torch.where(keep, dy, torch.zeros_like(dy)) if relu else dy, what=what + " dres")
    return dx.clone()


def _case(m, c, relu, res, fwd, bwd, ysrc, acc, seed=0):
    what = "[%d, %d] relu %d res %d %s/%s mask %s acc %d" % (m, c, relu, res, fwd, bwd, ysrc, acc)
    x, r, gamma, beta, dy = _inputs(m, c, seed, res)
    y, mean, rstd, bits = _forward(fwd, x, r, gamma, beta, relu, bits=ysrc in ("bits", "premasked"), what=what)
    _backward(bwd, x, r, gamma, beta, relu, y, mean, rstd, dy, ysrc, acc, bits=bits, what=what)


# ResNet50_vd at batch 32 (tools/bn_shapes.py), one or two modes per shape
RESNET = [
    (401408, 32, True, False, "stream", "stream", "x", False),
    (401408, 32, True, False, "regs", "regs", "x", True),
    (100352, 64, True, False, "fused", "fused", "x", False),
    (100352, 64, False, False, "stream", "stream", "x", True),
    (100352, 256, True, True, "stream", "stream", "bits", False),
    (100352, 256, True, True, "stream", "stream", "premasked", True),
    (25088, 512, True, True, "stream", "stream", "y", True),
    (25088, 512, True, True, "regs", "regs", "y", False),
    (6272, 1024, True, True, "fused", "stream", "y", False),       # fits the fused forward, not the 3-operand backward
    (6272, 1024, True, True, "stream", "stream", "bits", True),
    (1568, 2048, True, True, "fused", "fused", "y", True),
    (1568, 2048, True, True, "stream", "stream", "premasked", False),
    (1568, 512, True, False, "fused", "fused", "x", True),
    (1568, 512, False, False, "regs", "regs", "x", False),
]

# chunk and switch edges, register grids with partial x-blocks and row tails
EDGES = [
    (8192, 8, True, False, "stream", "stream", "x", False),       # C = 8: one channel group; M C = 65536
    (8191, 8, True, True, "regs", "regs", "y", True),              # M C = 65528: the largest register tensor
    (2048, 32, False, True, "stream", "stream", "x", False),       # M C = 65536: the smallest streaming tensor
    (64, 4096, True, True, "stream", "stream", "bits", False),     # C = 4096: all 512 consumers hold one group
    (64, 4096, True, False, "fused", "fused", "x", True),
    (1000, 256, True, True, "stream", "stream", "bits", True),     # the last 16 KB chunk is partial
    (1000, 256, True, True, "fused", "fused", "y", False),
    (17024, 64, True, False, "stream", "stream", "x", True),       # 133 chunks: one more than 132 CTAs
    (17024, 64, True, True, "fused", "stream", "y", False),
    (3000, 24, True, False, "regs", "regs", "x", False),
    (37, 72, True, True, "regs", "regs", "y", True),
    (2, 200, True, False, "regs", "regs", "x", False),
    (3, 1000, False, True, "regs", "regs", "x", True),
    (777, 1000, True, True, "regs", "regs", "y", False),
]


@pytest.mark.parametrize("m,c,relu,res,fwd,bwd,ysrc,acc", RESNET + EDGES)
def test_bn_bounds(m, c, relu, res, fwd, bwd, ysrc, acc):
    _case(m, c, relu, res, fwd, bwd, ysrc, acc)


def _largest_fused_m(c, nt):
    lo, hi = 1, 1 << 22
    assert nat().bn_fused_fits(lo, c, nt) and not nat().bn_fused_fits(hi, c, nt)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if nat().bn_fused_fits(mid, c, nt) else (lo, mid)
    return lo


@pytest.mark.parametrize("nt", [1, 2, 3])
def test_bn_fused_at_resident_capacity(nt):
    """The largest M the SM-resident kernels accept for 1, 2 and 3 staged operands (every CTA's staging full)."""
    c = 256
    m = _largest_fused_m(c, nt)
    assert not nat().bn_fused_fits(m + 1, c, nt)
    if nt == 1:
        _case(m, c, True, False, "fused", "stream", "x", False)
    elif nt == 2:
        _case(m, c, False, True, "fused", "fused", "x", True)     # 2-operand forward, 2-operand backward
    else:
        _case(m, c, True, True, "stream", "fused", "y", False)


@pytest.mark.parametrize("fwd", ["regs", "stream", "fused"])
def test_recomputed_relu_mask_equals_stored_output(fwd):
    """Without a residual the backward recomputes the ReLU mask as ``fmaf(x, g r, b - m g r) > 0``, in a different
    kernel from the one that stored y, and so does the dgrad epilogue that carries the BatchNorm's reduction.  If one of
    them formed the shift ``b - m g r`` with an fma and another as a product and a subtraction, the masks would differ
    only where the pre-activation lies within an ulp of the shift, which random data practically never hits.  So the
    data is built to sit there: integer x (exact fp32 sums, so every path saves the same statistics) and, from the
    saved statistics, the gamma and beta of ``f64_bounds.bn_mask_edge``, which make the shift 0 under one contraction and
    a positive residual under the other.  Every x == 0 element is then on the edge.  For the y stored by each forward,
    each backward must agree with (stored y > 0): the register and streaming applies bit for bit (dx from the
    recomputed mask against dx from y, identical dsums), the reductions, the fused backward and the dgrad epilogue
    within their rounding bounds with no allowance for ambiguous elements."""
    m, c = 6272, 256
    n = nat()
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randint(-3, 4, (m, c), generator=g, device=DEV).bfloat16()
    dy = torch.randn(m, c, generator=g, device=DEV).bfloat16()
    gamma0 = torch.rand(c, generator=g, device=DEV) + 0.5
    what = "mask edge, %s forward" % fwd
    _, mean, rstd, _ = _forward(fwd, x, None, gamma0, torch.zeros(c, device=DEV), True, what=what)
    gamma, beta, resid = fb.bn_mask_edge(mean, rstd, gamma0)
    edge = (x == 0) & (resid > 0)
    assert int(edge.sum()) > m * c // 10, "the construction puts too few elements on the edge: %d" % int(edge.sum())
    y, mean2, rstd2, _ = _forward(fwd, x, None, gamma, beta, True, what=what)
    fb.check_exact(mean2, mean, what=what + ": saved mean independent of gamma and beta")
    fb.check_exact(rstd2, rstd, what=what + ": saved rstd independent of gamma and beta")
    keep = y > 0
    ref, mag, _ = fb.bn_dsums_ref(dy, x, mean, rstd, gamma, beta, True, y=y)
    dsums = torch.zeros(2 * c, device=DEV)
    _set_path("stream", m, c, 2)
    n.bn_bwd_reduce(dy, x, y, gamma, beta, mean, rstd, dsums, True)
    for bwd in ("regs", "stream"):
        _set_path(bwd, m, c, 2)
        ds = torch.zeros(2 * c, device=DEV)
        n.bn_bwd_reduce(dy, x, None, gamma, beta, mean, rstd, ds, True)
        fb.check_sums(ds, ref, mag, m, tau_s=fb.bn_reduce_tau(bwd, m, c), what="%s, %s reduction" % (what, bwd))
        outs = []
        for ysrc in (None, y):
            dx = torch.empty_like(x)
            n.bn_bwd_apply(dy, x, ysrc, gamma, beta, mean, rstd, dsums, dx, None, None, None, True, False)
            outs.append(dx)
        diff = outs[0].view(torch.int16) != outs[1].view(torch.int16)
        assert not diff.any(), "%s, %s apply: %d elements differ, first at %s" % (
            what, bwd, int(diff.sum()), diff.nonzero()[0].tolist())
    _set_path("fused", m, c, 2)
    ds, dx = torch.zeros(2 * c, device=DEV), torch.empty_like(x)
    n.bn_bwd_fused(dy, x, None, gamma, beta, mean, rstd, ds, dx, None, None, None, True, False,
                   torch.zeros(1, device=DEV, dtype=torch.int32))
    fb.check_sums(ds, ref, mag, m, tau_s=fb.bn_reduce_tau("fused", m, c), what=what + ", fused reduction")
    fb.check_bf16(dx, *fb.bn_dx_ref(dy, x, mean, rstd, gamma, ds, m, keep), tau=fb.BN_DX_TAU, criteria=(1,),
                  what=what + ", fused dx")
    # the 1x1 dgrad whose epilogue carries this BatchNorm's reduction, mask recomputed from x
    from edl_b200.ops.bn import BNBackwardHook

    h = BNBackwardHook()
    h.x, h.y, h.mask, h.relu = x, None, None, True
    h.mean, h.rstd, h.gamma, h.beta, h.dsums = mean, rstd, gamma, beta, torch.zeros(2 * c, device=DEV)
    a = torch.randn(m, 64, generator=g, device=DEV).bfloat16()
    w = (torch.randn(64, c, generator=g, device=DEV) * 0.1).bfloat16()
    d = ops.gemm_bf16(a, w, b_mn_major=True, bn=h)
    assert h.done, "the dgrad epilogue did not carry the reduction"
    dref, dmag, _ = fb.bn_dsums_ref(d, x, mean, rstd, gamma, beta, True, y=y)
    fb.check_sums(h.dsums, dref, dmag, m, what=what + ", dgrad epilogue reduction")


@pytest.mark.parametrize("path", ["regs", "stream", "fused"])
def test_batch_norm_act_autograd(path):
    """One step of ``ops.batch_norm_act`` per path against float64 F.batch_norm autograd on the same bf16 tensors
    (ReLU mask of the stored output).  The register and streaming paths take the statistics delivered by
    ``ops.conv1x1``; the fused forward computes its own (it runs only without delivered statistics)."""
    torch.manual_seed(5)
    n_, cin, c, h, w = 8, 64, 256, 28, 28
    m = n_ * h * w
    ops.set_fused_bn(path == "fused")
    _set_path(path, m, c, 3 if path == "fused" else 1)
    if path == "fused":
        assert nat().bn_fused_fits(m, c, 2)
    a = torch.randn(n_, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(c, cin, device=DEV) * 0.2).bfloat16()
    stats = torch.zeros(2 * c, device=DEV)
    xc = ops.conv1x1(a, wt, stats).detach().requires_grad_()
    fb.check_sums(stats, *fb.stats_ref(xc.detach()), m, what="conv1x1 stats")
    r = torch.randn(n_, c, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_()
    gamma = (torch.rand(c, device=DEV) + 0.5).requires_grad_()
    beta = (torch.randn(c, device=DEV) * 0.2).requires_grad_()
    rm, rv = torch.zeros(c, device=DEV), torch.ones(c, device=DEV)
    y = ops.batch_norm_act(xc, gamma, beta, rm, rv, residual=r, relu=True,
                           sums=None if path == "fused" else stats.clone())
    dy = torch.randn(n_, c, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    x2 = fb.rows(xc.detach())
    ex = fb.bn_exact(x2, gamma.detach(), beta.detach(), EPS, fb.rows(r.detach()), True, y=fb.rows(y.detach()),
                     dy=fb.rows(dy))
    cols = _e2e_cols(x2)
    for name, got in (("y", y.detach()), ("dx", xc.grad), ("dres", r.grad)):
        ref, mag = ex[name]
        fb.check_bf16(got, ref, mag, criteria=(2,), columns=cols, what="%s batch_norm_act %s" % (path, name))
    # the exact statistics differ from the kernel's by their rounding (about 1e-6 relative here): 2^-12 of the sum of
    # |terms| admits that and still fails a gradient left unmasked or a wrong scale
    for name, got in (("dgamma", gamma.grad), ("dbeta", beta.grad)):
        fb.check_sums(got, *ex[name], m, what="%s batch_norm_act %s" % (path, name), tau_s=2 ** -12)


@pytest.mark.parametrize("m,c,relu,res", [(1000, 256, True, True), (37, 72, False, False), (50176, 64, True, False)])
def test_scale_shift_act(m, c, relu, res):
    x, r, gamma, beta, _ = _inputs(m, c, 6, res)
    scale, shift = gamma * 0.7, beta - 0.3
    X, Y = _mat(m, c, x), _mat(m, c, fill=SENT)
    nat().scale_shift_act(X.t, _mat(m, c, r).t if res else None, Y.t, scale, shift, relu)
    Y.assert_untouched("scale_shift_act y")
    fb.check_bf16(Y.t, *fb.scale_shift_ref(x, scale, shift, r, relu), tau=2 * fb.EPS32, what="scale_shift_act")


# ------------------------------------------------------------------------------------------------------------ pooling
def _img(shape, values=None, fill=float("nan")):
    return fb.guarded(shape, 3, fill=fill, values=values)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


@pytest.mark.parametrize("shape,kind", [((2, 64, 112, 112), "relu"), ((3, 32, 17, 19), "negative"),
                                        ((2, 64, 9, 8), "integers"), ((4, 256, 7, 7), "relu"),
                                        ((2, 72, 15, 15), "integers")])
def test_maxpool(shape, kind):
    """Ties are the common case (a ReLU output is zero on half of each window): the first maximum in (kh, kw) order
    gets the gradient.  All-negative windows at the border: padding acts as -inf."""
    n, c, h, w = shape
    g = torch.Generator(device=DEV).manual_seed(7)
    v = torch.randn(shape, generator=g, device=DEV)
    v = {"relu": v.relu(), "negative": -v.abs() - 0.01,
         "integers": torch.randint(-2, 3, shape, generator=g, device=DEV).float()}[kind]
    x = v.bfloat16()
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    X, Y = _img(shape, x), _img((n, c, ho, wo), fill=SENT)
    I = fb.guarded((n * ho * wo, c), 2, fill=0xEE, dtype=torch.uint8)
    nat().maxpool3x3s2_fwd(_nhwc(X.t), _nhwc(Y.t), I.t.view(n, ho, wo, c))
    Y.assert_untouched("maxpool y")
    I.assert_untouched("maxpool idx")
    idx = fb.check_maxpool(Y.t, I.t.view(n, ho, wo, c).permute(0, 3, 1, 2), x, what="maxpool %s" % kind)
    dy = torch.randn(n, c, ho, wo, generator=g, device=DEV).bfloat16()
    DY, DX = _img(dy.shape, dy.contiguous(memory_format=torch.channels_last)), _img(shape, fill=SENT)
    nat().maxpool3x3s2_bwd(_nhwc(DY.t), I.t.view(n, ho, wo, c), _nhwc(DX.t))
    DX.assert_untouched("maxpool dx")
    fb.check_bf16(DX.t, *fb.maxpool_bwd_ref(dy, idx, shape), tau=3 * fb.EPS32, what="maxpool dx %s" % kind)


@pytest.mark.parametrize("shape", [(2, 64, 56, 56), (2, 2048, 7, 7), (3, 72, 9, 11), (2, 200, 14, 13)])
def test_avgpool_gap(shape):
    n, c, h, w = shape
    g = torch.Generator(device=DEV).manual_seed(8)
    x = (torch.randn(shape, generator=g, device=DEV) + 0.5).bfloat16()
    ho, wo = (h + 1) // 2, (w + 1) // 2
    X, Y = _img(shape, x), _img((n, c, ho, wo), fill=SENT)
    nat().avgpool2x2_fwd(_nhwc(X.t), _nhwc(Y.t))
    Y.assert_untouched("avgpool y")
    fb.check_bf16(Y.t, *fb.avgpool_ref(x), tau=3 * fb.EPS32, what="avgpool y")
    dy = torch.randn(n, c, ho, wo, generator=g, device=DEV).bfloat16()
    DY, DX = _img(dy.shape, dy), _img(shape, fill=SENT)
    nat().avgpool2x2_bwd(_nhwc(DY.t), _nhwc(DX.t))
    DX.assert_untouched("avgpool dx")
    fb.check_bf16(DX.t, *fb.avgpool_bwd_ref(dy, shape), tau=fb.EPS32, what="avgpool dx")
    G = fb.guarded((n, c), 2, fill=SENT)
    nat().gap_fwd(_nhwc(X.t), G.t)
    G.assert_untouched("gap y")
    fb.check_bf16(G.t, *fb.gap_ref(x), tau=fb.gap_tau(h * w), what="gap y")
    dg = torch.randn(n, c, generator=g, device=DEV).bfloat16()
    DG, DX2 = fb.guarded((n, c), 2, values=dg), _img(shape, fill=SENT)
    nat().gap_bwd(DG.t, _nhwc(DX2.t))
    DX2.assert_untouched("gap dx")
    fb.check_bf16(DX2.t, *fb.gap_bwd_ref(dg, shape), tau=2 * fb.EPS32, what="gap dx")


@pytest.mark.parametrize("shape", [(2, 64, 7, 9), (1, 8, 1, 1), (3, 200, 14, 14)])
def test_dilate2(shape):
    n, c, h, w = shape
    x = torch.randn(shape, device=DEV).bfloat16()
    X, O = _img(shape, x), _img((n, c, 2 * h, 2 * w), fill=SENT)
    nat().dilate2(X.t, O.t)
    O.assert_untouched("dilate2")
    fb.check_exact(O.t, fb.dilate2_ref(x), what="dilate2")
