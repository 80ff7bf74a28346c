"""The float64 oracle of tests/f64_bounds.py without a GPU: its convolution references against naive loops, the checker
accepting correctly rounded outputs (``ops.gemm_bf16``'s CPU path, the CPU BatchNorm statistics) and rejecting each
corruption a broken kernel schedule or epilogue would make."""
import itertools

import numpy as np
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.ops.bn import bn_stats_into


def _bf(*shape, scale=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).bfloat16()


def _naive_conv(x, w, stride, pad, groups):
    """NCHW float64 convolution with an OIHW weight, by loops over the output."""
    x, w = x.double().numpy(), w.double().numpy()
    n, c, h, wd = x.shape
    o, cg, kh, kw = w.shape
    ho, wo = (h + 2 * pad - kh) // stride + 1, (wd + 2 * pad - kw) // stride + 1
    xp = np.zeros((n, c, h + 2 * pad, wd + 2 * pad))
    xp[:, :, pad:pad + h, pad:pad + wd] = x
    y = np.zeros((n, o, ho, wo))
    og = o // groups
    for oc, i, j in itertools.product(range(o), range(ho), range(wo)):
        g = oc // og
        win = xp[:, g * cg:(g + 1) * cg, i * stride:i * stride + kh, j * stride:j * stride + kw]
        y[:, oc, i, j] = (win * w[oc]).sum((1, 2, 3))
    return torch.from_numpy(y)


@pytest.mark.parametrize("stride,groups,h,w", [(1, 1, 5, 7), (2, 1, 6, 5), (2, 2, 7, 8), (1, 4, 4, 3)])
def test_float64_conv_references_match_naive_loops(stride, groups, h, w):
    n, cin, cout = 2, 8, 12
    x = _bf(n, cin, h, w, seed=1)
    wt = _bf(cout, 3, 3, cin // groups, scale=0.3, seed=2)            # KRSC
    w_oihw = wt.permute(0, 3, 1, 2)
    ref, mag = fb.conv_ref(x, wt, stride, 1, groups)
    assert torch.allclose(ref, _naive_conv(x, w_oihw, stride, 1, groups), rtol=1e-12, atol=1e-12)
    assert torch.allclose(mag, _naive_conv(x.abs(), w_oihw.abs(), stride, 1, groups), rtol=1e-12, atol=1e-12)
    # the gradients are the adjoints of that convolution: <dy, conv(x)> = <dgrad(dy), x> = <wgrad(x, dy), w>
    dy = _bf(*ref.shape, seed=3)
    inner = (dy.double() * ref).sum()
    dx, dxm = fb.dgrad_ref(dy, wt, x.shape, stride, 1, groups)
    dw, dwm = fb.wgrad_ref(x, dy, wt.shape, stride, 1, groups)
    assert torch.allclose((dx * x.double()).sum(), inner, rtol=1e-10)
    assert torch.allclose((dw * wt.double()).sum(), inner, rtol=1e-10)
    assert (dxm >= dx.abs() - 1e-12).all() and (dwm >= dw.abs() - 1e-12).all()


def test_bf16_round_is_nearest_even_and_ulp_is_defined_once():
    import test_loss_link_gpu

    assert test_loss_link_gpu.ulp is fb.ulp
    x = torch.randn(100000, dtype=torch.float64) * 10
    # against torch's float32 -> bf16 rounding, on float64 values that are exact in float32 (no double rounding)
    xf = x.float().double()
    assert torch.equal(fb.bf16_round(xf), xf.float().bfloat16().double())
    assert fb.bf16_round(torch.tensor([1.0 + 2 ** -8], dtype=torch.float64)).item() == 1.0          # tie to even
    assert fb.bf16_round(torch.tensor([1.0 + 3 * 2 ** -8], dtype=torch.float64)).item() == 1.0 + 2 ** -6


# ------------------------------------------------------------------------------------------- accepting and rejecting
SHAPES = [(300, 192, 64), (777, 256, 128), (1000, 72, 1568), (133, 320, 25088)]


def _gemm_case(m, n, k, epi, seed=0):
    a = _bf(m, k, seed=seed)
    b = _bf(n, k, scale=0.1, seed=seed + 1)
    kw = {}
    if epi in ("ssr", "all"):
        g = torch.Generator().manual_seed(seed + 2)
        kw = dict(col_scale=torch.rand(n, generator=g) + 0.5, col_shift=torch.randn(n, generator=g), relu=True)
    if epi == "all":
        kw["add"] = _bf(m, n, seed=seed + 3)
    ref, mag = fb.gemm_ref(a, b, add=kw.get("add"), scale=kw.get("col_scale"), shift=kw.get("col_shift"),
                           relu=kw.get("relu", False))
    return a, b, kw, ref, mag


def _kernel_like(a, b, kw, drop=None):
    """fp32 accumulation then one bf16 rounding, in gemm_bf16's epilogue order (its CPU path).  ``drop`` = (row tile,
    column tile, k slice) leaves that k slice out of that 128 x 128 tile."""
    acc = a.float() @ b.float().t()
    if drop is not None:
        ti, tj, ks = drop
        r, c = slice(128 * ti, 128 * ti + 128), slice(128 * tj, 128 * tj + 128)
        acc[r, c] -= a[r, ks].float() @ b[c, ks].float().t()
    if "add" in kw:
        acc = acc + kw["add"].float()
    if "col_scale" in kw:
        acc = acc * kw["col_scale"]
    if "col_shift" in kw:
        acc = acc + kw["col_shift"]
    if kw.get("relu"):
        acc = torch.relu(acc)
    return acc


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("epi", ["none", "ssr", "all"])
def test_checker_accepts_correctly_rounded_outputs(m, n, k, epi):
    a, b, kw, ref, mag = _gemm_case(m, n, k, epi)
    d = ops.gemm_bf16(a, b, **kw)                       # the CPU path: fp32 matmul, epilogue, one bf16 rounding
    c1, c2 = fb.check_bf16(d, ref, mag, k, what="cpu gemm")
    assert c1 <= 1.0 and c2 <= fb.C2_FACTOR
    # the correctly rounded exact result is the yardstick itself
    fb.check_bf16(fb.bf16_round(ref).bfloat16(), ref, mag, k, what="bf16(ref)")


@pytest.mark.parametrize("m", [777, 5000])
def test_checker_accepts_cpu_batchnorm_statistics(m):
    d = _bf(m, 96, seed=4)
    stats = torch.zeros(192)
    bn_stats_into(d.t().reshape(1, 96, m, 1), stats)
    ref, mag = fb.stats_ref(d)
    fb.check_sums(stats, ref, mag, m, what="cpu stats")
    st2 = torch.zeros(192)
    ops.gemm_bf16(_bf(m, 64, seed=5), _bf(96, 64, seed=6), col_stats=st2)
    d2 = ops.gemm_bf16(_bf(m, 64, seed=5), _bf(96, 64, seed=6))
    fb.check_sums(st2, *fb.stats_ref(d2), m, what="cpu gemm stats")


def _rejects(fn, *args, match, **kw):
    with pytest.raises(AssertionError, match=match):
        fn(*args, **kw)


def test_rejects_zeroed_m_tail_rows():
    m, n, k = 128 * 148 * 3 + 5, 128, 64
    a, b, kw, ref, mag = _gemm_case(m, n, k, "none")
    d = ops.gemm_bf16(a, b)
    d[-5:] = 0
    _rejects(fb.check_bf16, d, ref, mag, k, what="tail", match=r"criterion 1: 6[0-9][0-9] of .*\(444, 0\)")


def test_rejects_one_channel_scale_off_by_0p3_percent():
    a, b, kw, ref, mag = _gemm_case(5000, 256, 192, "ssr")
    kw["col_scale"] = kw["col_scale"].clone()
    kw["col_scale"][37] *= 1.003
    d = ops.gemm_bf16(a, b, **kw)
    _rejects(fb.check_bf16, d, ref, mag, 192, what="scale", match=r"criterion 2: 1 of 256 columns .* worst 37:")


def test_rejects_one_channel_shift_off_by_0p02():
    a, b, kw, ref, mag = _gemm_case(5000, 256, 192, "ssr")
    kw["col_shift"] = kw["col_shift"].clone()
    kw["col_shift"][200] += 0.02
    d = ops.gemm_bf16(a, b, **kw)
    _rejects(fb.check_bf16, d, ref, mag, 192, what="shift", match=r"columns .* worst 200:")


@pytest.mark.parametrize("m,n,k", SHAPES)
def test_rejects_rounding_toward_zero(m, n, k):
    a, b, kw, ref, mag = _gemm_case(m, n, k, "none")
    acc = _kernel_like(a, b, kw)
    rtz = (acc.view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()          # truncate the low 16 bits
    _rejects(fb.check_bf16, rtz, ref, mag, k, what="rtz", match="criterion 2")


@pytest.mark.parametrize("m,n,k,what", [s + (w,) for s in SHAPES for w in ("term", "block")
                                          if w == "term" or s[2] >= 128])      # a block of a 64-deep K would be all of K
def test_rejects_one_k_term_or_block_missing_from_one_tile(m, n, k, what):
    a, b, kw, ref, mag = _gemm_case(m, n, k, "ssr")
    kb = 64 * max(1, k // 128)                          # a 64-wide block strictly inside K, never its first
    ks = slice(k // 2, k // 2 + 1) if what == "term" else slice(kb, kb + 64)
    assert ks.stop - ks.start < k
    tj = (n - 1) // 128                                 # the last column tile (partial for n = 72, 192, 320)
    d = _kernel_like(a, b, kw, drop=(1, tj, ks)).bfloat16()
    _rejects(fb.check_bf16, d, ref, mag, k, what=what, match=r"\(1, %d\)" % tj)


def test_rejects_one_row_missing_from_col_stats():
    m = 777
    a, b, kw, ref, mag = _gemm_case(m, 192, 64, "none")
    d = ops.gemm_bf16(a, b)
    stats = torch.zeros(2 * 192)
    ops.gemm_bf16(a[:-1], b, col_stats=stats)                            # the last row is missing
    _rejects(fb.check_sums, stats, *fb.stats_ref(d), m, what="stats", match="sums out of bounds")


def test_rejects_a_nan_output():
    a, b, kw, ref, mag = _gemm_case(300, 192, 64, "none")
    d = ops.gemm_bf16(a, b)
    d[299, 191] = float("nan")
    _rejects(fb.check_bf16, d, ref, mag, 64, what="nan", match=r"first at \(299, 191\): out nan")


@pytest.mark.parametrize("shape,pad_rows,pad_cols", [((37, 72), 3, 8), ((1000,), 8, 0), ((2, 64, 3, 5), 2, 0)])
def test_guarded_window_detects_a_stray_store(shape, pad_rows, pad_cols):
    g = fb.guarded(shape, pad_rows, pad_cols, fill=-7.0, device="cpu")
    assert tuple(g.t.shape) == shape
    g.t.copy_(torch.randn(shape).bfloat16())          # writes inside the window are fine
    g.assert_untouched()
    if len(shape) == 2:
        assert g.t.stride(0) == shape[1] + pad_cols
    g.buf.view(-1)[-1] = 1.0                           # one sentinel overwritten
    _rejects(g.assert_untouched, what="guard", match="1 sentinel elements overwritten")
    nan = fb.guarded(shape, pad_rows, pad_cols, device="cpu", values=torch.ones(shape))
    nan.assert_untouched()                             # NaN sentinels compare bit for bit
    assert bool(nan.t.eq(1).all()) and bool(nan.buf.isnan().sum() == nan.buf.numel() - nan.t.numel())


def test_bn_backward_reference_and_ambiguous_mask():
    m, n = 300, 64
    g = torch.Generator().manual_seed(9)
    d, x = _bf(m, n, seed=10), _bf(m, n, seed=11)
    mean, rstd = torch.randn(n, generator=g) * 0.1, torch.rand(n, generator=g) + 0.5
    gamma, beta = torch.rand(n, generator=g) + 0.5, torch.randn(n, generator=g) * 0.2
    keep, amb = fb.bn_mask_fp32(x, mean, rstd, gamma, beta)
    # the fp32 fmaf reproduced on the CPU: fp32(x * sc + sh) in float64, rounded once
    sc = gamma * rstd
    sh = beta - mean * sc
    pre = (x.double() * sc.double() + sh.double()).float()
    assert bool(((pre > 0) == keep)[~amb].all())
    ref, mag, extra = fb.bn_dsums_ref(d, x, mean, rstd, gamma, beta, True)
    dm = d.double() * keep
    xh = (x.double() - mean.double()) * rstd.double()
    assert torch.allclose(ref, torch.cat([dm.sum(0), (dm * xh).sum(0)]))
    assert (mag >= ref.abs() - 1e-9).all() and (extra >= 0).all()
    # a sum that misses one row fails
    bad = ref.clone()
    bad[3] += float(dm[5, 3]) if dm[5, 3] != 0 else 1.0
    _rejects(fb.check_sums, bad, ref, mag, m, what="dsums", extra=extra, match=r"\[3\]")


def test_pair_terms_allow_their_own_rounding_only():
    """A sum of two bf16-rounded partials may be off by their half ulps, not by more: 2 % scaling or 1 % noise fails."""
    g = torch.Generator().manual_seed(12)
    t0, t1 = torch.randn(300, 200, generator=g, dtype=torch.float64) * 5, torch.randn(300, 200, generator=g,
                                                                                      dtype=torch.float64) * 5
    m0, m1 = t0.abs() * 30, t1.abs() * 30                 # weight-gradient-like magnitudes, far above the values
    ref, mag = t0 + t1, m0 + m1
    out = fb.bf16_round(fb.bf16_round(t0) + fb.bf16_round(t1)).bfloat16()
    fb.check_bf16(out, ref, mag, 64, terms=[(t0, m0), (t1, m1)], what="pair")
    _rejects(fb.check_bf16, (ref * 1.02).bfloat16(), ref, mag, 64, terms=[(t0, m0), (t1, m1)], what="x1.02",
             match="criterion")
    noisy = (ref * (1 + 0.01 * torch.randn(ref.shape, generator=g, dtype=torch.float64))).bfloat16()
    _rejects(fb.check_bf16, noisy, ref, mag, 64, terms=[(t0, m0), (t1, m1)], what="noise", match="criterion")
