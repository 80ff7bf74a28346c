"""Persistent wgmma GEMM / conv kernel (csrc/gemm_persist.cu) against the one-tile-per-CTA kernels and
the fp32 reference: many tiles per CTA (ring wrap-around across tiles)."""
import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _restore():
    yield
    ops.native().set_persistent_gemm(True)


@pytest.mark.parametrize("m,n,k", [(100352, 64, 64), (100352, 256, 64), (25088, 512, 128), (6272, 1024, 256),
                                   (1568, 2048, 512), (40000, 192, 72), (300, 128, 64), (128 * 148 * 3 + 5, 128, 64)])
@pytest.mark.parametrize("b_mn", [False, True])
def test_persistent_gemm_matches_reference_and_stats(m, n, k, b_mn):
    torch.manual_seed(0)
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = (torch.randn(k, n, device=DEV) if b_mn else torch.randn(n, k, device=DEV)).bfloat16()
    ref = fb.gemm_ref(a, b, b_mn_major=b_mn)
    outs = []
    for persistent in (True, False):
        ops.native().set_persistent_gemm(persistent)
        stats = torch.zeros(2 * n, device=DEV)
        d = ops.gemm_bf16(a, b, b_mn_major=b_mn, col_stats=None if b_mn else stats)
        fb.check_bf16(d, *ref, k, what="gemm persistent=%s" % persistent)
        if not b_mn:
            fb.check_sums(stats, *fb.stats_ref(d), m, what="gemm stats persistent=%s" % persistent)
        outs.append(d)
    assert torch.equal(outs[0], outs[1])          # same MMA order => bit-identical results


@pytest.mark.parametrize("m,n,k,res", [(25088, 512, 512, False), (6272, 2048, 1024, True), (100352, 512, 256, True),
                                       (1568, 4096, 2048, False)])
def test_wide_tile_gemm_matches_the_128_wide_tiles(m, n, k, res):
    """128 x 256 tiles for the teacher's large-N 1x1 convolutions: same
    results as the 128 x 128 tiles, with the folded-BN epilogue and the TMA-fetched residual addend."""
    torch.manual_seed(2)
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = (torch.randn(n, k, device=DEV) * 0.05).bfloat16()
    sh = torch.randn(n, device=DEV)
    add = torch.randn(m, n, device=DEV).bfloat16() if res else None
    ref = fb.gemm_ref(a, b, add=add, shift=sh, relu=True)
    outs = []
    try:
        for wide in (True, False):
            ops.native().set_wide_gemm_tiles(wide)
            d = ops.gemm_bf16(a, b, col_shift=sh, relu=True, add=add)
            fb.check_bf16(d, *ref, k, what="gemm wide=%s" % wide)
            outs.append(d)
    finally:
        ops.native().set_wide_gemm_tiles(True)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("m,n,k,res,scale", [(25088, 512, 512, False, False), (6272, 2048, 1024, True, False),
                                             (100352, 512, 256, True, True), (1568, 4096, 2048, False, True),
                                             (19000, 256, 320, True, False), (9601, 768, 4096, False, False)])
def test_inference_gemm_epilogue_on_large_shapes(m, n, k, res, scale):
    """The teacher's large GEMMs against fp32: M tails, K tails (k = 320: the last k-block is half out of bounds), the
    addend and the scale / shift / ReLU epilogue; persistent and one-tile-per-CTA kernels accumulate in the same order."""
    torch.manual_seed(3)
    nat = ops.native()
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = (torch.randn(n, k, device=DEV) * 0.05).bfloat16()
    sh = torch.randn(n, device=DEV)
    sc = (torch.rand(n, device=DEV) + 0.5) if scale else None
    add = torch.randn(m, n, device=DEV).bfloat16() if res else None
    d = ops.gemm_bf16(a, b, col_scale=sc, col_shift=sh, relu=True, add=add)
    fb.check_bf16(d, *fb.gemm_ref(a, b, add=add, scale=sc, shift=sh, relu=True), k, what="gemm epilogue")
    if not res:
        nat.set_persistent_gemm(False)
        assert torch.equal(d, ops.gemm_bf16(a, b, col_scale=sc, col_shift=sh, relu=True))


@pytest.mark.parametrize("m,n,k", [(100352, 256, 64), (25088, 128, 512), (5000, 384, 192)])
def test_sixteen_epilogue_warps_match_eight(m, n, k):
    """The 128- / 256-column kernels can run 16 consumer warps (64 rows x half of the tile's columns per warpgroup;
    EDL_EPI_WARPS=16 / set_epilogue_warps(16)) instead of 8: identical outputs, statistics within summation-order noise, for
    the forward GEMM with BN statistics, the dgrad with the fused BN-backward reduction and the 3x3 convolution."""
    torch.manual_seed(7)
    nat = ops.native()
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = (torch.randn(n, k, device=DEV) * 0.05).bfloat16()
    wmn = (torch.randn(k, n, device=DEV) * 0.05).bfloat16()
    x = torch.randn(m, n, device=DEV).bfloat16()
    xc = torch.randn(8, 128, 28, 28, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wc = (torch.randn(128, 3, 3, 128, device=DEV) * 0.05).bfloat16()
    res = []
    h = fb.bn_hook(x, None, n, True)
    try:
        for warps in (16, 8):
            nat.set_epilogue_warps(warps)
            st = torch.zeros(2 * n, device=DEV)
            d = ops.gemm_bf16(a, b, col_stats=st)
            h.dsums = torch.zeros(2 * n, device=DEV)
            g = ops.gemm_bf16(a, wmn, b_mn_major=True, bn=h)
            cst = torch.zeros(256, device=DEV)
            yc = ops.conv3x3(xc, wc, cst)
            res.append((d, st, g, h.dsums, yc, cst))
    finally:
        nat.set_epilogue_warps(8)
    for i in (0, 2, 4):
        assert torch.equal(res[0][i], res[1][i]), i
    for warps, (d, st, g, dsums, yc, cst) in zip((16, 8), res):
        # the statistics sum in a different order per warp count: both pass the oracle
        fb.check_bf16(d, *fb.gemm_ref(a, b), k, what="gemm %d warps" % warps)
        fb.check_sums(st, *fb.stats_ref(d), m, what="gemm stats %d warps" % warps)
        fb.check_bf16(g, *fb.gemm_ref(a, wmn, b_mn_major=True), k, what="dgrad %d warps" % warps)
        ref, mag, extra = fb.bn_dsums_ref(g, x, h.mean, h.rstd, h.gamma, h.beta, True)
        fb.check_sums(dsums, ref, mag, m, what="dgrad dsums %d warps" % warps, extra=extra)
        fb.check_bf16(yc, *fb.conv_ref(xc, wc), 9 * 128, what="conv3x3 %d warps" % warps)
        fb.check_sums(cst, *fb.stats_ref(yc), yc.numel() // 128, what="conv3x3 stats %d warps" % warps)


@pytest.mark.parametrize("kind,shape", [("gemm", (100352, 256, 64)), ("gemm", (5000, 192, 192)), ("gemm", (6272, 1024, 256)),
                                        ("gemm", (300, 128, 64)), ("conv", (32, 128, 128, 28, 28)), ("conv", (5, 128, 256, 11, 20)),
                                        ("conv", (9, 256, 256, 14, 14)), ("conv", (7, 512, 512, 7, 7))])
def test_forward_bn_statistics_match_fp32_sums_of_the_stored_output(kind, shape):
    """Forward BatchNorm statistics of the 128-column kernels against fp32 sums of the stored output: M tails, a partial N
    tile (192), alternating N tiles per CTA (1024 columns), conv tiles with partial patches and tail images."""
    torch.manual_seed(11)
    if kind == "gemm":
        m, n, k = shape
        a = torch.randn(m, k, device=DEV).bfloat16()
        b = (torch.randn(n, k, device=DEV) * 0.05).bfloat16()
    else:
        nb, c, n, h, w = shape
        x = torch.randn(nb, c, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
        wt = (torch.randn(n, 3, 3, c, device=DEV) * 0.05).bfloat16()
    st = torch.zeros(2 * n, device=DEV)
    y = ops.gemm_bf16(a, b, col_stats=st) if kind == "gemm" else ops.conv3x3(x, wt, st)
    if kind == "gemm":
        fb.check_bf16(y, *fb.gemm_ref(a, b), k, what="gemm")
    else:
        fb.check_bf16(y, *fb.conv_ref(x, wt), 9 * c, what="conv3x3")
    fb.check_sums(st, *fb.stats_ref(y), y.numel() // n, what="%s stats" % kind)


def test_persistent_gemm_epilogue_scale_shift_relu():
    torch.manual_seed(1)
    m, n, k = 5000, 256, 192
    a = torch.randn(m, k, device=DEV).bfloat16()
    b = torch.randn(n, k, device=DEV).bfloat16()
    sc, sh = torch.rand(n, device=DEV) + 0.5, torch.randn(n, device=DEV)
    d = ops.gemm_bf16(a, b, col_scale=sc, col_shift=sh, relu=True)
    fb.check_bf16(d, *fb.gemm_ref(a, b, scale=sc, shift=sh, relu=True), k, what="gemm ssr")


@pytest.mark.parametrize("n,cin,cout,h,w", [(32, 64, 64, 56, 56), (32, 128, 128, 28, 28), (32, 256, 256, 14, 14),
                                            (32, 512, 512, 7, 7), (5, 64, 192, 11, 20)])
def test_persistent_conv3x3_matches_tile_kernel(n, cin, cout, h, w):
    torch.manual_seed(2)
    x = torch.randn(n, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 3, 3, cin, device=DEV) * 0.05).bfloat16()
    res = []
    for persistent in (True, False):
        ops.native().set_persistent_gemm(persistent)
        st = torch.zeros(2 * cout, device=DEV)
        y = ops.conv3x3(x, wt, st)
        res.append((y, st))
    # the haloed-tile version accumulates in (filter row, k-block, tap) order, the tile kernel in (tap, k-block) order:
    # both pass the oracle
    ref = fb.conv_ref(x, wt)
    for persistent, (y, st) in zip((True, False), res):
        fb.check_bf16(y, *ref, 9 * cin, what="conv3x3 persistent=%s" % persistent)
        fb.check_sums(st, *fb.stats_ref(y), n * h * w, what="conv3x3 stats persistent=%s" % persistent)
    if cin <= 64 or cin % 128 == 0:
        dy = torch.randn_like(res[0][0])
        dref = fb.dgrad_ref(dy, wt, x.shape)
        for persistent in (True, False):
            ops.native().set_persistent_gemm(persistent)
            dx = torch.empty_like(x)
            ops.native().conv3x3(dy, wt, dx, True, None, None, False)
            fb.check_bf16(dx, *dref, 9 * cout, what="conv3x3 dgrad persistent=%s" % persistent)


@pytest.mark.parametrize("n,cin,cout,h,w,groups", [(32, 64, 64, 56, 56, 1), (8, 128, 128, 28, 28, 1), (9, 256, 256, 14, 14, 1),
                                                   (7, 512, 512, 7, 7, 1), (5, 64, 192, 11, 20, 1), (3, 128, 64, 9, 30, 1),
                                                   (2, 64, 64, 5, 127, 1), (3, 512, 512, 14, 14, 8), (2, 256, 512, 6, 6, 2),
                                                   (32, 2048, 2048, 14, 14, 32), (40, 192, 192, 7, 7, 3)])
def test_haloed_conv3x3_tiles_match_the_shifted_box_version(n, cin, cout, h, w, groups):
    """One A tile per filter row read through three shifted descriptors (EDL_CONV_HALO, the default) against one TMA box per
    tap, and both against the fp32 convolution: fprop with statistics / folded-BN epilogue, dgrad, grouped fprop."""
    torch.manual_seed(5)
    nat = ops.native()
    x = torch.randn(n, cin, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 3, 3, cin // groups, device=DEV) * 0.05).bfloat16()
    scale = torch.rand(cout, device=DEV) + 0.5
    shift = torch.randn(cout, device=DEV) * 0.1
    assert nat.get_conv_halo()
    outs = []
    try:
        for halo, resident in ((True, True), (True, False), (False, False)):
            nat.set_conv_halo(halo)
            nat.set_conv_resident_weights(resident)     # 64-channel layers / groups: weights loaded once per run of tiles
            if groups == 1:
                st = torch.zeros(2 * cout, device=DEV)
                y = ops.conv3x3(x, wt, st)
            else:
                st = None
                y = ops.conv3x3_infer(x, wt, scale, shift, relu=True, groups=groups)
            dx = None
            if groups == 1 and (cin <= 64 or cin % 128 == 0):
                dy = torch.randn_like(y)
                dx = torch.empty_like(x)
                nat.conv3x3(dy, wt, dx, True, None, None, False)
            outs.append((y, st, dx, dy if dx is not None else None))
    finally:
        nat.set_conv_halo(True)
        nat.set_conv_resident_weights(True)
    epi = dict(scale=scale.view(1, -1, 1, 1), shift=shift.view(1, -1, 1, 1), relu=True) if groups > 1 else {}
    ref = fb.conv_ref(x, wt, groups=groups, **epi)
    assert torch.equal(outs[0][0], outs[1][0])          # same accumulation order, only the tile schedule differs
    for (halo, resident), (y, st, dx, dy) in zip(((True, True), (True, False), (False, False)), outs):
        what = "conv3x3 halo=%s resident=%s" % (halo, resident)
        fb.check_bf16(y, *ref, 9 * cin // groups, what=what)
        if st is not None:
            fb.check_sums(st, *fb.stats_ref(y), n * h * w, what=what + " stats")
        if dx is not None:
            fb.check_bf16(dx, *fb.dgrad_ref(dy, wt, x.shape), 9 * cout, what=what + " dgrad")


def test_conv1x1_fork_sums_both_gradients_in_the_dgrad_epilogue():
    torch.manual_seed(3)
    x = torch.randn(8, 256, 14, 14, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = (torch.randn(64, 1, 1, 256, device=DEV) * 0.05).bfloat16().requires_grad_(True)
    r = torch.randn(8, 256, 14, 14, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    dy = torch.randn(8, 64, 14, 14, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    y, xa = ops.conv1x1(x, w, None, fork=True)
    torch.autograd.backward([y, xa], [dy, r])
    wd = w.detach()
    fb.check_bf16(x.grad, *fb.dgrad_ref(dy, wd, x.shape, padding=0, add=r), 64, what="fork dgrad + addend")
    fb.check_bf16(w.grad.view(64, 256), *fb.gemm_ref(fb.rows(dy), fb.rows(x.detach()), a_mn_major=True, b_mn_major=True),
                  8 * 14 * 14, ops.gemm._split_k_for(64, 256, 8 * 14 * 14), what="fork wgrad")
    # alias unused downstream: plain dgrad
    x2 = x.detach().clone().requires_grad_(True)
    y2, _ = ops.conv1x1(x2, w, None, fork=True)
    y2.backward(dy)
    fb.check_bf16(x2.grad, *fb.dgrad_ref(dy, wd, x.shape, padding=0), 64, what="fork dgrad")


@pytest.mark.parametrize("m,k,n", [(2048, 64, 32), (5000, 64, 128), (6272, 512, 256), (300, 64, 1024)])
@pytest.mark.parametrize("relu,has_y", [(True, False), (True, True), (False, False)])
def test_dgrad_epilogue_bn_backward_reduction_gemm(m, k, n, relu, has_y):
    """(experimental path, off by default) the 1x1 dgrad epilogue reduces sum(dy_m), sum(dy_m * xhat) of the tile."""
    torch.manual_seed(5)
    a = torch.randn(m, k, device=DEV).bfloat16()
    w = (torch.randn(k, n, device=DEV) * 0.1).bfloat16()
    x = torch.randn(m, n, device=DEV).bfloat16()
    y = torch.randn(m, n, device=DEV).bfloat16() if has_y else None
    h = fb.bn_hook(x, y, n, relu)
    d = ops.gemm_bf16(a, w, b_mn_major=True, bn=h)
    assert h.done
    fb.check_bf16(d, *fb.gemm_ref(a, w, b_mn_major=True), k, what="dgrad")
    fb.check_dsums(h, d, m, "dgrad dsums")


@pytest.mark.parametrize("nb,c,hh,ww", [(8, 64, 16, 16), (32, 256, 14, 14), (5, 64, 11, 20), (8, 256, 2, 2)])
def test_dgrad_epilogue_bn_backward_reduction_conv3x3(nb, c, hh, ww):
    torch.manual_seed(6)
    dy = torch.randn(nb, c, hh, ww, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(c, 3, 3, c, device=DEV) * 0.05).bfloat16()
    x = torch.randn(nb, c, hh, ww, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    h = fb.bn_hook(x, None, c, True)
    dx = torch.empty_like(x)
    ops.native().conv3x3(dy, wt, dx, True, None, h.as_list(nb * hh * ww, c), True)
    fb.check_bf16(dx, *fb.dgrad_ref(dy, wt, x.shape), 9 * c, what="conv3x3 dgrad")
    fb.check_dsums(h, dx, nb * hh * ww, "conv3x3 dgrad dsums")


@pytest.mark.parametrize("n,c,cout,h,w,groups", [(4, 2048, 2048, 14, 14, 32), (4, 4096, 4096, 7, 7, 32), (2, 256, 256, 12, 12, 4),
                                                 (3, 128, 256, 9, 9, 1)])
def test_grouped_conv3x3_inference_with_folded_bn_epilogue(n, c, cout, h, w, groups):
    torch.manual_seed(4)
    x = torch.randn(n, c, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 3, 3, c // groups, device=DEV) * 0.05).bfloat16()
    scale, shift = torch.rand(cout, device=DEV) + 0.5, torch.randn(cout, device=DEV) * 0.1
    assert ops.conv3x3_infer_supported(x, wt, groups)
    y = ops.conv3x3_infer(x, wt, scale, shift, True, groups)
    ref = fb.conv_ref(x, wt, groups=groups, scale=scale.view(1, -1, 1, 1), shift=shift.view(1, -1, 1, 1), relu=True)
    fb.check_bf16(y, *ref, 9 * c // groups, what="grouped conv3x3 infer")


def test_phase_trace_of_the_persistent_kernel():
    """set_persist_trace: CTA 0 stamps clock64() at the phase boundaries of its first tiles (tools/trace_persist.py)."""
    nat = ops.native()
    a = torch.randn(4096 * 8, 64, device=DEV).bfloat16()
    b = (torch.randn(128, 64, device=DEV) * 0.05).bfloat16()
    st = torch.zeros(256, device=DEV)
    buf = torch.zeros(3 * 16 * 8, dtype=torch.int64, device=DEV)
    nat.set_persist_trace(buf)
    try:
        ops.gemm_bf16(a, b, col_stats=st)
        torch.cuda.synchronize()
    finally:
        nat.set_persist_trace(None)
    t = buf.view(3, 16, 8).cpu()
    epi = t[2]
    assert (epi[0, :5] > 0).all()                          # tile 0: loop top .. store issued
    assert (epi[0, 1:5] >= epi[0, :4]).all()               # in order
    assert epi[1, 0] > epi[0, 4]                           # the second tile starts after the first one's store
    buf.zero_()
    ops.gemm_bf16(a, b, col_stats=st)                      # tracing off: nothing is written
    torch.cuda.synchronize()
    assert int(buf.abs().sum()) == 0


@pytest.mark.parametrize("n,h,w,cout", [(4, 224, 224, 64), (3, 65, 97, 64), (2, 32, 48, 128)])
def test_stem7_im2col_gemm_matches_the_convolution(n, h, w, cout):
    """The teacher's 7x7 / stride 2 / pad 3 stem: im2col kernel (window rows in KRSC order, zero-padded to 160 columns) +
    persistent GEMM with the folded-BN / ReLU epilogue, against the fp32 convolution; odd sizes exercise the padding."""
    torch.manual_seed(13)
    x = torch.randn(n, 3, h, w, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, 7, 7, 3, device=DEV) * 0.05).bfloat16()
    sc, sh = torch.rand(cout, device=DEV) + 0.5, torch.randn(cout, device=DEV) * 0.1
    assert ops.stem7_supported(x, wt)
    y = ops.stem7_infer(x, wt, sc, sh, relu=True)
    ref = fb.conv_ref(x, wt, 2, 3, scale=sc.view(1, -1, 1, 1), shift=sh.view(1, -1, 1, 1), relu=True)
    assert y.shape == ref[0].shape and y.is_contiguous(memory_format=torch.channels_last)
    fb.check_bf16(y, *ref, 160, what="stem7 infer")
