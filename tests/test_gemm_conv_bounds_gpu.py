"""Element-wise float64 bounds (tests/f64_bounds.py) for the GEMM / convolution paths no other test reaches: every
schedule switch of the persistent kernel, M / N / K tails and K block counts around each variant's pipeline depth,
padded row pitches with NaN around the operands and sentinels around the outputs, the fused BatchNorm-backward hook in
its three mask forms, both 3x3 weight-gradient versions, stride 2 and the stem kernels."""
import itertools
import math

import pytest
import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.ops import gemm as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = -3.0          # finite sentinel around outputs and sinks


def _bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).bfloat16()


def _nhwc(n, c, h, w, scale=1.0):
    return _bf(n, c, h, w, scale=scale).contiguous(memory_format=torch.channels_last)


@pytest.fixture(autouse=True)
def _restore_switches():
    C = ops.native()
    v3 = C.get_wgrad3_version()
    yield
    C.set_persistent_gemm(True)
    C.set_wide_gemm_tiles(True)
    C.set_epilogue_warps(8)
    C.set_conv_halo(True)
    C.set_conv_resident_weights(True)
    C.set_wgrad3_version(v3, 0)


# ------------------------------------------------------------------------------------------------------ GEMM forward
def _stages(n):
    return 6 if n <= 64 else 5          # 64- / 128-column variants of the persistent kernel


def _ks(n):
    s = _stages(n)
    return [72] + [64 * kb for kb in (s - 1, s, s + 1)]


def _operands(m, n, k, epi):
    """A, B (NaN padding, padded pitches), the epilogue and a guarded D."""
    a = fb.guarded((m, k), 1, 8, values=_bf(m, k))
    b = fb.guarded((n, k), 1, 16, values=_bf(n, k, scale=0.1))
    kw = {}
    if epi in ("stats",):
        kw["col_stats"] = torch.zeros(2 * n, device=DEV)
    if epi in ("bias", "all"):
        kw["col_shift"] = torch.randn(n, device=DEV)
        kw["relu"] = True
    if epi == "all":
        kw["col_scale"] = torch.rand(n, device=DEV) + 0.5
        kw["add"] = fb.guarded((m, n), 2, 8, values=_bf(m, n)).t
    return a, b, kw


def _run_gemm(a, b, kw, m, n, k, what):
    d = fb.guarded((m, n), 2, 24, fill=SENT)
    stats = kw.get("col_stats")
    if stats is not None:
        stats.zero_()
    ops.reset_fallbacks()
    ops.gemm_bf16(a.t, b.t, out=d.t, **kw)
    assert not ops.fallbacks(), ops.fallbacks()
    ref = fb.gemm_ref(a.t, b.t, add=kw.get("add"), scale=kw.get("col_scale"), shift=kw.get("col_shift"),
                      relu=kw.get("relu", False))
    fb.check_bf16(d.t, *ref, k, what=what)
    d.assert_untouched(what)
    if stats is not None:
        fb.check_sums(stats, *fb.stats_ref(d.t), m, what=what + " stats")
    return d.t.clone()


@pytest.mark.parametrize("epi", ["none", "stats", "bias", "all"])
@pytest.mark.parametrize("n", [8, 72, 192, 320])
@pytest.mark.parametrize("m", [1, 127, 129, 777, 128 * 132 + 1])
def test_gemm_forward_every_schedule_guarded(m, n, epi):
    """Persistent and one-tile-per-CTA, K = 72 (a partial last block) and stages - 1 .. stages + 1 k blocks.  The two
    schedules accumulate in the same order: identical bits."""
    C = ops.native()
    torch.manual_seed(m * 7 + n)
    for k in _ks(n):
        a, b, kw = _operands(m, n, k, epi)
        outs = []
        for persistent in (True, False):
            C.set_persistent_gemm(persistent)
            what = "gemm %dx%dx%d %s persistent=%s" % (m, n, k, epi, persistent)
            if not persistent and "add" in kw:
                # an addend followed by scale / shift / ReLU exists only as the persistent kernel's fused epilogue
                with pytest.raises(RuntimeError, match="addend"):
                    ops.gemm_bf16(a.t, b.t, **kw)
                continue
            outs.append(_run_gemm(a, b, kw, m, n, k, what))
        C.set_persistent_gemm(True)
        a.assert_untouched("A")
        b.assert_untouched("B")
        if len(outs) == 2:
            assert torch.equal(outs[0], outs[1]), (m, n, k, epi)


@pytest.mark.parametrize("m,n,k", [(128 * 132 + 1, 256, 256), (33000, 512, 320), (17000, 768, 256)])
@pytest.mark.parametrize("epi", ["none", "bias", "all"])
def test_gemm_forward_wide_tiles_and_epilogue_warps(m, n, k, epi):
    """128 x 256 tiles (N % 256 == 0, K >= 256, >= 132 tiles; 3 stages: K = 256 is stages + 1 k blocks) against the
    128-column tiles, and 16 against 8 epilogue warps: all identical bits, all within the bounds."""
    C = ops.native()
    torch.manual_seed(m + n + k)
    a, b, kw = _operands(m, n, k, epi)
    outs = []
    for wide, warps in ((True, 8), (False, 8), (True, 16), (False, 16)):
        C.set_wide_gemm_tiles(wide)
        C.set_epilogue_warps(warps)
        outs.append(_run_gemm(a, b, kw, m, n, k, "gemm %dx%dx%d %s wide=%s warps=%d" % (m, n, k, epi, wide, warps)))
    a.assert_untouched("A")
    b.assert_untouched("B")
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


# ------------------------------------------------------------------------------------------------------------ dgrad
@pytest.mark.parametrize("m,k", [(777, 64), (5001, 256), (129, 512)])
@pytest.mark.parametrize("n", [32, 64, 192, 1024])
@pytest.mark.parametrize("bn", [None, "x", "y", "bits"])
@pytest.mark.parametrize("with_add", [False, True])
def test_dgrad_with_addend_and_bn_hook_guarded(m, k, n, bn, with_add):
    """B MN-major (the dgrad form) into a guarded D with a padded pitch; the BatchNorm input / output share D's pitch and
    have NaN padding.  With mask bits the stored gradient is ``where(mask, ref, 0)``."""
    if bn == "bits" and n % 128 != 0:
        pytest.skip("mask bits need N % 128 == 0")
    torch.manual_seed(m + n + k)
    pad = 8 if bn is None else 0          # the fused reduction reads x / y with D's pitch and needs a dense D
    a = fb.guarded((m, k), 1, 8, values=_bf(m, k))
    w = fb.guarded((k, n), 1, 8, values=_bf(k, n, scale=0.1))
    add = fb.guarded((m, n), 1, pad, values=_bf(m, n)).t if with_add else None
    d = fb.guarded((m, n), 1, pad, fill=SENT)
    h = None
    if bn is not None:
        x = fb.guarded((m, n), 1, pad, values=_bf(m, n)).t
        y = fb.guarded((m, n), 1, pad, values=_bf(m, n)).t if bn == "y" else None
        keep = torch.rand(m, n, device=DEV) > 0.4 if bn == "bits" else None
        h = fb.bn_hook(x, y, n, True, mask=fb.mask_bits(keep) if keep is not None else None)
    ops.reset_fallbacks()
    ops.gemm_bf16(a.t, w.t, out=d.t, b_mn_major=True, add=add, bn=h)
    assert not ops.fallbacks(), ops.fallbacks()
    what = "dgrad %dx%dx%d bn=%s add=%s" % (m, n, k, bn, with_add)
    ref, mag = fb.gemm_ref(a.t, w.t, b_mn_major=True, add=add)
    if bn == "bits":
        ref = torch.where(keep, ref, torch.zeros_like(ref))
    fb.check_bf16(d.t, ref, mag, k, what=what)
    d.assert_untouched(what)
    a.assert_untouched("A")
    w.assert_untouched("B")
    if h is not None:
        assert h.done
        fb.check_dsums(h, d.t, m, what + " dsums", bits_keep=keep)


# ----------------------------------------------------------------------------------------------- weight-gradient GEMM
# the partial tiles of a split are fp32 [split, tiles, 128, block_n]; "max" (one k block per split) is capped where
# that buffer would exceed 1 GB, i.e. for the two large outputs at K >= 25088 (128 and 256 splits instead of 392 - 1568)
PARTIALS_CAP = 1 << 30


def _max_wgrad_split(cout, cin, k):
    block_n = 64 if cin <= 64 else 128
    tiles = ((cout + 127) // 128) * ((cin + block_n - 1) // block_n)
    return min(math.ceil(k / 64), PARTIALS_CAP // (tiles * 128 * block_n * 4))


@pytest.mark.parametrize("shape", [(64, 64), (256, 64), (64, 256), (1000, 2048), (2048, 512)])
@pytest.mark.parametrize("k", [1000, 1568, 25088, 100352])
def test_wgrad_gemm_fresh_and_into_a_guarded_sink(shape, k):
    """Splits 1, 3, automatic and one k block per split, each fresh and added into a prefilled window of a guarded
    flat gradient bucket."""
    cout, cin = shape
    torch.manual_seed(cout + cin + k)
    dy = _bf(k, cout)
    x = _bf(k, cin, scale=0.1)
    ref = fb.gemm_ref(dy, x, a_mn_major=True, b_mn_major=True)
    for split in (1, 3, None, "max"):
        sp = _max_wgrad_split(cout, cin, k) if split == "max" else split
        eff = sp if sp is not None else G._split_k_for(cout, cin, k)
        what = "wgrad gemm %dx%d k %d split %s (%d)" % (cout, cin, k, split, eff)
        d = G._wgrad_impl(dy, x, (cout, cin), None, split_k=sp)
        fb.check_bf16(d, *ref, k, eff, what=what)
        prior = _bf(cout * cin)
        sink = fb.guarded((cout * cin,), 64, fill=SENT, values=prior)
        assert G._wgrad_impl(dy, x, (cout, cin), sink.t, split_k=sp) is None
        fb.check_bf16(sink.t.view(cout, cin), *fb.epilogue(ref[0], ref[1], add=prior.view(cout, cin)), k, eff,
                      what=what + " sink")
        sink.assert_untouched(what + " sink")


# --------------------------------------------------------------------------------------------------- 3x3, stride 1
GEOMS = [(1, 64, 64, 9, 30), (3, 64, 128, 1, 40), (2, 64, 64, 6, 1), (2, 128, 64, 7, 2), (2, 64, 64, 5, 127),
         (1, 64, 192, 4, 128), (5, 64, 192, 11, 20), (2, 128, 128, 5, 127),
         (32, 64, 64, 56, 56), (32, 128, 128, 28, 28), (32, 256, 256, 14, 14), (32, 512, 512, 7, 7)]


def _conv_switches():
    return list(itertools.product((True, False), (True, False), (True, False)))      # halo, resident, persistent


def _set_conv(halo, resident, persistent):
    C = ops.native()
    C.set_conv_halo(halo)
    C.set_conv_resident_weights(resident)
    C.set_persistent_gemm(persistent)


@pytest.mark.parametrize("n,cin,cout,h,w", GEOMS)
def test_conv3x3_fprop_stats_every_switch(n, cin, cout, h, w):
    torch.manual_seed(n * h + w)
    x = _nhwc(n, cin, h, w)
    wt = _bf(cout, 3, 3, cin, scale=0.05)
    if not ops.conv3x3_supported(x, wt):
        pytest.skip("geometry not supported by the planner")
    ref = fb.conv_ref(x, wt)
    outs = {}
    for sw in _conv_switches():
        _set_conv(*sw)
        st = torch.zeros(2 * cout, device=DEV)
        y = ops.conv3x3(x, wt, st)
        what = "conv3x3 %s halo/resident/persistent=%s" % ((n, cin, cout, h, w), sw)
        fb.check_bf16(y, *ref, 9 * cin, what=what)
        fb.check_sums(st, *fb.stats_ref(y), n * h * w, what=what + " stats")
        outs[sw] = y
    # resident weights only change which tiles a CTA takes, not the accumulation order
    for persistent in (True, False):
        assert torch.equal(outs[(True, True, persistent)], outs[(True, False, persistent)]), persistent


@pytest.mark.parametrize("n,c,cout,h,w,groups", [(2, 256, 256, 12, 12, 4), (3, 512, 512, 7, 9, 8), (1, 128, 128, 5, 127, 1),
                                                 (4, 2048, 2048, 14, 14, 32), (2, 64, 64, 1, 33, 1)])
def test_conv3x3_infer_grouped_every_switch(n, c, cout, h, w, groups):
    torch.manual_seed(groups + h)
    x = _nhwc(n, c, h, w)
    wt = _bf(cout, 3, 3, c // groups, scale=0.05)
    sc, sh = torch.rand(cout, device=DEV) + 0.5, torch.randn(cout, device=DEV) * 0.1
    if not ops.conv3x3_infer_supported(x, wt, groups):
        pytest.skip("geometry not supported by the planner")
    ref = fb.conv_ref(x, wt, groups=groups, scale=sc.view(1, -1, 1, 1), shift=sh.view(1, -1, 1, 1), relu=True)
    for sw in _conv_switches():
        _set_conv(*sw)
        if not sw[2]:
            # the folded-BN epilogue and the groups exist only in the persistent kernel
            with pytest.raises(RuntimeError):
                ops.conv3x3_infer(x, wt, sc, sh, True, groups)
            continue
        y = ops.conv3x3_infer(x, wt, sc, sh, True, groups)
        fb.check_bf16(y, *ref, 9 * c // groups, what="conv3x3 infer g%d %s" % (groups, sw))


@pytest.mark.parametrize("n,cin,cout,h,w", [g for g in GEOMS if g[1] % 64 == 0 and (g[2] <= 64 or g[2] % 128 == 0)])
@pytest.mark.parametrize("bn", [False, True])
def test_conv3x3_dgrad_guarded_with_and_without_bn_hook(n, cin, cout, h, w, bn):
    torch.manual_seed(n + h + w + bn)
    C = ops.native()
    dy = _nhwc(n, cout, h, w)
    wt = _bf(cout, 3, 3, cin, scale=0.05)
    xs = (n, cin, h, w)
    if not C.conv3x3_supported(n, h, w, cin, cout, True, 1):
        pytest.skip("geometry not supported by the planner")
    ref = fb.dgrad_ref(dy, wt, xs)
    x = _nhwc(*xs)
    for persistent in (True, False) if not bn else (True,):
        C.set_persistent_gemm(persistent)
        dx = fb.guarded(xs, 3, fill=SENT)
        h_ = None
        if bn:
            h_ = fb.bn_hook(x, None, cin, True)
        C.conv3x3(dy, wt, dx.t, True, None, h_.as_list(n * h * w, cin) if bn else None, bn)
        what = "conv3x3 dgrad %s bn=%s persistent=%s" % ((n, cin, cout, h, w), bn, persistent)
        fb.check_bf16(dx.t, *ref, 9 * cout, what=what)
        dx.assert_untouched(what)
        if bn:
            fb.check_dsums(h_, dx.t, n * h * w, what + " dsums")


def _wgrad3_max_split(n, h, w, s2=False):
    C = ops.native()
    return C.conv3x3_wgrad_s2_kblocks(n, h, w) if s2 else C.conv3x3_wgrad_kblocks(n, h, w)


def _check_wgrad3(x, dy, shape, split, stride, what):
    """Fresh and into a guarded sink; ``split`` in {int, None, "max"}."""
    cout = shape[0]
    n, _, ho, wo = dy.shape
    s2 = stride == 2
    sp = _wgrad3_max_split(n, ho, wo, s2) if split == "max" else split
    eff = sp if sp is not None else G.conv3x3_wgrad_split(n, ho, wo, shape[3], cout, s2)
    ref, mag = [t.reshape(cout, -1) for t in fb.wgrad_ref(x, dy, shape, stride)]
    k = n * ho * wo
    got = ops.conv3x3_wgrad(x, dy, shape, None, split_k=sp)
    fb.check_bf16(got.reshape(cout, -1), ref, mag, k, eff, what=what)
    prior = _bf(cout * 9 * shape[3])
    sink = fb.guarded(prior.shape, 64, fill=SENT, values=prior)
    assert ops.conv3x3_wgrad(x, dy, shape, sink.t, split_k=sp) is None
    fb.check_bf16(sink.t.view(cout, -1), *fb.epilogue(ref, mag, add=prior.view(cout, -1)), k, eff, what=what + " sink")
    sink.assert_untouched(what + " sink")


WGRAD3 = [(2, 64, 64, 9, 30), (1, 64, 128, 4, 128), (5, 64, 192, 11, 20), (2, 128, 64, 5, 127),
          (8, 64, 64, 56, 56), (8, 128, 128, 28, 28), (8, 256, 256, 14, 14), (32, 512, 512, 7, 7)]


@pytest.mark.parametrize("n,cin,cout,h,w", WGRAD3)
@pytest.mark.parametrize("version", [1, 2])
def test_conv3x3_wgrad_both_versions(n, cin, cout, h, w, version):
    C = ops.native()
    torch.manual_seed(n + h + version)
    x = _nhwc(n, cin, h, w)
    dy = _nhwc(n, cout, h, w, scale=0.1)
    shape = (cout, 3, 3, cin)
    C.set_wgrad3_version(version, 0)
    if not ops.conv3x3_wgrad_supported(x, torch.empty(shape, device=DEV, dtype=torch.bfloat16)):
        pytest.skip("geometry not supported by the pixel-box planner")
    for split in (1, 4, None, "max"):
        _check_wgrad3(x, dy, shape, split, 1, "conv3x3 wgrad v%d %s split %s" % (version, (n, cin, cout, h, w), split))


# --------------------------------------------------------------------------------------------------------- stride 2
S2 = [(32, 128, 128, 56, 56), (32, 256, 256, 28, 28), (32, 512, 512, 14, 14), (3, 64, 128, 18, 42)]


@pytest.mark.parametrize("n,cin,cout,h,w", S2)
def test_conv3x3_stride2_fprop_dgrad_wgrad(n, cin, cout, h, w):
    C = ops.native()
    torch.manual_seed(h + w)
    x = _nhwc(n, cin, h, w)
    wt = _bf(cout, 3, 3, cin, scale=0.05)
    if not ops.conv3x3_s2_supported(x, wt):
        pytest.skip("shape not supported")
    st = torch.zeros(2 * cout, device=DEV)
    y = ops.conv3x3_s2(x, wt, st)
    what = "conv3x3 s2 %s" % ((n, cin, cout, h, w),)
    fb.check_bf16(y, *fb.conv_ref(x, wt, 2), 9 * cin, what=what)
    fb.check_sums(st, *fb.stats_ref(y), y.numel() // cout, what=what + " stats")
    dy = _nhwc(n, cout, h // 2, w // 2)
    if C.conv3x3_dgrad_s2_supported(n, h // 2, w // 2, cin, cout):
        dx = fb.guarded(x.shape, 3, fill=SENT)
        C.conv3x3_dgrad_s2(dy, wt, dx.t)
        fb.check_bf16(dx.t, *fb.dgrad_ref(dy, wt, x.shape, 2), 9 * cout, what=what + " dgrad")
        dx.assert_untouched(what + " dgrad")
    if C.conv3x3_wgrad_s2_supported(n, h // 2, w // 2, cin, cout):
        for split in (1, 4, None, "max"):
            _check_wgrad3(x, dy * 0.1, (cout, 3, 3, cin), split, 2, what + " wgrad split %s" % split)


# ------------------------------------------------------------------------------------------------------------- stem
@pytest.mark.parametrize("n,h,w", [(4, 224, 224), (3, 34, 46), (2, 17, 33)])
def test_stem_conv_stats_and_weight_gradient(n, h, w):
    torch.manual_seed(h)
    x = _nhwc(n, 3, h, w)
    wt = _bf(32, 3, 3, 3, scale=0.2)
    st = torch.zeros(64, device=DEV)
    y = ops.stem_conv(x, wt, st)
    fb.check_bf16(y, *fb.conv_ref(x, wt, 2), 27, what="stem conv")
    fb.check_sums(st, *fb.stats_ref(y), y.numel() // 32, what="stem conv stats")
    if h % 2 or w % 2:
        return                                              # odd images take the library weight gradient
    dy = _nhwc(*y.shape)
    ref, mag = [t.reshape(32, -1) for t in fb.wgrad_ref(x, dy, wt.shape, 2)]
    k = dy.numel() // 32
    C = ops.native()
    ws, counters = G._stem_scratch(x.device)
    # two calls in a row: the second starts from the scratch the first left behind, which must be zero again.  (The
    # CTAs' partials meet in fp32 atomics, so the two results may differ in their last bit: both pass the oracle.)
    for i in range(2):
        out = torch.empty_like(wt)
        C.stem_wgrad(x, dy, out, ws, counters, False)
        torch.cuda.synchronize()
        assert not ws.any() and not counters.any(), "the in-kernel reduction left its scratch dirty"
        fb.check_bf16(out.view(32, -1), ref, mag, k, 132, what="stem wgrad call %d" % i)
    prior = _bf(32 * 27)
    sink = fb.guarded(prior.shape, 64, fill=SENT, values=prior)
    C.stem_wgrad(x, dy, sink.t.view(wt.shape), ws, counters, True)
    fb.check_bf16(sink.t.view(32, -1), *fb.epilogue(ref, mag, add=prior.view(32, -1)), k, 132, what="stem wgrad sink")
    sink.assert_untouched("stem wgrad sink")
    assert not ws.any() and not counters.any()


@pytest.mark.parametrize("n,cout,h,w", [(2, 32, 112, 112), (3, 64, 20, 24), (1, 32, 7, 130)])
def test_pair_conv_fprop_dgrad_wgrad(monkeypatch, n, cout, h, w):
    monkeypatch.setattr(G, "OWN_STEM23", True)
    torch.manual_seed(h)
    x = _nhwc(n, 32, h, w).requires_grad_(True)
    wt = _bf(cout, 3, 3, 32, scale=0.1).requires_grad_(True)
    if not ops.conv3x3_pair_supported(x, wt):
        pytest.skip("geometry not supported")
    st = torch.zeros(2 * cout, device=DEV)
    y = ops.conv3x3_pair(x, wt, st)
    xd, wd = x.detach(), wt.detach()
    fb.check_bf16(y, *fb.conv_ref(xd, wd), 9 * 64, what="pair conv")
    fb.check_sums(st, *fb.stats_ref(y), y.numel() // cout, what="pair conv stats")
    dy = _nhwc(*y.shape)
    y.backward(dy)
    fb.check_bf16(x.grad, *fb.dgrad_ref(dy, wd, x.shape), 9 * 2 * cout, what="pair dgrad")
    # the 64-channel weight gradient over n h w / 2 pixel pairs (its automatic split), then one fp32 addition per element
    fb.check_pair_wgrad(wt.grad, xd, dy, wd.shape, n * h * w // 2, G.conv3x3_wgrad_split(n, h, w // 2, 64, 2 * cout) + 1)


@pytest.mark.parametrize("n,h,w,cout", [(2, 224, 224, 64), (1, 9, 13, 32)])
def test_stem7_infer(n, h, w, cout):
    torch.manual_seed(w)
    x = _nhwc(n, 3, h, w)
    wt = _bf(cout, 7, 7, 3, scale=0.05)
    sc, sh = torch.rand(cout, device=DEV) + 0.5, torch.randn(cout, device=DEV) * 0.1
    y = ops.stem7_infer(x, wt, sc, sh, relu=True)
    fb.check_bf16(y, *fb.conv_ref(x, wt, 2, 3, scale=sc.view(1, -1, 1, 1), shift=sh.view(1, -1, 1, 1), relu=True), 160,
                  what="stem7")
