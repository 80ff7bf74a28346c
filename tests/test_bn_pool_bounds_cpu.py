"""The BatchNorm and pooling references of tests/f64_bounds.py without a GPU: against independent ones (float64
F.batch_norm and its autograd, naive pooling loops), the propagated statistics bound against an fp32 emulation of the
streaming kernels' reduction, the checker accepting kernel-like fp32 outputs and rejecting each corruption a broken
kernel would make, with a message that names the channel, tile or element."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import f64_bounds as fb
from edl_b200 import ops

EPS, MOM = 1e-5, 0.1


def _rejects(fn, *args, match, **kw):
    with pytest.raises(AssertionError, match=match):
        fn(*args, **kw)


def _bn_inputs(m, c, seed=0, res=True):
    g = torch.Generator().manual_seed(seed)
    offs = torch.tensor([0.0, 4.0, -16.0, 16.0, -4.0, 0.0])[torch.arange(c) % 6]
    x = ((torch.randn(m, c, generator=g) + offs) * (torch.rand(c, generator=g) * 1.5 + 0.5)).bfloat16()
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.2
    gamma[2], gamma[3] = 0.0, -gamma[3]
    r = torch.randn(m, c, generator=g).bfloat16() if res else None
    dy = torch.randn(m, c, generator=g).bfloat16()
    return x, r, gamma, beta, dy


# ------------------------------------------------------------------------------------------ independent references
def test_bn_references_match_float64_batch_norm_and_autograd():
    m, c = 500, 24
    x, r, gamma, beta, dy = _bn_inputs(m, c)
    x64 = x.double().requires_grad_()
    g64, b64 = gamma.double().requires_grad_(), beta.double().requires_grad_()
    r64 = r.double().requires_grad_()
    z = F.batch_norm(x64, None, None, g64, b64, True, 0.0, fb.f32(EPS)) + r64
    y = z.relu().bfloat16()                              # a stored output, whose mask the backward takes
    keep = (y > 0).double()
    (z * keep).backward(dy.double())
    ex = fb.bn_exact(x, gamma, beta, EPS, r, True, y=y, dy=dy)
    assert torch.allclose(ex["y"][0], z.relu().detach(), rtol=1e-12, atol=1e-12)
    for name, want in (("dx", x64.grad), ("dres", r64.grad), ("dgamma", g64.grad), ("dbeta", b64.grad)):
        assert torch.allclose(ex[name][0], want, rtol=1e-9, atol=1e-9), name
        assert (ex[name][1] >= ex[name][0].abs() - 1e-9).all(), name
    # the staged references with exact statistics and exact dsums are the same functions
    mu, var, _, _ = fb.bn_exact_stats(x)
    rstd = torch.rsqrt(var + fb.f32(EPS))
    assert torch.allclose(fb.bn_y_ref(x, mu, rstd, gamma, beta, r, True)[0], ex["y"][0], rtol=1e-12, atol=1e-12)
    dsums = torch.cat([ex["dbeta"][0], ex["dgamma"][0]])
    assert torch.allclose(fb.bn_dx_ref(dy, x, mu, rstd, gamma, dsums, m, y > 0)[0], ex["dx"][0], rtol=1e-9, atol=1e-9)


def _naive_maxpool(x, last=False, pad_value=float("-inf")):
    """Loops over the windows, first maximum in (kh, kw) order (``last``: the last one; ``pad_value``: what a padded tap
    reads).  Returns (values, flat h W + w index)."""
    n, c, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    xv = x.double().numpy()
    val, idx = np.zeros((n, c, ho, wo)), np.zeros((n, c, ho, wo), dtype=np.int64)
    for b, ch, i, j in itertools.product(range(n), range(c), range(ho), range(wo)):
        best, bi = float("-inf"), -1
        for kh, kw in itertools.product(range(3), range(3)):
            ih, iw = 2 * i - 1 + kh, 2 * j - 1 + kw
            inside = 0 <= ih < h and 0 <= iw < w
            v = xv[b, ch, ih, iw] if inside else pad_value
            if v > best or (last and v == best):
                best, bi = v, ih * w + iw
        val[b, ch, i, j], idx[b, ch, i, j] = best, bi
    return torch.from_numpy(val), torch.from_numpy(idx)


def _pool_inputs(shape, kind, seed=1):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(shape, generator=g)
    return {"relu": v.relu(), "negative": -v.abs() - 0.01,
            "integers": torch.randint(-2, 3, shape, generator=g).float()}[kind].bfloat16()


@pytest.mark.parametrize("shape,kind", [((2, 8, 7, 9), "relu"), ((1, 8, 6, 5), "negative"), ((2, 8, 5, 5), "integers")])
def test_pool_references_match_naive_loops(shape, kind):
    x = _pool_inputs(shape, kind)
    ref, idx = fb.maxpool_ref(x)
    nv, ni = _naive_maxpool(x)
    assert torch.equal(ref, nv) and torch.equal(idx, ni)
    slots = fb.maxpool_slots(idx, shape[3])
    assert bool(((slots >= 0) & (slots < 9)).all())
    dy = torch.randn(ref.shape).bfloat16()
    dx, mag = fb.maxpool_bwd_ref(dy, idx, shape)
    naive = torch.zeros(shape, dtype=torch.float64).view(shape[0], shape[1], -1)
    for b, ch, i, j in itertools.product(*(range(s) for s in ref.shape)):
        naive[b, ch, idx[b, ch, i, j]] += float(dy[b, ch, i, j])
    assert torch.equal(dx, naive.view(shape)) and (mag >= dx.abs()).all()
    # average pool: exclusive 2 x 2 windows in ceil mode
    n, c, h, w = shape
    ap, _ = fb.avgpool_ref(x)
    for b, ch, i, j in itertools.product(range(n), range(c), range((h + 1) // 2), range((w + 1) // 2)):
        win = x.double()[b, ch, 2 * i:2 * i + 2, 2 * j:2 * j + 2]
        assert ap[b, ch, i, j] == win.sum() / win.numel()
    assert torch.equal(fb.dilate2_ref(x)[:, :, ::2, ::2], x) and fb.dilate2_ref(x).sum() == x.sum()


def test_bn_reduce_plan_covers_every_row():
    """chain x threads per channel x partials >= M for every path: no row is left out of the bound."""
    for (m, c), path in itertools.product([(401408, 32), (100352, 64), (100352, 256), (25088, 512), (6272, 1024),
                                            (1568, 2048), (1568, 512), (8192, 8), (64, 4096), (1000, 256),
                                            (17024, 64), (2048, 32)], ["regs", "stream", "fused"]):
        chain, tree, parts = fb.bn_reduce_plan(path, m, c)
        assert chain * 2 ** tree * parts >= m, (path, m, c)
    for m, c in [(3000, 24), (37, 72), (2, 200), (3, 1000), (8191, 8)]:
        chain, tree, parts = fb.bn_reduce_plan("regs", m, c)
        assert chain * 2 ** tree * parts >= m, (m, c)
    assert fb.bn_reduce_plan("stream", 401408, 64) == (48, 6, 132)


def _stream_emulation(x, m, c):
    """fp32 sums of one channel in the streaming kernels' order: ``partials`` CTAs x 2^tree threads, each adding a
    chain of rows (fma for the squares), a tree over the threads, then the partials in some order."""
    chain, tree, parts = fb.bn_reduce_plan("stream", m, c)
    nthr = parts * 2 ** tree
    xs = np.concatenate([x.float().numpy(), np.zeros(chain * nthr - m, np.float32)]).reshape(chain, nthr)
    s, q = np.zeros(nthr, np.float32), np.zeros(nthr, np.float32)
    for row in xs:
        s = (s + row).astype(np.float32)
        q = (q.astype(np.float64) + row.astype(np.float64) ** 2).astype(np.float32)
    s, q = s.reshape(parts, -1), q.reshape(parts, -1)
    while s.shape[1] > 1:
        h = s.shape[1] // 2
        s, q = (s[:, :h] + s[:, h:]).astype(np.float32), (q[:, :h] + q[:, h:]).astype(np.float32)
    order = np.random.default_rng(0).permutation(parts)
    S, Q = np.float32(0), np.float32(0)
    for p in order:
        S, Q = np.float32(S + s[p, 0]), np.float32(Q + q[p, 0])
    return torch.tensor([S, Q])


def _kernel_stats(sums, m, eps):
    """The apply kernels' statistics in fp32: mean = s fl(1/M), var = max(q fl(1/M) - mean^2, 0), rsqrt(var + eps)."""
    c = sums.numel() // 2
    inv = torch.tensor(1.0) / torch.tensor(float(m))
    mean = sums[:c] * inv
    var = (sums[c:] * inv - mean * mean).clamp_min(0)
    return mean, torch.rsqrt(var + eps), var


@pytest.mark.parametrize("ratio", [0, 4, 16])
def test_propagated_statistics_bound_holds_for_the_stream_chains(ratio):
    m, c = 401408, 64
    g = torch.Generator().manual_seed(ratio)
    x = (torch.randn(m, 1, generator=g) + ratio).bfloat16()
    sums = _stream_emulation(x[:, 0], m, c)
    fb.check_sums(sums, *fb.stats_ref(x), m, tau_s=fb.bn_reduce_tau("stream", m, c), what="emulated sums")
    mean, rstd, _ = _kernel_stats(sums, m, EPS)
    fb.check_bn_saved_stats(sums, mean, rstd, m, EPS, what="emulated")
    r1, r2 = fb.check_bn_stats_e2e(x, mean, rstd, EPS, fb.bn_reduce_tau("stream", m, c), what="emulated")
    assert r1 < 1 and r2 < 1


# ----------------------------------------------------------------------------------------- accepting and rejecting
def _kernel_fwd(x, r, gamma, beta, relu=True, m_scale=None):
    """fp32 BatchNorm apply as the kernels do it (statistics from fp32 sums, fmaf(x, scale, shift), + res, ReLU) and the
    running-statistics update.  ``m_scale``: a per-channel factor on ``scale`` (a corruption)."""
    m, c = x.shape
    sums = torch.cat([x.float().sum(0), x.float().square().sum(0)])
    mean, rstd, var = _kernel_stats(sums, m, EPS)
    sc = gamma * rstd
    sh = beta - mean * sc
    if m_scale is not None:
        sc = sc * m_scale
    y = (x.double() * sc.double() + sh.double()).float()
    if r is not None:
        y = y + r.float()
    y = y.relu() if relu else y
    return sums, mean, rstd, var, y


def _kernel_bwd(d, x, mean, rstd, gamma, keep):
    m, c = x.shape
    g = d.float() * keep if keep is not None else d.float()
    xhat = (x.float() - mean) * rstd
    dsums = torch.cat([g.sum(0), (g * xhat).sum(0)])
    inv = torch.tensor(1.0) / torch.tensor(float(m))
    dx = (gamma * rstd) * (g - dsums[:c] * inv - xhat * (dsums[c:] * inv))
    return dsums, dx


def test_checker_accepts_kernel_like_batchnorm():
    m, c = 3000, 48
    x, r, gamma, beta, dy = _bn_inputs(m, c)
    sums, mean, rstd, var, yf = _kernel_fwd(x, r, gamma, beta)
    y = yf.bfloat16()
    fb.check_sums(sums, *fb.stats_ref(x), m, tau_s=fb.bn_reduce_tau("regs", m, c))
    rm0, rv0 = torch.randn(c) * 0.1, torch.rand(c) + 0.5
    mom = torch.tensor(MOM, dtype=torch.float32)
    rm = (1 - mom) * rm0 + mom * mean
    rv = (1 - mom) * rv0 + mom * (var * (torch.tensor(float(m)) / torch.tensor(float(m - 1))))
    fb.check_bn_saved_stats(sums, mean, rstd, m, EPS, running=(rm0, rv0, rm, rv, MOM))
    fb.check_bf16(y, *fb.bn_y_ref(x, mean, rstd, gamma, beta, r, True), tau=fb.BN_Y_TAU, criteria=(1,))
    ex = fb.bn_exact(x, gamma, beta, EPS, r, True, y=y, dy=dy)
    fb.check_bf16(y, *ex["y"], criteria=(2,))
    keep = y > 0
    dsums, dx = _kernel_bwd(dy, x, mean, rstd, gamma, keep)
    fb.check_sums(dsums, *fb.bn_dsums_ref(dy, x, mean, rstd, gamma, beta, True, y=y)[:2], m,
                  tau_s=fb.bn_reduce_tau("regs", m, c))
    fb.check_bf16(dx.bfloat16(), *fb.bn_dx_ref(dy, x, mean, rstd, gamma, dsums, m, keep), tau=fb.BN_DX_TAU,
                  criteria=(1,))
    fb.check_bf16(dx.bfloat16(), *ex["dx"], criteria=(2,))


def test_checker_accepts_the_cpu_batch_norm_act():
    """``ops.batch_norm_act``'s fp32 CPU path, end to end (criterion 2) against the exact statistics."""
    m, c = 2000, 32
    x, r, gamma, beta, dy = _bn_inputs(m, c, seed=2)
    xi = x.clone().requires_grad_()
    ri = r.clone().requires_grad_()
    y = ops.batch_norm_act(xi, gamma, beta, torch.zeros(c), torch.ones(c), residual=ri, relu=True)
    y.backward(dy)
    ex = fb.bn_exact(x, gamma, beta, EPS, r, True, y=y.detach(), dy=dy)
    fb.check_bf16(y.detach(), *ex["y"], criteria=(2,), what="cpu y")
    fb.check_bf16(xi.grad, *ex["dx"], criteria=(2,), what="cpu dx")
    fb.check_exact(ri.grad, torch.where(y.detach() > 0, dy, torch.zeros_like(dy)), what="cpu dres")


def test_rejects_one_channel_group_scale_off_by_0p3_percent():
    m, c = 3000, 48
    x, r, gamma, beta, _ = _bn_inputs(m, c)
    f = torch.ones(c)
    f[16:24] = 1.003
    _, mean, rstd, _, y = _kernel_fwd(x, r, gamma, beta, relu=False, m_scale=f)
    ex = fb.bn_exact(x, gamma, beta, EPS, r, False)
    _rejects(fb.check_bf16, y.bfloat16(), *ex["y"], criteria=(2,), what="scale",
             match=r"criterion 2: .* columns .* worst (1[6-9]|2[0-3]):")
    # with a column left out of criterion 2, the message still names the channels by their own index
    _rejects(fb.check_bf16, y.bfloat16(), *ex["y"], criteria=(2,), columns=torch.arange(c) != 1, what="scale",
             match=r"criterion 2: .* columns .* worst (1[6-9]|2[0-3]):")


def test_rejects_rounding_toward_zero():
    m, c = 3000, 48
    x, r, gamma, beta, _ = _bn_inputs(m, c)
    _, mean, rstd, _, y = _kernel_fwd(x, r, gamma, beta)
    rtz = (y.view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
    _rejects(fb.check_bf16, rtz, *fb.bn_exact(x, gamma, beta, EPS, r, True)["y"], criteria=(2,), what="rtz",
             match="criterion 2")


def test_rejects_a_stale_last_partial_chunk_of_dx():
    """(1000, 256): 31 whole 16 KB chunks and a partial one, rows 992 .. 999; the partial chunk left as it was."""
    m, c = 1000, 256
    x, r, gamma, beta, dy = _bn_inputs(m, c, res=False)
    _, mean, rstd, _, y = _kernel_fwd(x, None, gamma, beta)
    keep = y.bfloat16() > 0
    dsums, dx = _kernel_bwd(dy, x, mean, rstd, gamma, keep)
    stale = dx.bfloat16()
    stale.view(-1)[31 * 8192:] = torch.randn(m * c - 31 * 8192).bfloat16()
    _rejects(fb.check_bf16, stale, *fb.bn_dx_ref(dy, x, mean, rstd, gamma, dsums, m, keep), tau=fb.BN_DX_TAU,
             criteria=(1,), what="stale", match=r"criterion 1: .* first at \(992, ")


def test_rejects_a_biased_running_variance():
    m, c = 1000, 16
    x, _, gamma, beta, _ = _bn_inputs(m, c)
    sums, mean, rstd, var, _ = _kernel_fwd(x, None, gamma, beta)
    rm0, rv0 = torch.zeros(c), torch.ones(c)
    mom = torch.tensor(MOM, dtype=torch.float32)
    rm = (1 - mom) * rm0 + mom * mean
    biased = (1 - mom) * rv0 + mom * var                 # M instead of M - 1
    _rejects(fb.check_bn_saved_stats, sums, mean, rstd, m, EPS, running=(rm0, rv0, rm, biased, MOM), what="biased",
             match=r"running var: \d+ of 16 channels")


def test_rejects_dres_stored_unmasked_and_dgamma_overwritten():
    m, c = 300, 16
    x, r, gamma, beta, dy = _bn_inputs(m, c)
    _, mean, rstd, _, y = _kernel_fwd(x, r, gamma, beta)
    keep = y.bfloat16() > 0
    _rejects(fb.check_exact, dy, torch.where(keep, dy, torch.zeros_like(dy)), what="dres", match=r"dres: \d+ of 4800")
    dsums, _ = _kernel_bwd(dy, x, mean, rstd, gamma, keep)
    prior = torch.randn(c)
    _rejects(fb.check_exact, dsums[c:], prior + dsums[c:], what="dgamma", match="dgamma: 16 of 16")


def _emulated_maxpool(x, last=False, pad_value=float("-inf")):
    """The kernel's max-pool in fp32 (``>`` over the taps in (kh, kw) order, best starting at -inf), vectorised;
    ``last`` (``>=``) and ``pad_value`` (padded taps read as a value) are corruptions.  Returns (y, slots)."""
    n, c, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    xp = F.pad(x.float(), (1, 2, 1, 2), value=pad_value if pad_value != float("-inf") else float("-inf"))
    best = torch.full((n, c, ho, wo), float("-inf"))
    slot = torch.zeros((n, c, ho, wo), dtype=torch.int64)
    for kh, kw in itertools.product(range(3), range(3)):
        v = xp[:, :, kh:kh + 2 * ho:2, kw:kw + 2 * wo:2]
        take = (v >= best) if last else (v > best)
        best, slot = torch.where(take, v, best), torch.where(take, kh * 3 + kw, slot)
    return best.bfloat16(), slot


@pytest.mark.parametrize("shape,kind", [((2, 8, 9, 11), "relu"), ((2, 8, 7, 7), "negative"),
                                        ((2, 8, 10, 8), "integers")])
def test_checker_accepts_emulated_pool_kernels(shape, kind):
    x = _pool_inputs(shape, kind)
    y, slots = _emulated_maxpool(x)
    idx = fb.check_maxpool(y, slots, x, what="emulated maxpool")
    dy = torch.randn(y.shape).bfloat16()
    n, c, h, w = shape
    dx = torch.zeros(n, c, h * w)
    dx.view(n, c, -1).scatter_add_(2, idx.view(n, c, -1), dy.float().view(n, c, -1))
    fb.check_bf16(dx.view(shape).bfloat16(), *fb.maxpool_bwd_ref(dy, idx, shape), tau=3 * fb.EPS32)
    ap = F.avg_pool2d(x.float(), 2, 2, 0, ceil_mode=True, count_include_pad=False).bfloat16()
    fb.check_bf16(ap, *fb.avgpool_ref(x), tau=3 * fb.EPS32, what="emulated avgpool")
    # global average pool: 8 chains of ceil(HW / 8), then the 8 partials, times fl(1 / HW)
    xs = x.float().reshape(n, c, -1)
    parts = torch.zeros(n, c, 8)
    for i in range(h * w):
        parts[:, :, i % 8] += xs[:, :, i]
    s = torch.zeros(n, c)
    for j in range(8):
        s += parts[:, :, j]
    gap = (s * (torch.tensor(1.0) / torch.tensor(float(h * w)))).bfloat16()
    fb.check_bf16(gap, *fb.gap_ref(x), tau=fb.gap_tau(h * w), what="emulated gap")
    dg = torch.randn(n, c).bfloat16()
    gdx = (dg.float() * (torch.tensor(1.0) / torch.tensor(float(h * w))))[:, :, None, None].expand(shape).bfloat16()
    fb.check_bf16(gdx, *fb.gap_bwd_ref(dg, shape), tau=2 * fb.EPS32, what="emulated gap dx")


def test_rejects_a_maxpool_tie_routed_to_the_last_maximum():
    x = _pool_inputs((2, 8, 9, 9), "relu")
    y, slots = _emulated_maxpool(x, last=True)
    _rejects(fb.check_maxpool, y, slots, x, what="last", match=r"last arg-max slot: \d+ of 400 elements differ")


def test_rejects_maxpool_padding_treated_as_zero():
    x = _pool_inputs((2, 8, 9, 9), "negative")
    y, slots = _emulated_maxpool(x, pad_value=0.0)
    _rejects(fb.check_maxpool, y, slots, x, what="pad0", match=r"pad0 y: \d+ of 400 elements differ, first at flat "
                                                                r"index 0 \(\[0, 0, 0, 0\]\)")


def test_mask_edge_construction_separates_fma_from_mul_sub():
    """``bn_mask_edge`` (the data of the GPU recomputed-mask test) makes a forward that forms the shift ``b - m g r`` as a
    product and a subtraction and a backward that forms it with one fma disagree on every x == 0 element of a channel
    with a positive residual, while random data leaves them in agreement."""
    m, c = 6272, 64
    g = torch.Generator().manual_seed(3)
    x = torch.randint(-3, 4, (m, c), generator=g).bfloat16()
    mean, rstd, _ = _kernel_stats(torch.cat([x.float().sum(0), x.float().square().sum(0)]), m, EPS)

    def masks(gamma, beta):
        sc = gamma * rstd                                                    # fp32
        sh_mul = beta - (mean * sc)                                          # fp32 product, then fp32 subtraction
        sh_fma = (beta.double() - mean.double() * sc.double()).float()       # one rounding
        pre = lambda sh: x.double() * sc.double() + sh.double()             # fmaf keeps the exact value's sign
        return pre(sh_mul) > 0, pre(sh_fma) > 0

    gamma0 = torch.rand(c, generator=g) + 0.5
    a, b = masks(gamma0, torch.randn(c, generator=g) * 0.2)
    assert int((a != b).sum()) < 10                                          # random beta: (almost) no element differs
    gamma, beta, resid = fb.bn_mask_edge(mean, rstd, gamma0)
    assert int((resid > 0).sum()) >= c - 2 and bool((resid >= 0).all())
    a, b = masks(gamma, beta)
    edge = (x == 0) & (resid > 0)
    assert torch.equal(a != b, edge) and int(edge.sum()) > m * c // 10
