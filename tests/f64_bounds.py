"""Float64 oracle for the bf16 GEMM and convolution kernels (csrc/gemm.cu, gemm_persist.cu, conv3x3.cu,
conv3x3_wgrad.cu, stem.cu) and the BatchNorm and pooling kernels (bn.cu, bn_stream.cu, bn_fused.cu, pool.cu):
element-wise bounds instead of a global relative norm, which hides one wrong row, column, channel, tile or tail.

Every reference is built in float64 from exactly the bf16 tensors the kernel read: ``ref`` is the value and ``mag`` the
same operation on absolute values (``sum_k |a_k b_k|``, then the epilogue with ``|add|``, ``|scale|``, ``|shift|`` and
no ReLU), i.e. the scale of the rounding errors an fp32 evaluation of the expression can make.  ``check_bf16`` applies
two criteria, both must hold:

1. per element: ``|out - ref| <= 1/2 ulp_bf16(|ref| + slack) + slack`` with ``slack = tau * mag`` and
   ``tau = (ceil(k / 16) + split + 1) * 2^-23``: one fp32 rounding per 16-deep MMA step, one per split-K partial, one for
   the epilogue, at 2^-23 rather than 2^-24 in case the tensor core truncates its adds.  Taking the ulp at
   ``|ref| + slack`` allows the extra half ulp where the accumulated value crossed a bf16 rounding boundary; a ReLU
   output whose pre-activation lies within the slack of 0 may be 0 or that small positive value (ReLU is 1-Lipschitz,
   so the same bound covers it).  NaN fails.
2. RMS per 128 x 128 output tile and per output column (channel):
   ``RMS(out - ref) <= 1.25 RMS(bf16(ref) - ref) + 2^-20 RMS(mag)``.  The yardstick is the error of rounding the exact
   result once to bf16; an fp32 accumulation that stays well below bf16 rounding keeps the ratio near 1, while rounding
   toward zero (2x), one channel's scale off by 0.3 % or shift off by 0.02, or one missing k term / k block exceed it.

``check_sums`` bounds the fused per-channel reductions (forward BatchNorm statistics of the stored output, the
BatchNorm-backward ``dsums`` of the dgrad epilogue) by ``tau_s * sum|terms|`` per channel with
``tau_s = (128 + ceil(M / 128)) * 2^-23``: the kernels sum a tile's rows in fp32 chains of at most 128 terms, then add one
partial per tile (atomics in any order).

``guarded`` places a tensor as a window inside a larger buffer filled with a sentinel: NaN around operands (a read past
M, N or K poisons the output), a finite value around outputs and sinks (``assert_untouched`` finds a stray store).

Worst ratios observed on one H100 SXM (80 GB, default power limit), over tests/test_gemm_gpu.py, test_persist_gpu.py,
test_conv3x3_gpu.py, test_round2_gpu.py, test_wgrad_splitk_gpu.py and test_gemm_conv_bounds_gpu.py (criterion 1 =
worst |out - ref| / bound, criterion 2 = worst RMS over tiles and columns / yardstick):

    GEMM forward (all schedules, wide tiles, 8 / 16 warps)   c1 1.000   c2 1.00
    1x1 dgrad (addend, BN hook)                              c1 1.000   c2 1.00
    weight-gradient GEMM (split 1 .. k blocks, sinks)        c1 1.000   c2 1.00
    3x3 / stride-2 / stem / 7x7 fprop                        c1 1.000   c2 1.00
    3x3 dgrad (stride 1 and 2)                               c1 0.999   c2 1.00
    3x3 weight gradient (versions 1 and 2, stride 2)         c1 0.999   c2 1.00
    stem weight gradient                                     c1 1.000   c2 1.00
    pixel-pair weight gradient (two bf16 partials, ``terms``)   c1 0.972   c2 1.00
    statistics and BN-backward sums (check_sums)             c1 0.05

and over tests/test_bn_pool_bounds_gpu.py, test_kernels_gpu.py and test_relu_mask_gpu.py (NVIDIA H100 80GB HBM3,
700 W power limit; register, streaming and SM-resident BatchNorm kernels alike):

    BatchNorm y, dx from the kernel's statistics (tau)       c1 1.000
    BatchNorm y, dx end to end (exact statistics)                        c2 1.01
    ops.batch_norm_act end to end (y, dx, dres)                          c2 1.00
    BatchNorm sums / dsums (bn_reduce_tau)                   c1 0.13
    saved mean / running statistics (staged)                 c1 0.50 / 0.28
    saved mean vs exact statistics (propagated bound)        c1 0.07
    saved rstd, staged and vs exact                          c1 1.000 (the constant channel: rsqrtf(eps) at the
                                                             interval's end, since the variance cannot go below 0)
    scale_shift_act, max-pool dx, average pool, global pool  c1 1.000   c2 1.00
and layer by layer inside whole training steps (tests/test_step_oracle_gpu.py: ResNet50_vd, ResNet18_vd and plain
ResNet50, every BatchNorm mode, the trainer and its graph replays; NVIDIA H100 80GB HBM3, 700 W power limit):

    conv fprop (all paths), BatchNorm y and dx, dgrad           c1 1.000   c2 1.00
    activation gradients summed over consumers (``terms``)      c1 0.991   c2 1.03
    weight gradients in .grad and bucket windows                c1 1.000   c2 1.06 (library layers, criterion 2 alone)
    dgamma / dbeta (check_sums)                                 c1 0.06
    saved statistics, staged / vs exact                         c1 0.50 / 0.10
    running statistics, staged / vs exact                       c1 0.17 / 0.08
    pools, global pool backward                                 c1 1.000   c2 1.00
and layer by layer inside the ResNeXt teacher's inference forward (tests/test_teacher_oracle_gpu.py: ResNeXt101_32x16d,
ResNeXt50_32x4d and ResNeXt_tiny with random folded BatchNorm, every convolution path, a graph replay; NVIDIA H100 80GB
HBM3, 700 W power limit):

    teacher bf16 layers (1x1, fused / two-kernel residual,     c1 1.000   c2 1.00
      widened / stride-2 / subsampled grouped 3x3, stem, classifier)
    FP8 block layers (fp8_tau, criterion 1 alone)              c1 0.773
    FP8 per-tensor layers (fp8_tensor_tau, criterion 1 alone;  c1 0.817
      the bound is derived from the block model, these are its first measurements)
c1 sits at 1 because a correctly rounded element near a rounding midpoint has an error of half an ulp.

Set ``EDL_F64_BOUNDS_LOG`` to a file name to append one JSON line per check with both ratios."""
import json
import math
import os

import torch
import torch.nn.functional as F

EPS32 = 2.0 ** -23           # per-rounding bound of an fp32 operation (truncating adds included)
C2_FACTOR = 1.25             # criterion 2: allowed RMS error relative to correct rounding of the exact result
C2_MAG = 2.0 ** -20          # criterion 2: floor relative to RMS(mag) (outputs whose rounding error is ~0)
TILE = 128


def ulp(x, mant_bits):
    """Unit in the last place of float64 values ``x`` in a format with ``mant_bits`` significant bits (0 at 0)."""
    _, e = torch.frexp(x)
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - mant_bits))


def tau(k, split=1):
    return (math.ceil(k / 16) + split + 1) * EPS32


_gemm_tau = tau


def bf16_round(x64):
    """float64 -> nearest bf16 (ties to even), as float64, without an intermediate float32 rounding."""
    x = x64.double()
    fin = torch.isfinite(x) & (x != 0)
    u = ulp(x.abs().where(fin, torch.ones_like(x)), 8)
    q = torch.round(x / u) * u           # round-half-even on the bf16 grid of x's binade (exact in float64)
    return torch.where(fin, q, x)


# ------------------------------------------------------------------------------------------------------- references
def epilogue(acc, mag, add=None, scale=None, shift=None, relu=False):
    """The kernels' epilogue in their order -- ``add``, then ``scale``, ``shift``, ``relu`` (ops/gemm.py:gemm_bf16's
    fallback) -- on the float64 accumulator and, with absolute values and no ReLU, on its magnitude."""
    if add is not None:
        acc, mag = acc + add.double(), mag + add.double().abs()
    if scale is not None:
        acc, mag = acc * scale.double(), mag * scale.double().abs()
    if shift is not None:
        acc, mag = acc + shift.double(), mag + shift.double().abs()
    if relu:
        acc = torch.relu(acc)
    return acc, mag


def gemm_ref(a, b, a_mn_major=False, b_mn_major=False, **epi):
    """(ref, mag) of ``ops.gemm_bf16``'s operand conventions: A [M, K] (or [K, M]), B [N, K] (or [K, N])."""
    a64 = a.double().t() if a_mn_major else a.double()
    b64 = b.double() if b_mn_major else b.double().t()
    return epilogue(a64 @ b64, a64.abs() @ b64.abs(), **epi)


def conv_ref(x, w_krsc, stride=1, padding=1, groups=1, **epi):
    """(ref, mag) of a convolution with a KRSC weight, as NCHW-shaped float64 tensors."""
    x64, w64 = x.double(), w_krsc.double().permute(0, 3, 1, 2)
    acc = F.conv2d(x64, w64, None, stride, padding, 1, groups)
    mag = F.conv2d(x64.abs(), w64.abs(), None, stride, padding, 1, groups)
    return epilogue(acc, mag.reshape(acc.shape), **epi)


def dgrad_ref(dy, w_krsc, x_shape, stride=1, padding=1, groups=1, add=None):
    """(ref, mag) of the input gradient of that convolution (+ ``add``)."""
    w64 = w_krsc.double().permute(0, 3, 1, 2)
    acc = torch.nn.grad.conv2d_input(x_shape, w64, dy.double(), stride, padding, 1, groups)
    mag = torch.nn.grad.conv2d_input(x_shape, w64.abs(), dy.double().abs(), stride, padding, 1, groups)
    return epilogue(acc, mag, add=add)


def wgrad_ref(x, dy, w_shape_krsc, stride=1, padding=1, groups=1, sink=None):
    """(ref, mag) of the KRSC weight gradient of that convolution (+ the prior ``sink`` contents)."""
    cout, kh, kw, cin = w_shape_krsc
    shp = (cout, cin, kh, kw)
    acc = torch.nn.grad.conv2d_weight(x.double(), shp, dy.double(), stride, padding, 1, groups).permute(0, 2, 3, 1)
    mag = torch.nn.grad.conv2d_weight(x.double().abs(), shp, dy.double().abs(), stride, padding, 1, groups).permute(0, 2, 3, 1)
    return epilogue(acc, mag, add=None if sink is None else sink.reshape(acc.shape))


def rows(t):
    """A kernel output as a 2-D [rows, channels] matrix: NCHW-shaped channels_last tensors as [N * H * W, C]."""
    if t.dim() == 4:
        return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])
    return t.reshape(t.shape[0], -1) if t.dim() != 2 else t


# -------------------------------------------------------------------------------------------------------- the check
def _log(what, c1, c2):
    path = os.environ.get("EDL_F64_BOUNDS_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"what": what, "c1": c1, "c2": c2}) + "\n")


def _tile_sums(x, tile):
    m, n = x.shape
    tm, tn = -(-m // tile), -(-n // tile)
    p = x.new_zeros(tm * tile, tn * tile)
    p[:m, :n] = x
    return p.view(tm, tile, tn, tile).sum((1, 3))


def check_bf16(out, ref, mag, k=0, split=1, what="", tile=TILE, c2_factor=C2_FACTOR, terms=None, tau=None,
               criteria=(1, 2), columns=None):
    """Criteria 1 and 2 above on a bf16 kernel output against its float64 (ref, mag).  4-D NCHW-shaped tensors are
    checked as [pixels, channels]; KRSC weight gradients are passed as [Cout, 9 Cin].  Returns the worst ratios
    (criterion 1: worst error / bound; criterion 2: worst RMS error / yardstick, failing above ``c2_factor``).

    ``tau``: the per-element slack factor of a non-GEMM operation (a count of fp32 roundings times ``EPS32``) in place
    of ``tau(k, split)``.  ``criteria``: the criteria that must hold (both by default); an end-to-end reference whose
    inputs differ from the kernel's by their own rounding bound is judged by criterion 2 alone.  ``columns``: a bool [N]
    of the columns criterion 2 judges (the others are left out of the tile and column RMS; indices in messages stay
    those of the full output).

    ``terms``: for a path that stores partial results as bf16 and then adds them (the pixel-pair weight gradient), the
    float64 (ref, mag) of each partial, with ``ref`` their sum.  Criterion 1 then also allows each partial its own half
    ulp (at ``|term| + slack``), and criterion 2's yardstick becomes the correct rounding of each stage:
    ``bf16(sum bf16(term))``."""
    o, r, g = rows(out).double(), rows(ref).double().to(out.device), rows(mag).double().to(out.device)
    assert o.shape == r.shape == g.shape, (what, o.shape, r.shape, g.shape)
    t_el = _gemm_tau(k, split) if tau is None else tau
    slack = t_el * g
    bound = 0.5 * ulp(r.abs() + slack, 8) + slack
    yard = bf16_round(r)
    if terms:
        tr = [rows(t).double().to(out.device) for t, _ in terms]
        tm = [rows(t).double().to(out.device) for _, t in terms]
        assert all(t.shape == r.shape for t in tr + tm), what
        for t, tg in zip(tr, tm):
            bound = bound + 0.5 * ulp(t.abs() + t_el * tg, 8)
        yard = bf16_round(sum(bf16_round(t) for t in tr))
    err = (o - r).abs()
    bad = ~(err <= bound)                                    # NaN fails
    c1 = float((err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max()) if o.numel() else 0.0
    m, n = o.shape
    judged = (torch.ones(n, dtype=torch.float64, device=o.device) if columns is None
              else columns.to(o.device, torch.float64)).expand(m, n)
    e2 = ((o - r).square().nan_to_num(float("inf")) * judged).nan_to_num(0.0, posinf=float("inf"))
    y2 = (yard - r).square() * judged
    g2 = g.square() * judged
    msgs = []
    c2 = 0.0
    for name, esum, ysum, gsum, cnt in (
            ("tile", _tile_sums(e2, tile), _tile_sums(y2, tile), _tile_sums(g2, tile), _tile_sums(judged, tile)),
            ("column", e2.sum(0), y2.sum(0), g2.sum(0), judged.sum(0))):
        cnt = cnt.clamp_min(1)                               # a tile or column with nothing judged has 0 / 1
        rms_e, rms_y, rms_g = (esum / cnt).sqrt(), (ysum / cnt).sqrt(), (gsum / cnt).sqrt()
        allowed = c2_factor * rms_y + C2_MAG * rms_g
        ratio = rms_e / (allowed / c2_factor).clamp_min(1e-300)
        c2 = max(c2, float(ratio.max())) if ratio.numel() else c2
        over = ~(rms_e <= allowed)
        if over.any() and 2 in criteria:
            worst = torch.argsort(ratio.flatten(), descending=True)[:4].tolist()
            if name == "tile":
                desc = ["(%d, %d): %.3g x yardstick" % (i // ratio.shape[1], i % ratio.shape[1], float(ratio.flatten()[i]))
                        for i in worst]
            else:
                desc = ["%d: %.3g x yardstick" % (i, float(ratio[i])) for i in worst]
            msgs.append("criterion 2: %d of %d %ss over %.2f x the RMS error of correct rounding, worst %s" % (
                int(over.sum()), over.numel(), name, c2_factor, ", ".join(desc)))
    c1 = c1 if 1 in criteria else None
    c2 = c2 if 2 in criteria else None
    _log(what, c1, c2)
    if bad.any() and c1 is not None:
        excess = torch.where(bad, (err - bound).nan_to_num(float("inf")), torch.zeros_like(err))
        cnt_t = _tile_sums(bad.double(), tile)
        ex_t = F.max_pool2d(F.pad(excess, (0, (-n) % tile, 0, (-m) % tile))[None, None], tile)[0, 0]
        order = torch.argsort(cnt_t.flatten(), descending=True)[:4].tolist()
        tiles = ", ".join("(%d, %d): %d bad, worst excess %.3g" % (i // cnt_t.shape[1], i % cnt_t.shape[1],
                                                                  int(cnt_t.flatten()[i]), float(ex_t.flatten()[i]))
                          for i in order if cnt_t.flatten()[i] > 0)
        i, j = bad.nonzero()[0].tolist()
        cols = torch.argsort(bad.sum(0), descending=True)[:4].tolist()
        msgs.insert(0, "criterion 1: %d of %d elements out of bounds; worst (row-tile, column-tile) blocks %s; first at "
                       "(%d, %d): out %r, ref %r, allowed +-%.3g; worst columns %s" % (
                           int(bad.sum()), bad.numel(), tiles, i, j, float(o[i, j]), float(r[i, j]), float(bound[i, j]),
                           ", ".join("%d (%d bad)" % (c, int(bad[:, c].sum())) for c in cols if bad[:, c].any())))
    if msgs:
        raise AssertionError("%s [%d x %d, k %d, split %d]: %s" % (what, m, n, k, split, "; ".join(msgs)))
    return c1, c2


def check_sums(got, ref, mag, m, what="", extra=None, tau_s=None):
    """Per-channel fp32 reductions over ``m`` rows: ``|got - ref| <= tau_s * mag + extra`` (``extra``: an absolute
    allowance, e.g. for mask elements that are ambiguous in fp32)."""
    ts = tau_s if tau_s is not None else (128 + math.ceil(m / TILE)) * EPS32
    gd, r, g = got.double(), ref.double().to(got.device), mag.double().to(got.device)
    bound = ts * g + (extra.double().to(got.device) if extra is not None else 0.0)
    err = (gd - r).abs()
    bad = ~(err <= bound)
    c1 = float((err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max()) if got.numel() else 0.0
    _log(what, c1, None)
    if bad.any():
        idx = torch.argsort((err - bound).nan_to_num(float("inf")), descending=True)[:4].tolist()
        raise AssertionError("%s: %d of %d sums out of bounds (tau_s %.3g), worst %s" % (
            what, int(bad.sum()), bad.numel(), ts, ", ".join("[%d] got %r ref %r allowed +-%.3g" % (
                i, float(gd[i]), float(r[i]), float(bound[i])) for i in idx)))
    return c1


def stats_ref(d):
    """(ref, mag) of the forward statistics [sum, sum of squares] per column of the STORED bf16 output."""
    d64 = rows(d).double()
    s, q = d64.sum(0), d64.square().sum(0)
    return torch.cat([s, q]), torch.cat([d64.abs().sum(0), q])


def bn_mask_fp32(x, mean, rstd, gamma, beta):
    """The dgrad epilogue's ReLU mask recomputed from the BatchNorm input: ``fmaf(x, g r, b - m g r) > 0`` with the
    per-channel constants formed in fp32.  An fmaf rounds once and keeps the sign of the exact value, which float64
    reproduces (a bf16 times an fp32 is exact in float64); the shift ``b - m g r`` may be compiled with or without a
    fused multiply-add, so both roundings are formed.  Returns (mask, ambiguous): elements where they disagree, or whose
    pre-activation lies within fp32 rounding of 0, may go either way."""
    sc = gamma.float() * rstd.float()
    sh_mul = beta.float() - mean.float() * sc                                    # two roundings
    sh_fma = (beta.double() - mean.float().double() * sc.double()).float()      # one rounding
    x64 = x.double()
    pre_mul = x64 * sc.double() + sh_mul.double()
    pre_fma = x64 * sc.double() + sh_fma.double()
    tol = 4 * EPS32 * ((x64 * sc.double()).abs() + sh_mul.double().abs())
    return pre_mul > 0, ((pre_mul > 0) != (pre_fma > 0)) | (pre_mul.abs() <= tol)


def bn_mask_edge(mean, rstd, gamma):
    """(gamma, beta, residual) that put every x == 0 element on the ReLU's edge, for saved statistics that do not depend
    on gamma and beta (integer inputs: their fp32 sums are exact, so every path saves the same mean and rstd).  With
    ``sc = fl(gamma rstd)`` and ``p = mean sc`` (exact in float64), ``beta = fl(p)`` makes the shift ``beta - mean sc``
    exactly 0 when it is formed as a product and a subtraction, and the product's rounding residual ``fl(p) - p`` when it
    is formed with one fma.  gamma's sign is chosen per channel so that the residual is positive: an x == 0 element is
    then masked (pre-activation 0) under one contraction and kept (pre-activation > 0) under the other.  ``residual`` is
    float64 [C], 0 in a channel whose product is exact."""
    def prod(g):
        sc = (g.float() * rstd.float()).double()
        return mean.double() * sc
    p = prod(gamma)
    gamma = torch.where(p.float().double() < p, -gamma, gamma)
    p = prod(gamma)
    pf = p.float().double()
    return gamma, pf.float(), pf - p


def bn_dsums_ref(d, x, mean, rstd, gamma, beta, relu, y=None, mask=None):
    """(ref, mag, extra) of the fused BatchNorm-backward reduction [sum dy_m, sum dy_m * xhat] per channel over the
    STORED gradient ``d``: ``dy_m = d * (y > 0)`` with the BN output, ``d`` itself with mask bits (the stored gradient
    is already masked), ``d * mask(x)`` otherwise.  The kernel forms ``rstd * (sum dy_m x - mean sum dy_m)``, so the
    magnitude of the second sum includes both terms; ``extra`` holds ``|d| (1 + |xhat|)`` of the ambiguous mask elements."""
    d64, x64 = rows(d).double(), rows(x).double()
    mean64, rstd64 = mean.double(), rstd.double()
    xhat = (x64 - mean64) * rstd64
    extra = None
    if relu and mask is None:
        if y is not None:
            keep = rows(y).double() > 0
        else:
            keep, amb = bn_mask_fp32(rows(x), mean, rstd, gamma, beta)
            t = d64.abs() * amb
            extra = torch.cat([t.sum(0), (t * xhat.abs()).sum(0)]) * 1.0001
        d64 = d64 * keep
    s = d64.sum(0)
    ref = torch.cat([s, (d64 * xhat).sum(0)])
    mag = torch.cat([d64.abs().sum(0), rstd64 * ((d64 * x64).abs().sum(0) + (mean64.abs() * d64.abs().sum(0)))])
    if extra is None:
        extra = torch.zeros_like(ref)
    return ref, mag, extra


def bn_hook(x, y, n, relu, mask=None):
    """A ``BNBackwardHook`` over BatchNorm input ``x`` (and output ``y`` or ReLU ``mask`` bits) with random per-channel
    constants and zeroed ``dsums``, as a train-mode BatchNorm leaves it for the dgrad that consumes its output."""
    from edl_b200.ops.bn import BNBackwardHook

    dev = x.device
    h = BNBackwardHook()
    h.x, h.y, h.mask, h.relu = x, y, mask, relu
    h.mean, h.rstd = torch.randn(n, device=dev) * 0.1, torch.rand(n, device=dev) + 0.5
    h.gamma, h.beta = torch.rand(n, device=dev) + 0.5, torch.randn(n, device=dev) * 0.2
    h.dsums = torch.zeros(2 * n, device=dev)
    return h


def check_dsums(h, d, m, what, bits_keep=None):
    """The fused BatchNorm-backward reduction in ``h.dsums`` against float64 sums over the STORED gradient ``d``
    (``bits_keep``: the bool mask behind ``h.mask``, whose gradient is stored already masked)."""
    ref, mag, extra = bn_dsums_ref(d, h.x, h.mean, h.rstd, h.gamma, h.beta, h.relu, y=h.y, mask=bits_keep)
    return check_sums(h.dsums, ref, mag, m, what=what, extra=extra)


def check_pair_wgrad(got, x, dy, shape, k, split, what="pair wgrad"):
    """Weight gradient of a 3x3 / stride 1 convolution with 32 input channels in pixel-pair form (ops/gemm.py
    ``_pair_wgrad``): the 64-channel weight gradient over pixel pairs is stored in bf16, then csrc/misc.cu
    pair_weight_fold adds two of its elements into each of ours.  Those two partials are the weight gradient restricted
    to output pixels of even and of odd column, each rounded to bf16 before the addition."""
    cout = shape[0]
    col = torch.arange(dy.shape[3], device=dy.device) % 2
    terms = [[t.reshape(cout, -1) for t in wgrad_ref(x, dy * (col == p).to(dy.dtype), shape)] for p in (0, 1)]
    ref, mag = [t.reshape(cout, -1) for t in wgrad_ref(x, dy, shape)]
    return check_bf16(got.reshape(cout, -1), ref, mag, k, split, what=what, terms=terms)


def mask_bits(keep):
    """uint8 [M, N / 8] ReLU mask bits (bit b of byte j = column 8 j + b) of a bool [M, N]."""
    m, n = keep.shape
    w = (2 ** torch.arange(8, device=keep.device, dtype=torch.int32))
    return (keep.view(m, n // 8, 8).int() * w).sum(-1).to(torch.uint8)


# ---------------------------------------------------------------------------------- BatchNorm and pooling references
NUM_SMS = 132
BN_Y_TAU = 4 * EPS32         # y = relu(fmaf(x, g r, b - m g r) + res): g r, m g r, the fma and the residual add
BN_DX_TAU = 8 * EPS32        # dx = g r (dy - db / M - xhat dg / M): 1/M, two quotients, xhat (2), the product, 2 subtractions
# criterion 2 end to end needs this many rows per channel: over fewer, the yardstick (the RMS of rounding the exact
# result to bf16) depends on whether those few values happen to sit near the bf16 grid
E2E_MIN_ROWS = 64


def bn_reduce_plan(path, m, c):
    """(chain, tree, partials) of the BatchNorm kernels' per-channel fp32 reductions over ``m`` rows: the longest
    chain of additions one thread makes, the depth of the in-block tree over the threads that share a channel, and the
    number of per-block partials added by atomics.  ``path``: "regs" (bn.cu, grid of ``bn_grid(M, C, 4 * 132)``),
    "stream" (bn_stream.cu ``reduce_grid``: 16 KB chunks, two 8-channel vectors per consumer thread and chunk) or
    "fused" (bn_fused.cu ``plan``)."""
    cv = c // 8
    if path == "regs":
        tx = 1 << (min(cv, 32).bit_length() - 1)
        ty = 256 // tx
        gx = -(-cv // tx)
        gy = max(1, min(4 * NUM_SMS // gx, -(-m // (4 * ty))))
        return -(-m // (gy * ty)), int(math.log2(ty)), gy
    n = -(-m * c // 8192)
    tree = int(math.log2(512 // cv))
    if path == "stream":
        grid = max(1, min(-(-n // 4), NUM_SMS))
        return 2 * -(-n // grid), tree, grid
    if path == "fused":
        k = -(-n // min(n, NUM_SMS))
        return 2 * k, tree, -(-n // k)
    raise ValueError(path)


def bn_reduce_tau(path, m, c):
    """fp32 rounding bound of those reductions relative to ``sum |terms|``: one rounding per addition on the deepest
    path, and 3 for the per-term ``xhat`` and fma."""
    chain, tree, parts = bn_reduce_plan(path, m, c)
    return (chain + tree + parts + 3) * EPS32


def f32(v):
    """A Python number rounded to fp32, as a float64 scalar (the kernels' ``(float)`` casts)."""
    return float(torch.tensor(v, dtype=torch.float64).float())


def f32_div(a, b):
    """fp32 ``a / b`` correctly rounded (the kernels' ``1.f / (float)M``)."""
    return float(torch.tensor([float(a)], dtype=torch.float32) / torch.tensor([float(b)], dtype=torch.float32))


def _rstd_interval(var, dvar, eps):
    """``rsqrtf(var + eps)`` for a variance within ``var +- dvar``: the add rounds once and rsqrtf is within 2 ulp."""
    lo = torch.rsqrt((var + dvar).clamp_min(0) + eps) * (1 - 3 * EPS32)
    hi = torch.rsqrt((var - dvar).clamp_min(0) + eps) * (1 + 3 * EPS32)
    return lo, hi


def check_interval(got, lo, hi, what=""):
    """Per-channel ``lo <= got <= hi``; returns the worst distance from the middle over the half-width."""
    g, lo, hi = got.double(), lo.double().to(got.device), hi.double().to(got.device)
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    ratio = ((g - mid).abs() / half.clamp_min(1e-300)).nan_to_num(float("inf"))
    c1 = float(ratio.max()) if g.numel() else 0.0
    _log(what, c1, None)
    bad = ~((g >= lo) & (g <= hi))
    if bad.any():
        idx = torch.argsort(ratio, descending=True)[:4].tolist()
        raise AssertionError("%s: %d of %d channels out of bounds, worst %s" % (
            what, int(bad.sum()), bad.numel(), ", ".join("[%d] got %r allowed [%r, %r]" % (
                i, float(g[i]), float(lo[i]), float(hi[i])) for i in idx)))
    return c1


def check_bn_saved_stats(sums, mean, rstd, m, eps, what="", running=None):
    """The saved ``mean``/``rstd`` (and, with ``running = (rm0, rv0, rm, rv, momentum)``, the running statistics before
    and after) against float64 formulas on the kernel's own fp32 ``sums`` [sum, sum of squares]: ``mean = s fl(1/M)``,
    ``var = max(q fl(1/M) - mean^2, 0)`` with the saved mean (within 2 ulps of ``q/M + mean^2``),
    ``rstd = rsqrt(var + eps)``, running statistics updated with the unbiased ``var M / (M - 1)``.  A wrong formula
    (biased running variance, eps outside the square root, momentum on the wrong side) fails."""
    c = mean.numel()
    inv = f32_div(1, m)
    s, q = sums[:c].double(), sums[c:].double()
    mref = s * inv
    check_interval(mean, mref - EPS32 * mref.abs(), mref + EPS32 * mref.abs(), what=what + " mean")
    m64 = mean.double()
    var = q * inv - m64 * m64
    dvar = 2 * EPS32 * (q * inv + m64 * m64)
    lo, hi = _rstd_interval(var, dvar, f32(eps))
    check_interval(rstd, lo, hi, what=what + " rstd")
    if running is not None:
        rm0, rv0, rm, rv, momentum = running
        mom = f32(momentum)
        one_m = f32(1.0 - mom)
        ratio = f32_div(m, m - 1) if m > 1 else 1.0
        a, b = one_m * rm0.double(), mom * m64
        ref, slack = a + b, 3 * EPS32 * (a.abs() + b.abs())
        check_interval(rm, ref - slack, ref + slack, what=what + " running mean")
        a, b = one_m * rv0.double(), mom * ratio * var.clamp_min(0)
        ref, slack = a + b, 3 * EPS32 * (a.abs() + b.abs()) + mom * ratio * dvar
        check_interval(rv, ref - slack, ref + slack, what=what + " running var")


def bn_exact_stats(x):
    """Exact float64 batch statistics of a bf16 [M, C] (or NCHW-shaped) input: (mean, var, mean |x|, mean x^2)."""
    x64 = rows(x).double()
    mean = x64.mean(0)
    return mean, (x64 - mean).square().mean(0), x64.abs().mean(0), x64.square().mean(0)


def check_bn_stats_e2e(x, mean, rstd, eps, tau_s, what=""):
    """The saved statistics against the exact statistics of ``x``, through the bound propagated from the reduction's
    ``tau_s`` (``bn_reduce_tau``):  d_mean <= tau_s mean|x| + u |mean|,
    d_var <= tau_s mean(x^2) + 2 |mean| d_mean + d_mean^2 + 3 u (mean(x^2) + mean^2),  rstd = rsqrt(var + eps) within
    the resulting interval (``1/2 d_var / (var + eps) + 2 u`` to first order).  The fp32 ``sum x^2 / M - mean^2`` loses
    accuracy as |mean| / std grows, and so does this bound.  Returns the ratios (mean, rstd)."""
    mu, var, a, q = bn_exact_stats(x)
    dmu = tau_s * a + EPS32 * mu.abs()
    dvar = tau_s * q + 2 * mu.abs() * dmu + dmu * dmu + 3 * EPS32 * (q + mu * mu)
    r1 = check_interval(mean, mu - dmu, mu + dmu, what=what + " mean vs exact")
    lo, hi = _rstd_interval(var, dvar, f32(eps))
    r2 = check_interval(rstd, lo, hi, what=what + " rstd vs exact")
    return r1, r2


def check_bn_running_e2e(x, rm0, rv0, rm, rv, momentum, tau_s, what=""):
    """The running statistics after ONE momentum update from ``(rm0, rv0)`` against the exact batch statistics of ``x``,
    through the bound of ``check_bn_stats_e2e`` (for a path whose per-channel sums cannot be read).  A second update (a
    recomputed forward that updates them again) or none at all fails.  Returns the ratios (mean, var)."""
    mu, var, a, q = bn_exact_stats(x)
    m = rows(x).shape[0]
    dmu = tau_s * a + EPS32 * mu.abs()
    dvar = tau_s * q + 2 * mu.abs() * dmu + dmu * dmu + 3 * EPS32 * (q + mu * mu)
    mom = f32(momentum)
    one_m = f32(1.0 - mom)
    ratio = m / (m - 1) if m > 1 else 1.0
    a0, b = one_m * rm0.double().to(mu.device), mom * mu
    slack = 3 * EPS32 * (a0.abs() + b.abs()) + mom * dmu
    r1 = check_interval(rm, a0 + b - slack, a0 + b + slack, what=what + " running mean vs exact")
    a0, b = one_m * rv0.double().to(mu.device), mom * ratio * var
    slack = 4 * EPS32 * (a0.abs() + b.abs()) + mom * ratio * dvar
    r2 = check_interval(rv, a0 + b - slack, a0 + b + slack, what=what + " running var vs exact")
    return r1, r2


def bn_y_ref(x, mean, rstd, gamma, beta, res=None, relu=False):
    """(ref, mag) of the BatchNorm apply from the saved statistics: ``relu(x g r + (b - m g r) + res)``; tau
    ``BN_Y_TAU``."""
    x64, m64 = rows(x).double(), mean.double()
    sc = gamma.double() * rstd.double()
    a, ms = x64 * sc, m64 * sc
    ref = a + (beta.double() - ms)
    mag = a.abs() + beta.double().abs() + ms.abs()
    if res is not None:
        ref, mag = ref + rows(res).double(), mag + rows(res).double().abs()
    return (ref.relu() if relu else ref), mag


def scale_shift_ref(x, scale, shift, res=None, relu=False):
    """(ref, mag) of ``scale_shift_act``: one fmaf, then the residual add (tau 2 EPS32)."""
    a = rows(x).double() * scale.double()
    ref, mag = a + shift.double(), a.abs() + shift.double().abs()
    if res is not None:
        ref, mag = ref + rows(res).double(), mag + rows(res).double().abs()
    return (ref.relu() if relu else ref), mag


def bn_dx_ref(d, x, mean, rstd, gamma, dsums, m, keep=None, dsums_err=None):
    """(ref, mag) of the BatchNorm input gradient from the kernel's own ``dsums``:
    ``g r (dy_m - db / M - xhat dg / M)`` with ``dy_m = d * keep`` (the ReLU mask of the STORED output; None: no ReLU or
    a gradient stored already masked); tau ``BN_DX_TAU``.  ``dsums_err``: when ``dsums`` is the float64 reference
    rather than the kernel's (which a caller cannot read), its error bound ``tau_s * mag`` from ``bn_dsums_ref``; the
    effect on dx, ``|g r| (e_db + |xhat| e_dg) / M``, is added to ``mag`` in units of ``BN_DX_TAU``."""
    c = mean.numel()
    g = rows(d).double()
    if keep is not None:
        g = g * keep
    xhat = (rows(x).double() - mean.double()) * rstd.double()
    k1, k2 = dsums[:c].double() / m, dsums[c:].double() / m
    sc = gamma.double() * rstd.double()
    mag = sc.abs() * (g.abs() + k1.abs() + (xhat * k2).abs())
    if dsums_err is not None:
        e = dsums_err.double().to(mag.device)
        mag = mag + sc.abs() * (e[:c] + xhat.abs() * e[c:]) / m / BN_DX_TAU
    return sc * (g - k1 - xhat * k2), mag


def bn_exact(x, gamma, beta, eps, res=None, relu=False, y=None, dy=None):
    """End-to-end float64 BatchNorm (+ residual) (+ ReLU) of the bf16 inputs with their exact batch statistics: a dict
    of (ref, mag) pairs ``y``, and with ``dy`` also ``dx``, ``dres``, ``dgamma``, ``dbeta``.  The ReLU mask of the
    backward is that of the STORED output ``y`` (the kernels' rule).  Equal to float64 ``F.batch_norm`` and its
    autograd (tests/test_bn_pool_bounds_cpu.py)."""
    x64 = rows(x).double()
    m = x64.shape[0]
    mu, var, _, _ = bn_exact_stats(x)
    rstd = torch.rsqrt(var + f32(eps))
    xhat = (x64 - mu) * rstd
    g64, b64 = gamma.double(), beta.double()
    yref = xhat * g64 + b64 + (rows(res).double() if res is not None else 0)
    out = {"y": (yref.relu() if relu else yref, bn_y_ref(x, mu, rstd, gamma, beta, res)[1])}
    if dy is not None:
        gm = rows(dy).double()
        if relu:
            gm = gm * (rows(y).double() > 0)
        db, dg = gm.sum(0), (gm * xhat).sum(0)
        sc = g64 * rstd
        out["dx"] = (sc * (gm - db / m - xhat * dg / m),
                     sc.abs() * (gm.abs() + (db / m).abs() + (xhat * dg / m).abs()))
        out["dres"] = (gm, gm.abs())
        out["dgamma"], out["dbeta"] = (dg, (gm * xhat).abs().sum(0)), (db, gm.abs().sum(0))
    return out


def maxpool_ref(x):
    """float64 3x3 / stride 2 / pad 1 max pool of the bf16 NCHW ``x`` and the flat (h W + w) index of the maximum.
    Torch takes the first maximum in (kh, kw) scan order and pads with -inf, which is the kernel's rule.  (NaN is out of
    scope: the kernel's ``>`` drops it, torch propagates it.)"""
    return F.max_pool2d(x.double(), 3, 2, 1, return_indices=True)


def check_exact(got, want, what=""):
    """Exact equality (outputs that involve no rounding: masked gradients, mask bits, parameter-gradient sinks, max-pool
    values and slots; +0 and -0 are equal, NaN is not); the message names the first differing element."""
    g, w = got.reshape(-1), want.to(got.device, got.dtype).reshape(-1)
    bad = g != w
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d of %d elements differ, first at flat index %d (%s): got %r, want %r" % (
            what, int(bad.sum()), bad.numel(), i, [int(t) for t in torch.unravel_index(torch.tensor(i), got.shape)],
            g[i].item(), w[i].item()))


def check_maxpool(y, slots, x, what=""):
    """Max-pool output [N, C, Ho, Wo] and the kernel's arg-max slots against ``maxpool_ref``: both exact.  Returns the
    flat indices of the maxima for the backward reference."""
    ref, idx = maxpool_ref(x)
    check_exact(y.double(), ref.to(y.device), what=what + " y")
    check_exact(slots.long(), maxpool_slots(idx, x.shape[3]).to(slots.device), what=what + " arg-max slot")
    return idx


def maxpool_slots(idx, w):
    """The kernel's window slot ``kh * 3 + kw`` of each flat maximum index [N, C, Ho, Wo]."""
    ho, wo = idx.shape[2], idx.shape[3]
    oh = torch.arange(ho, device=idx.device).view(1, 1, ho, 1)
    ow = torch.arange(wo, device=idx.device).view(1, 1, 1, wo)
    return (idx // w - (2 * oh - 1)) * 3 + (idx % w - (2 * ow - 1))


def maxpool_bwd_ref(dy, idx, x_shape):
    """(ref, mag) of the max-pool input gradient: ``dy`` routed to the maxima in float64.  A pixel is in at most 4
    windows: tau 3 EPS32."""
    n, c, h, w = x_shape
    flat = idx.reshape(n, c, -1)
    d64 = dy.double().reshape(n, c, -1)
    ref = torch.zeros(n, c, h * w, dtype=torch.float64, device=dy.device).scatter_add_(2, flat, d64)
    mag = torch.zeros_like(ref).scatter_add_(2, flat, d64.abs())
    return ref.view(n, c, h, w), mag.view(n, c, h, w)


def avgpool_ref(x):
    """(ref, mag) of the 2x2 / stride 2 average pool (ceil mode, exclusive): at most 4 terms and a power-of-two scale,
    tau 3 EPS32."""
    x64 = x.double()
    return tuple(F.avg_pool2d(t, 2, 2, 0, ceil_mode=True, count_include_pad=False) for t in (x64, x64.abs()))


def avgpool_bwd_ref(dy, x_shape):
    """(ref, mag) of its input gradient (each pixel in one window; the power-of-two scale is exact: tau EPS32)."""
    outs = []
    for d in (dy.double(), dy.double().abs()):
        z = torch.zeros(x_shape, dtype=torch.float64, device=dy.device, requires_grad=True)
        F.avg_pool2d(z, 2, 2, 0, ceil_mode=True, count_include_pad=False).backward(d)
        outs.append(z.grad)
    return tuple(outs)


def gap_tau(hw):
    """Global average pool forward: a chain of ceil(HW / 8) additions per thread, 8 partials, and ``fl(1 / HW)``
    (inexact for HW = 49) times the sum."""
    return (math.ceil(hw / 8) + 8 + 2) * EPS32


def gap_ref(x):
    """(ref, mag) [N, C] of the global average pool of NCHW-shaped ``x`` (tau ``gap_tau(H W)``)."""
    x64 = x.double()
    return x64.mean((2, 3)), x64.abs().mean((2, 3))


def gap_bwd_ref(dy, x_shape):
    """(ref, mag) of its input gradient ``dy / HW`` on every pixel: ``fl(1 / HW)`` and the product, tau 2 EPS32."""
    n, c, h, w = x_shape
    ref = (dy.double() / (h * w)).view(n, c, 1, 1).expand(n, c, h, w)
    return ref, ref.abs()


def dilate2_ref(x):
    """Zero insertion: out[:, :, 2 h, 2 w] = x[:, :, h, w], every other element 0 (exact)."""
    n, c, h, w = x.shape
    out = torch.zeros(n, c, 2 * h, 2 * w, dtype=x.dtype, device=x.device)
    out[:, :, ::2, ::2] = x
    return out


# ------------------------------------------------------------------------------------------------------ fp8 GEMMs
# The tensor core adds the e4m3 products of a 32-deep MMA with fewer significant bits than fp32 (about 14): 2^-12 of the
# magnitude per MMA.  The block-scaled GEMM promotes each 128-deep k-block (four MMAs) into an fp32 accumulator; the
# per-tensor GEMM keeps one accumulator in the MMA chain for all of K.
def fp8_tau(k):
    """Per-element slack factor (times the magnitude) of the block-scaled GEMM: the tensor core's k-block sums, one fp32
    promotion per k-block, the bias, the addend and the bf16 conversion's input."""
    return 2.0 ** -10 + (math.ceil(k / 128) + 3) * EPS32


def fp8_tensor_tau(k):
    """The same model for the per-tensor GEMM, with no per-k-block promotion: 2^-12 per 32-deep MMA over all of K, then
    the epilogue's fma and the bf16 conversion's input.  Derived, not fitted."""
    return math.ceil(k / 32) * 2.0 ** -12 + 3 * EPS32


def check_gelu_e4m3(q, sa, pre, mag, k, what=""):
    """The GELU -> e4m3 epilogue of the block-scaled GEMM (``fp8.gemm_fp8_gelu_e4m3``): e4m3 bytes ``q`` [M, N] and block
    scales ``sa`` [ceil(N / 128), M] against float64 ``pre``, the dequantised product plus bias, and its magnitude ``mag``.

    g = gelu(pre) in float64.  The kernel's g is within e_g = 1.13 fp8_tau(K) mag of it (GELU is 1.13-Lipschitz), plus
    half a bf16 ulp (it quantises the bf16 g).  Each dequantised element q s is then within
    e_g + 2^-4 (|g| + e_g) + 2^-10 s + 2^-22 (|g| + e_g) of g: half an e4m3 ulp (3 mantissa bits), half the subnormal
    step 2^-9 s, and the fp32 division by s.  Each block's scale is exactly 1 when its g are all 0, and otherwise
    448 s = its max|g| within the block's largest element bound.  Returns the worst element error / bound."""
    n = q.shape[1]
    e_g = 1.13 * fp8_tau(k) * mag
    g64 = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
    e_g = e_g + 0.5 * ulp(g64.abs() + e_g, 8)
    s = sa.t().repeat_interleave(128, 1)[:, :n].double()         # [M, N]: each element's block scale
    deq = q.view(torch.float8_e4m3fn).double() * s
    bound = e_g + 2.0 ** -4 * (g64.abs() + e_g) + 2.0 ** -10 * s + 2.0 ** -22 * (g64.abs() + e_g)
    err = (deq - g64).abs()
    ratio = float((err / bound).nan_to_num(float("inf")).max()) if err.numel() else 0.0
    _log(what, ratio, None)
    bad = ~(err <= bound)
    if bad.any():
        raise AssertionError("%s: %d elements out of bounds, first %s: q*s %r, g %r, bound %r, worst ratio %.3g" % (
            what, int(bad.sum()), bad.nonzero()[0].tolist(), float(deq[bad][0]), float(g64[bad][0]),
            float(bound[bad][0]), ratio))
    nb = sa.shape[0]
    pad = nb * 128 - n
    gmax = F.pad(g64.abs(), (0, pad)).view(-1, nb, 128).amax(2)
    emax = F.pad(bound, (0, pad)).view(-1, nb, 128).amax(2)
    s_blk = sa.t().double()
    zero = gmax == 0
    if not torch.equal(s_blk[zero], torch.ones_like(s_blk[zero])):
        raise AssertionError("%s: an all-zero block's scale is not 1" % what)
    off = ~((448 * s_blk - gmax).abs() <= emax) & ~zero
    if off.any():
        r, b = off.nonzero()[0].tolist()
        raise AssertionError("%s: %d block scales off, first row %d block %d: 448 s %r, max|g| %r" % (
            what, int(off.sum()), r, b, float(448 * s_blk[r, b]), float(gmax[r, b])))
    return ratio


def dequant_a(q, sa):
    """float64 [M, K] = e4m3(q) * sa[k // 128, m]"""
    k = q.shape[1]
    return q.view(torch.float8_e4m3fn).double() * sa.double().t().repeat_interleave(128, 1)[:, :k]


def dequant_w(q, sw):
    """float64 [N, K] = e4m3(q) * sw[n // 128, k // 128]"""
    n, k = q.shape
    return q.view(torch.float8_e4m3fn).double() * sw.double().repeat_interleave(128, 0)[:n].repeat_interleave(128, 1)[:, :k]


# ----------------------------------------------------------------------------------------------- guarded windows
class Guarded:
    """A tensor ``t`` placed as a window in a larger buffer whose other elements hold a sentinel."""

    def __init__(self, buf, t, fill):
        self.buf, self.t, self.fill = buf, t, fill
        self._in = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
        self._in.view(-1)[_window_index(buf, t)] = True
        self._bits = buf.clone()

    def write(self, values):
        self.t.copy_(values)
        self._bits = self.buf.clone()
        return self

    def assert_untouched(self, what=""):
        """Every element outside the window still holds the sentinel, bit for bit."""
        a, b = _bits(self.buf), _bits(self._bits)
        changed = (a != b) & ~self._in
        if changed.any():
            i = changed.view(-1).nonzero()[0].item()
            raise AssertionError("%s: %d sentinel elements overwritten outside the window, first at flat offset %d: %r" % (
                what, int(changed.sum()), i, float(self.buf.view(-1)[i])))


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 1: torch.uint8}[t.element_size()])


def _window_index(buf, t):
    """Flat indices (into ``buf``) of the elements of the view ``t``."""
    off = t.storage_offset() - buf.storage_offset()
    idx = torch.full(t.shape, off, dtype=torch.int64, device=buf.device)
    for d, (size, st) in enumerate(zip(t.shape, t.stride())):
        shp = [1] * t.dim()
        shp[d] = size
        idx = idx + (torch.arange(size, device=buf.device) * st).view(shp)
    return idx.reshape(-1)


def guarded(shape, pad_rows=0, pad_cols=0, fill=float("nan"), dtype=torch.bfloat16, device="cuda", values=None):
    """A ``shape`` tensor inside a sentinel-filled buffer.

    2-D [R, C]: ``pad_rows`` sentinel rows above and below, row pitch ``C + pad_cols`` (a padded pitch);
    1-D [n]: ``pad_rows`` sentinel elements on each side;
    4-D NCHW-shaped channels_last: ``pad_rows`` sentinel pixels (of C channels) before and after.
    ``values`` (optional) is copied into the window.  Keep ``pad_cols`` and ``pad_rows * C`` multiples of 8 for
    16-byte-aligned TMA operands."""
    if len(shape) == 2:
        r, c = shape
        buf = torch.full((r + 2 * pad_rows, c + pad_cols), fill, dtype=dtype, device=device)
        t = buf[pad_rows:pad_rows + r, :c]
    elif len(shape) == 1:
        buf = torch.full((shape[0] + 2 * pad_rows,), fill, dtype=dtype, device=device)
        t = buf[pad_rows:pad_rows + shape[0]]
    else:
        n, c, h, w = shape
        numel = n * c * h * w
        buf = torch.full((numel + 2 * pad_rows * c,), fill, dtype=dtype, device=device)
        t = buf[pad_rows * c:pad_rows * c + numel].view(n, h, w, c).permute(0, 3, 1, 2)
    g = Guarded(buf, t, fill)
    if values is not None:
        g.write(values)
    return g
