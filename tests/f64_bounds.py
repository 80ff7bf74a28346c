"""Float64 oracle for the bf16 GEMM and convolution kernels (csrc/gemm.cu, gemm_persist.cu, conv3x3.cu,
conv3x3_wgrad.cu, stem.cu): element-wise bounds instead of a global relative norm, which hides one wrong row, column,
tile or tail.

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


def _tile_counts(m, n, tile, dev):
    return _tile_sums(torch.ones(m, n, dtype=torch.float64, device=dev), tile)


def check_bf16(out, ref, mag, k, split=1, what="", tile=TILE, c2_factor=C2_FACTOR, terms=None):
    """Criteria 1 and 2 above on a bf16 kernel output against its float64 (ref, mag).  4-D NCHW-shaped tensors are
    checked as [pixels, channels]; KRSC weight gradients are passed as [Cout, 9 Cin].  Returns the worst ratios
    (criterion 1: worst error / bound; criterion 2: worst RMS error / yardstick, failing above ``c2_factor``).

    ``terms``: for a path that stores partial results as bf16 and then adds them (the pixel-pair weight gradient), the
    float64 (ref, mag) of each partial, with ``ref`` their sum.  Criterion 1 then also allows each partial its own half
    ulp (at ``|term| + slack``), and criterion 2's yardstick becomes the correct rounding of each stage:
    ``bf16(sum bf16(term))``."""
    o, r, g = rows(out).double(), rows(ref).double().to(out.device), rows(mag).double().to(out.device)
    assert o.shape == r.shape == g.shape, (what, o.shape, r.shape, g.shape)
    slack = tau(k, split) * g
    bound = 0.5 * ulp(r.abs() + slack, 8) + slack
    yard = bf16_round(r)
    if terms:
        tr = [rows(t).double().to(out.device) for t, _ in terms]
        tm = [rows(t).double().to(out.device) for _, t in terms]
        assert all(t.shape == r.shape for t in tr + tm), what
        for t, tg in zip(tr, tm):
            bound = bound + 0.5 * ulp(t.abs() + tau(k, split) * tg, 8)
        yard = bf16_round(sum(bf16_round(t) for t in tr))
    err = (o - r).abs()
    bad = ~(err <= bound)                                    # NaN fails
    c1 = float((err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max()) if o.numel() else 0.0
    m, n = o.shape
    e2 = (o - r).square().nan_to_num(float("inf"))
    y2 = (yard - r).square()
    g2 = g.square()
    msgs = []
    c2 = 0.0
    for name, esum, ysum, gsum, cnt in (
            ("tile", _tile_sums(e2, tile), _tile_sums(y2, tile), _tile_sums(g2, tile), _tile_counts(m, n, tile, o.device)),
            ("column", e2.sum(0), y2.sum(0), g2.sum(0), torch.full((n,), float(m), dtype=torch.float64, device=o.device))):
        rms_e, rms_y, rms_g = (esum / cnt).sqrt(), (ysum / cnt).sqrt(), (gsum / cnt).sqrt()
        allowed = c2_factor * rms_y + C2_MAG * rms_g
        ratio = rms_e / (allowed / c2_factor).clamp_min(1e-300)
        c2 = max(c2, float(ratio.max())) if ratio.numel() else c2
        over = ~(rms_e <= allowed)
        if over.any():
            worst = torch.argsort(ratio.flatten(), descending=True)[:4].tolist()
            if name == "tile":
                desc = ["(%d, %d): %.3g x yardstick" % (i // ratio.shape[1], i % ratio.shape[1], float(ratio.flatten()[i]))
                        for i in worst]
            else:
                desc = ["%d: %.3g x yardstick" % (i, float(ratio[i])) for i in worst]
            msgs.append("criterion 2: %d of %d %ss over %.2f x the RMS error of correct rounding, worst %s" % (
                int(over.sum()), over.numel(), name, c2_factor, ", ".join(desc)))
    _log(what, c1, c2)
    if bad.any():
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
