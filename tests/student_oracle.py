"""Float64 oracle of an ErnieStudent training step, layer by layer (the tests/step_oracle.py pattern for the Transformer
student, padded or packed, with or without dropout, gradients in ``.grad`` or in flat-bucket windows).

``StudentRecorder`` patches module attributes for one step and records every call the step makes, cloning inside the
wrappers: the GEMMs of ``ops.gemm`` (forward, the dctx / dx dgrads with their residual addend, the pooler and
classifier of ``_LinearFn``, the GELU and residual-dropout epilogues, ``_wgrad``), the attention forward / backward
pair of either layout with its saved ``lse``, ``_dropout_apply``, every dropout draw (``_draw``) in draw order, and the
LayerNorm / embedding-LayerNorm entry points of ``ops``, whose output and input gradients come from tensor hooks.  A
backward call is matched to its layer by the data pointers of the saved forward operands (the per-step bf16 weight
copies, qkv, u and the GEMM inputs).  Everything is undone on exit.

``check()`` judges every recorded call against float64 built from exactly the tensors that call read (teacher-forced,
so the per-kernel bounds hold inside the model without compounding), in three parts:

1. each kernel call, with the bounds the suite already uses: GEMMs, gelu_train's u, dgrads and weight gradients (with
   their split-K) by ``f64_bounds.check_bf16`` at ``tau(K)``; gelu_train's y bitwise the inference GELU epilogue;
   residual dropout and the GELU dgrad as tests/test_dropout_gpu.py and test_ernie_student_gpu.py (a dropped element
   stores the addend bit for bit); attention O by ``attention_ref`` at p = 0 and by 2^-8 |ref| + 2^-6 mag with Z;
   dQ / dK / dV by 2^-8 |ref| + 2^-6 mag; LayerNorm y by ``ln_ref``, dx by 2^-8 |ref| + 2^-16 mag, dgamma, dbeta and
   the three table gradients by 2^-12 sum |terms|; ``_dropout_apply`` bit for bit;
2. the saved ``lse`` (below);
3. wiring and coverage, bit for bit: each call's operand is its producer's output, every dropout site's Z is rebuilt
   with ``dropout_keep_reference`` at the documented index, order and offsets (4 per site), the backward uses the
   forward's draw, the last LayerNorm's output gradient is 0 outside the [CLS] rows, and every parameter's gradient is
   checked exactly once, in its bucket window or ``.grad`` (a non-sink weight's ``.grad`` is its recorded bf16 weight
   gradient cast to fp32; bias gradients within 2^-12 sum |terms| of float64 column sums); the logits gradient as
   ``step_oracle.check_logits_grad``.

A failure names the layer and the pass, e.g. ``layers.2.ffn dgrad dx`` or ``layers.0.attention backward (packed)``.
With ``EDL_F64_BOUNDS_LOG`` set, every check appends its worst error / bound ratio to that file.

lse bound.  The kernel stores lse = m + log2(l), l the row sum of p~_j = 2^(c s~_j - m) with c = log2(e) / 8, against
lse = log2 sum_j 2^(c s_j) over the valid keys.  The common m cancels, so lse~ - lse = log2(l~ / l), and l~ / l = 1 + r
with |r| <= eps + tau_acc: each p~_j is within eps_j <= eps of its exact value (the eps model of tests/test_ernie_gpu.py:
exponent error delta_j, ex2.approx, and the bf16 rounding of P if the sum is taken after it), and the fp32 accumulation
of l with its per-tile rescales adds tau_acc = (8 n_tiles + 32) 2^-23.  |log2(1 + r)| <= |r| / (ln 2 (1 - |r|)), and
with |r| < 2^-7 that is below 1.4427 * 1.008 |r| < 1.45 |r|.  The fp32 add m + log2f(l) and log2f itself add
2^-23 |lse|.  Hence
    |lse~ - lse| <= 1.45 (eps + tau_acc) + 2^-23 |lse|,
+inf exactly for a row without a valid key, and bitwise the p = 0 lse under dropout.

Worst ratios observed over tests/test_student_oracle_gpu.py's five recorded steps and the bucket step (one NVIDIA
H100 80GB HBM3, 700 W power limit), read from ``EDL_F64_BOUNDS_LOG`` (criterion 1 = worst error / bound; criterion 2
of ``check_bf16`` where it applies):

    GEMM forward (QKV, out, FFN1 u, FFN2, pooler, classifier)   c1 0.999   c2 1.00
    GEMM dgrad (dctx, dx with its addend, pooler, classifier)   c1 1.000   c2 1.00
    weight gradients (.grad and fp32 bucket windows)            c1 1.000   c2 1.00
    residual-dropout epilogue (kept elements)                   c1 0.992
    GELU dgrad                                                  c1 0.957
    attention O (p = 0 and with Z)                              c1 0.412
    lse (the first measurement of this bound)                   c1 0.482
    attention dQ / dK / dV                                      c1 0.400
    LayerNorm and embedding-LayerNorm y                         c1 0.992   c2 1.00
    LayerNorm dx                                                c1 0.354
    dgamma, dbeta, embedding-table gradients                    c1 0.002
    bias gradients                                              c1 0.001
    logits gradient                                             not measured (``check_logits_grad`` does not log)"""
import math

import torch

import f64_bounds as fb
import step_oracle as so
from edl_b200 import ops
from edl_b200.ops import gemm as G
from edl_b200.ops import transformer as T

EPS32 = fb.EPS32
LOG2E = math.log2(math.e)


# --------------------------------------------------------------------------------------------- float64 references
def attention_ref(qkv, mask, b, l, h, d=64):
    """(ref, slack) of the attention kernel's output [B * L, H * d] in float64 (see tests/test_ernie_gpu.py's docstring
    for the bound, written there for d = 64: the scores take d / 16 + 1 fp32 roundings and the exponent scale is
    c = log2(e) / sqrt(d), as in tests/test_attention_hd32_gpu.py)."""
    x = qkv.double().view(b, l, 3, h, d)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))                       # [B, H, L, d]
    s = q @ k.transpose(-1, -2)
    smag = q.abs() @ k.abs().transpose(-1, -2)
    keep = (torch.ones(b, l, dtype=torch.bool, device=qkv.device) if mask is None else mask != 0).view(b, 1, 1, l)
    rd = math.sqrt(d)
    c = LOG2E / rd
    cs = (s * c).masked_fill(~keep, float("-inf"))
    m = cs.amax(-1, keepdim=True)
    w = torch.softmax((s / rd).masked_fill(~keep, float("-inf")), -1).nan_to_num(0.0)   # 2^(c s) = e^(s / sqrt d)
    ref = w @ v
    wv = w @ v.abs()
    delta = c * (d / 16 + 1) * EPS32 * smag + EPS32 * (cs.abs() + (cs - m).abs())
    eps_j = 2.0 ** -8 + 2.0 ** -21 + 1.01 * math.log(2) * delta
    eps = eps_j.masked_fill(~keep, 0.0).amax(-1, keepdim=True)
    n_tiles = -(-l // 64)
    slack = (2 * eps / (1 - eps) + (8 * n_tiles + 32) * EPS32) * wv
    flat = lambda t: t.transpose(1, 2).reshape(b * l, h * d)                      # noqa: E731
    return flat(ref), flat(slack)


def lse_ref(qkv, mask, b, l, h):
    """(ref, bound) of the saved lse [B, H, L] in float64: log2 sum_j 2^(s_j log2(e) / 8) over the valid keys (+inf for a
    row without one) and 1.45 (eps + tau_acc) + 2^-23 |lse| (the module docstring)."""
    x = qkv.double().view(b, l, 3, h, 64)
    q, k = (x[:, :, i].transpose(1, 2) for i in range(2))
    s = q @ k.transpose(-1, -2)
    smag = q.abs() @ k.abs().transpose(-1, -2)
    keep = (torch.ones(b, l, dtype=torch.bool, device=qkv.device) if mask is None else mask != 0).view(b, 1, 1, l)
    c = LOG2E / 8
    cs = (s * c).masked_fill(~keep, float("-inf"))
    m = cs.amax(-1, keepdim=True)
    mf = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    tot = torch.exp2(cs - mf).sum(-1, keepdim=True)
    ref = torch.where(tot > 0, mf + torch.log2(tot.clamp_min(1e-300)), torch.full_like(tot, float("inf")))
    delta = c * 5 * EPS32 * smag + EPS32 * (cs.abs() + (cs - mf).abs())
    eps = (2.0 ** -8 + 2.0 ** -21 + 1.01 * math.log(2) * delta).masked_fill(~keep, 0.0).amax(-1, keepdim=True)
    tau_acc = (8 * -(-l // 64) + 32) * EPS32
    bound = 1.45 * (eps + tau_acc) + EPS32 * ref.abs().nan_to_num(0.0, posinf=0.0)
    return ref.squeeze(-1), bound.squeeze(-1)


def ln_ref(x64, gamma, beta, eps, dx=None):
    """(ref, slack) of LayerNorm's output in float64 (tests/test_ernie_gpu.py's docstring); ``dx``: the rounding of an
    fp32 input sum (embedding-LayerNorm)."""
    c = x64.shape[1]
    mean = x64.mean(1, keepdim=True)
    d = x64 - mean
    rstd = torch.rsqrt(d.square().mean(1, keepdim=True) + eps)
    g, b = gamma.double(), beta.double()
    ref = d * rstd * g + b
    dmu = c * EPS32 * x64.abs().mean(1, keepdim=True)
    eps_r = (c + 2) * EPS32 / 2 + 2.0 ** -21 + (dmu * rstd).square() / 2
    dxx = 0.0 if dx is None else dx
    dxm = 0.0 if dx is None else dx.mean(1, keepdim=True)
    slack = g.abs() * rstd * (dmu + dxm + dxx + d.abs() * eps_r) + 4 * EPS32 * (d.abs() * rstd * g.abs() + b.abs())
    return ref, slack


def attention_f64(qkv, mask, do, b, l, h, z=None):
    """O and dQ | dK | dV (float64) of attention with dropout Z [B, H, L, L] on the probabilities (None: no dropout),
    with the magnitudes of their rounding errors: (o, mo, dqkv, mag)."""
    x = qkv.double().view(b, l, 3, h, 64)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))
    dO = do.double().view(b, l, h, 64).transpose(1, 2)
    keep = (mask != 0).view(b, 1, 1, l)
    s = ((q @ k.transpose(-1, -2)) / 8).masked_fill(~keep, float("-inf"))
    mx = s.amax(-1, keepdim=True)
    e = torch.exp(s - torch.where(torch.isinf(mx), torch.zeros_like(mx), mx))
    den = e.sum(-1, keepdim=True)
    p = e / torch.where(den > 0, den, torch.ones_like(den))
    z = torch.ones_like(p) if z is None else z
    pz = p * z
    o = pz @ v
    mo = pz @ v.abs()
    dp = dO @ v.transpose(-1, -2)
    ds = p * (z * dp - (dO * o).sum(-1, keepdim=True))
    dq, dk, dv = ds @ k / 8, ds.transpose(-1, -2) @ q / 8, pz.transpose(-1, -2) @ dO
    mds = p * (z * (dO.abs() @ v.abs().transpose(-1, -2)) + (dO.abs() * o.abs()).sum(-1, keepdim=True))
    mq, mk, mv = mds @ k.abs() / 8, mds.transpose(-1, -2) @ q.abs() / 8, pz.transpose(-1, -2) @ dO.abs()

    def flat(t):
        return t.transpose(1, 2).reshape(b * l, h * 64)

    return (flat(o), flat(mo), torch.cat([flat(dq), flat(dk), flat(dv)], 1),
            torch.cat([flat(mq), flat(mk), flat(mv)], 1))


def ln_f64(x, dy, gamma, eps):
    """LayerNorm backward in float64: (xhat, dx, mag of dx, dgamma, its mag, dbeta, its mag)."""
    x, dy, g = x.double(), dy.double(), gamma.double()
    c = x.shape[1]
    mean = x.mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(1, keepdim=True) + eps)
    xh = (x - mean) * rstd
    gg = dy * g
    dx = rstd * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    mag = rstd * (gg.abs() + gg.abs().mean(1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(1, keepdim=True)) * c
    return xh, dx, mag, (dy * xh).sum(0), (dy * xh).abs().sum(0), dy.sum(0), dy.abs().sum(0)


# ---------------------------------------------------------------------------------------------------- the checks
def check_bound(out, ref, bound, what):
    """|out - ref| <= bound element-wise (NaN fails); returns the worst error / bound, logged as criterion 1."""
    o, r, bd = out.double(), ref.double().to(out.device), bound.double().to(out.device)
    err = (o - r).abs()
    ratio = float((err / bd.clamp_min(1e-300)).nan_to_num(float("inf")).max()) if o.numel() else 0.0
    fb._log(what, ratio, None)
    bad = ~(err <= bd)
    if bad.any():
        i = [int(v) for v in bad.nonzero()[0]]
        raise AssertionError("%s: %d of %d elements out of bounds, worst error / bound %.3g, first at %s: got %r, ref %r, "
                             "allowed +-%.3g" % (what, int(bad.sum()), bad.numel(), ratio, i, float(o[tuple(i)]),
                                                 float(r[tuple(i)]), float(bd[tuple(i)])))
    return ratio


def check_same(got, want, what):
    """Bitwise equality of a recorded operand with its producer's output (or of a gradient with its source)."""
    if tuple(got.shape) != tuple(want.shape) or got.dtype != want.dtype:
        raise AssertionError("%s: %s %s, expected %s %s" % (what, tuple(got.shape), got.dtype, tuple(want.shape),
                                                            want.dtype))
    fb.check_exact(got, want, what=what)


def check_gemm(out, a, b, what, b_mn_major=False, add=None, shift=None):
    """A forward or dgrad GEMM (``ops.gemm_bf16`` conventions) by ``check_bf16`` at tau(K)."""
    k = a.shape[1]
    ref, mag = fb.gemm_ref(a, b, b_mn_major=b_mn_major, add=add, shift=None if shift is None else shift.float())
    return so.check_bf16(out, ref, mag, k, what=what)


def check_wgrad(g, dy, x, split, what):
    """A weight gradient dW = dy^T x (bf16 values, any float dtype) by ``check_bf16`` at tau(M) with its split-K."""
    ref, mag = fb.gemm_ref(dy, x, a_mn_major=True, b_mn_major=True)
    return so.check_bf16(g.reshape(ref.shape), ref, mag, dy.shape[0], split, what=what)


def check_bias(got, dy, what):
    """A bias gradient within 2^-12 sum |terms| of the float64 column sums of ``dy``."""
    d = dy.double()
    return fb.check_sums(got.reshape(-1), d.sum(0), d.abs().sum(0), d.shape[0], what=what, tau_s=2.0 ** -12)


def site_z(draw, index):
    """float64 Z = keep * fp32(1 / (1 - p)) of a recorded draw (seed, offset, p) at the flat indices ``index``."""
    seed, off, p = draw
    scale = torch.tensor(1.0 / (1.0 - p), dtype=torch.float32).item()
    return T.dropout_keep_reference(seed, off, index, p).double() * scale


def rowwise_z(draw, rows, c, device):
    return None if draw is None else site_z(draw, torch.arange(rows * c, device=device)).view(rows, c)


def check_residual_dropout(out, a, b, shift, add, z, what):
    """D = add + Z o (a b^T + shift): kept elements within 2^-8 |ref| + 2^-16 mag, dropped ones the addend bitwise."""
    branch = a.double() @ b.double().t() + shift.double()
    ref = add.double() + z * branch
    mag = add.double().abs() + z * (a.double().abs() @ b.double().abs().t() + shift.double().abs())
    kept = z != 0
    check_same(out[~kept], add[~kept], what + " (dropped elements store the addend)")
    return check_bound(out[kept], ref[kept], (2.0 ** -8 * ref.abs() + 2.0 ** -16 * mag)[kept], what)


def check_gelu_grad(du, dy, w, u, what):
    ud = u.double()
    gp = 0.5 * (1 + torch.erf(ud / 2 ** 0.5)) + ud * torch.exp(-0.5 * ud * ud) / (2 * math.pi) ** 0.5
    ref = (dy.double() @ w.double()) * gp
    mag = (dy.double().abs() @ w.double().abs()) * (gp.abs() + 1)
    return check_bound(du, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -16 * mag, what)


def check_dropout_apply(y, x, draw, what):
    """``_dropout_apply``: y = bf16(fp32(x) * scale) where kept, 0 where dropped, bit for bit."""
    scale = torch.tensor(1.0 / (1.0 - draw[2]), dtype=torch.float32).item()
    keep = site_z(draw, torch.arange(x.numel(), device=x.device)).view(x.shape) != 0
    check_same(y, torch.where(keep, (x.float() * scale).to(x.dtype), torch.zeros_like(x)), what)


def segments(r):
    """(row slice, mask [b, l] uint8, b, l, sequence index) per attention problem of a recorded attention call: the
    whole batch in the padded layout, one sequence at a time in the packed one."""
    if r["layout"] == "padded":
        b, l = r["b"], r["l"]
        m = r["mask"] if r["mask"] is not None else torch.ones(b, l, dtype=torch.uint8, device=r["qkv"].device)
        yield slice(0, b * l), m, b, l, None
        return
    for i, (s, e) in enumerate(zip(r["cu"][:-1], r["cu"][1:])):
        km = r["key_mask"]
        m = (km[s:e] if km is not None else torch.ones(e - s, dtype=torch.uint8, device=r["qkv"].device)).view(1, -1)
        yield slice(s, e), m, 1, e - s, i


def attention_z(r, seq, b, l):
    """float64 Z [b, H, l, l] of a recorded attention call's probability site, or None at p = 0."""
    if r["drop"] is None:
        return None
    h, dev = r["heads"], r["qkv"].device
    hh = torch.arange(h, device=dev).view(1, -1, 1, 1)
    i = torch.arange(l, device=dev)
    if seq is None:                                   # padded: ((b H + h) L + i) L + j
        bb = torch.arange(b, device=dev).view(-1, 1, 1, 1)
        idx = (((bb * h + hh) * l + i.view(1, 1, -1, 1)) * l + i.view(1, 1, 1, -1))
    else:                                             # packed: ((b H + h) 512 + i) 512 + j
        idx = (((seq * h + hh) * 512 + i.view(1, 1, -1, 1)) * 512 + i.view(1, 1, 1, -1))
    return site_z(r["drop"], idx)


def _lse_rows(r, lse, rows, b, l):
    h = r["heads"]
    if r["layout"] == "padded":
        return lse
    return lse[:, rows].view(h, 1, l).transpose(0, 1)            # [H, T] -> [1, H, n]


def check_attention_forward(r, what):
    """O of a recorded attention call against float64 (attention_ref at p = 0, 2^-8 |ref| + 2^-6 mag with Z) and its
    lse (``lse_ref``).  Returns (ratio O, ratio lse)."""
    outs, refs, bounds, lo, lr, lb = [], [], [], [], [], []
    for rows, m, b, l, seq in segments(r):
        z = attention_z(r, seq, b, l)
        qkv = r["qkv"][rows]
        if z is None:
            ref, slack = attention_ref(qkv, m, b, l, r["heads"])
            bounds.append(0.5 * fb.ulp(ref.abs() + slack, 8) + slack)
        else:
            ref, mo, _, _ = attention_f64(qkv, m, torch.zeros(b * l, r["heads"] * 64, device=qkv.device), b, l,
                                          r["heads"], z)
            bounds.append(2.0 ** -8 * ref.abs() + 2.0 ** -6 * mo)
        outs.append(r["out"][rows])
        refs.append(ref)
        ref_l, bound_l = lse_ref(qkv, m, b, l, r["heads"])
        lo.append(_lse_rows(r, r["lse"], rows, b, l).reshape(-1))
        lr.append(ref_l.reshape(-1))
        lb.append(bound_l.reshape(-1))
    ratio = check_bound(torch.cat(outs), torch.cat(refs), torch.cat(bounds), what)
    got, ref, bound = torch.cat(lo), torch.cat(lr), torch.cat(lb)
    inf = torch.isinf(ref)
    if not torch.equal(torch.isinf(got) & (got > 0), inf):
        i = int((torch.isinf(got) != inf).nonzero()[0])
        raise AssertionError("%s lse: element %d is %r, expected %s" % (what, i, float(got[i]),
                                                                        "+inf (no valid key)" if inf[i] else "finite"))
    return ratio, check_bound(got[~inf], ref[~inf], bound[~inf], what + " lse")


def check_attention_backward(r, dqkv, dout, what):
    """dQ | dK | dV of a recorded attention call against float64: 2^-8 |ref| + 2^-6 mag, with Z."""
    refs, mags = [], []
    for rows, m, b, l, seq in segments(r):
        _, _, ref, mag = attention_f64(r["qkv"][rows], m, dout[rows], b, l, r["heads"], attention_z(r, seq, b, l))
        refs.append(ref)
        mags.append(mag)
    ref, mag = torch.cat(refs), torch.cat(mags)
    return check_bound(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, what)


def check_layernorm(x, gamma, beta, eps, y, what, z=None, terms=None):
    """LayerNorm y (embedding-LayerNorm with ``terms``, the float64 table rows, and ``z`` its dropout) against
    float64: ``ln_ref`` at p = 0, 2^-8 |ref| + 2^-16 mag under dropout."""
    x64 = sum(terms) if terms is not None else x.double()
    if z is None:
        dx = None if terms is None else 2 * EPS32 * sum(t.abs() for t in terms)
        return so.check_bf16(y, *ln_ref(x64, gamma, beta, eps, dx=dx), tau=1.0, what=what)
    xh = ln_f64(x64, torch.zeros_like(x64), gamma, eps)[0]
    ref = z * (xh * gamma.double() + beta.double())
    mag = z * (xh.abs() * gamma.double().abs() + beta.double().abs())
    return check_bound(y, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -16 * mag, what)


def check_layernorm_backward(x, dy, gamma, eps, dx, dg, db, what):
    _, rdx, mag, rg, mg, rb, mb = ln_f64(x, dy, gamma, eps)
    out = [check_bound(dg, rg, 2.0 ** -12 * mg, what + " dgamma"), check_bound(db, rb, 2.0 ** -12 * mb, what + " dbeta")]
    if dx is not None:
        out.append(check_bound(dx, rdx, 2.0 ** -8 * rdx.abs() + 2.0 ** -16 * mag, what + " dx"))
    return max(out)


def check_draw_order(draws, expected, what="dropout draws"):
    """The recorded draws ((seed, offset, p, site)) name the ``expected`` sites in order, from one seed, with offsets
    advancing by 4 per site."""
    sites = [d[3] for d in draws]
    if sites != list(expected):
        raise AssertionError("%s: sites drawn %s, expected %s" % (what, sites, list(expected)))
    for k, d in enumerate(draws):
        if d[0] != draws[0][0] or d[1] != draws[0][1] + 4 * k:
            raise AssertionError("%s: %s drew (seed %d, offset %d), expected (seed %d, offset %d)" % (
                what, d[3], d[0], d[1], draws[0][0], draws[0][1] + 4 * k))


def check_coverage(names, seen):
    """Every trainable parameter's gradient was checked exactly once: ``seen`` maps a name to its count."""
    for n in names:
        if seen.get(n, 0) != 1:
            raise AssertionError("%s: gradient checked %d times (every element exactly once expected)" % (
                n, seen.get(n, 0)))


# ------------------------------------------------------------------------------------------------------- recorder
def _c(t):
    return None if t is None else t.detach().clone()


class StudentRecorder:
    """Records one training step of ``model`` (an ErnieStudent on CUDA) between ``attach()`` and ``detach()`` (or as a
    context manager); ``check(labels)`` then judges it."""

    def __init__(self, model):
        self.model = model
        self.pname = {id(p): n for n, p in model.named_parameters()}
        self.params = dict(model.named_parameters())
        self._undo = []
        self.fwd, self.bwd, self.ln, self.draws, self.order = {}, {}, [], [], []
        self.emb = None
        self.cur, self.count = None, {}
        self.aptr, self.wptr, self.qptr, self.dropname = {}, {}, {}, {}
        self.orig = {}

    # -------------------------------------------------------------------------------------------------- capture
    def _patch(self, obj, attr, new):
        old = getattr(obj, attr)
        setattr(obj, attr, new)
        self._undo.append(lambda: setattr(obj, attr, old))
        self.orig[attr] = old
        return old

    def _draw_of(self, drop, site=None):
        if drop is None:
            return None
        d = self.draws[self.dropname[id(drop)]]
        if site is not None:
            d[3] = site
        return tuple(d[:3])

    def _role(self):
        k = self.count.get(self.cur, 0)
        self.count[self.cur] = k + 1
        return k

    def _ctx(self, attr, name_of):
        rec = self
        orig = self._patch(ops, attr, None)

        def wrapped(*args, **kw):
            prev, rec.cur = rec.cur, name_of(args)
            try:
                return orig(*args, **kw)
            finally:
                rec.cur = prev
        setattr(ops, attr, wrapped)

    def attach(self):
        rec = self
        layer_of = lambda p: self.pname[id(p)].rsplit(".", 1)[0]           # noqa: E731
        self._ctx("attention_block", lambda a: layer_of(a[1]) + ".attention")
        self._ctx("attention_block_varlen", lambda a: layer_of(a[1]) + ".attention")
        self._ctx("gelu_ffn", lambda a: layer_of(a[1]) + ".ffn")
        self._ctx("dropout", lambda a: "pooled")
        lin = self._patch(ops, "linear_bf16", None)

        def linear(x, w, bias=None, **kw):
            prev, rec.cur = rec.cur, ("pooler" if self.pname.get(id(bias)) == "pool_b" else "classifier")
            try:
                return lin(x, w, bias, **kw)
            finally:
                rec.cur = prev
        ops.linear_bf16 = linear

        draw = self._patch(T, "_draw", None)

        def _draw(device, p):
            d = draw(device, p)
            rec.dropname[id(d)] = len(rec.draws)
            rec.draws.append([int(d.seed), int(d.offset), float(p), None, d])
            return d
        T._draw = _draw

        gemm = self._patch(G, "gemm_bf16", None)

        def gemm_bf16(a, b, *args, **kw):
            d = gemm(a, b, *args, **kw)
            if kw.get("gelu"):
                return d
            assert not args, "the oracle expects keyword arguments"
            if rec.cur is not None:
                name = rec.cur
                if name.endswith(".attention"):
                    role = ("qkv", "out")[rec._role()]
                elif name.endswith(".ffn"):
                    role = "ffn2"
                else:
                    role = "fc"
                rec._fwd(name, role, a, b, d, kw.get("col_shift"), kw.get("add"), None)
            else:
                name, role = rec.wptr[b.data_ptr()]
                pas = {"qkv": "dgrad dx", "out": "dgrad dctx", "ffn1": "dgrad dx", "fc": "dgrad"}[role]
                rec._bwd(name, pas, a=_c(a), b=_c(b), add=_c(kw.get("add")), out=_c(d))
            return d
        G.gemm_bf16 = gemm_bf16

        rd = self._patch(G, "gemm_bf16_residual_dropout", None)

        def residual_dropout(x, w, bias, add, drop):
            d = rd(x, w, bias, add, drop)
            role = ("qkv", "out")[rec._role()] if rec.cur.endswith(".attention") else "ffn2"
            rec._fwd(rec.cur, role, x, w, d, bias, add, rec._draw_of(drop, rec.cur + " branch"))
            return d
        G.gemm_bf16_residual_dropout = residual_dropout

        gt = self._patch(G, "gemm_bf16_gelu_train", None)

        def gelu_train(x, w, bias=None):
            y, u = gt(x, w, bias)
            rec._fwd(rec.cur, "ffn1", x, w, u, bias, None, None, y=_c(y))
            return y, u
        G.gemm_bf16_gelu_train = gelu_train

        gg = self._patch(G, "gemm_bf16_gelu_grad", None)

        def gelu_grad(dy, w, u):
            du = gg(dy, w, u)
            name, _ = rec.wptr[w.data_ptr()]
            rec._bwd(name, "gelu dgrad", a=_c(dy), b=_c(w), u=_c(u), out=_c(du))
            return du
        G.gemm_bf16_gelu_grad = gelu_grad

        wg = self._patch(G, "_wgrad", None)

        def _wgrad(dy2, x2, weight_shape, sink, ready):
            g = wg(dy2, x2, weight_shape, sink, ready)
            name, role = rec.aptr[x2.data_ptr()]
            rec._bwd(name, role + " wgrad", dy=_c(dy2), x=_c(x2), out=_c(g), sink=sink is not None,
                     split=G._split_k_for(dy2.shape[1], x2.shape[1], dy2.shape[0]))
            return g
        G._wgrad = _wgrad

        af = self._patch(T, "attention_forward_saved", None)

        def attention_forward_saved(qkv, mask, batch, seq_len, heads, drop=None):
            out, lse = af(qkv, mask, batch, seq_len, heads, drop)
            rec._attn(dict(layout="padded", mask=_c(mask), b=batch, l=seq_len), qkv, heads, drop, out, lse)
            return out, lse
        T.attention_forward_saved = attention_forward_saved

        avf = self._patch(T, "attention_varlen_forward_saved", None)

        def attention_varlen_forward_saved(qkv, cu_seqlens, max_len, heads, key_mask=None, drop=None):
            out, lse = avf(qkv, cu_seqlens, max_len, heads, key_mask, drop)
            rec._attn(dict(layout="packed", cu=[int(v) for v in cu_seqlens.tolist()], cu_t=_c(cu_seqlens),
                           max_len=int(max_len), key_mask=_c(key_mask)), qkv, heads, drop, out, lse)
            return out, lse
        T.attention_varlen_forward_saved = attention_varlen_forward_saved

        ab = self._patch(T, "attention_backward", None)

        def attention_backward(qkv, mask, out, lse, dout, batch, seq_len, heads, drop=None):
            d = ab(qkv, mask, out, lse, dout, batch, seq_len, heads, drop)
            rec._attn_bwd(qkv, out, lse, dout, drop, d, "")
            return d
        T.attention_backward = attention_backward

        avb = self._patch(T, "attention_varlen_backward", None)

        def attention_varlen_backward(qkv, cu_seqlens, max_len, heads, key_mask, out, lse, dout, drop=None):
            d = avb(qkv, cu_seqlens, max_len, heads, key_mask, out, lse, dout, drop)
            rec._attn_bwd(qkv, out, lse, dout, drop, d, " (packed)")
            return d
        T.attention_varlen_backward = attention_varlen_backward

        da = self._patch(T, "_dropout_apply", None)

        def _dropout_apply(x, drop):
            y = da(x, drop)
            if rec.cur == "pooled":
                rec.fwd[("pooled", "dropout")] = dict(x=_c(x), y=_c(y), draw=rec._draw_of(drop, "pooled"), yt=y)
            else:
                site = rec.draws[rec.dropname[id(drop)]][3]
                rec._bwd(site, "dropout backward", x=_c(x), out=_c(y), draw=rec._draw_of(drop))
            return y
        T._dropout_apply = _dropout_apply

        ln = self._patch(ops, "layer_norm_trainable", None)

        def layer_norm_trainable(x, gamma, beta, eps=1e-12):
            y = ln(x, gamma, beta, eps)
            r = dict(name=self.pname[id(gamma)].rsplit("_", 1)[0], x=_c(x), gamma=_c(gamma), beta=_c(beta), eps=eps,
                     y=_c(y), gp=gamma, bp=beta, dy=None, dx=None, yptr=y.data_ptr())
            y.register_hook(lambda g: r.__setitem__("dy", _c(g)))
            if x.requires_grad:
                x.register_hook(lambda g: r.__setitem__("dx", _c(g)))
            rec.ln.append(r)
            return y
        ops.layer_norm_trainable = layer_norm_trainable

        el = self._patch(ops, "embedding_layernorm_trainable", None)

        def embedding_layernorm_trainable(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps=1e-12,
                                          dropout_p=0.0):
            n0 = len(rec.draws)
            prev, rec.cur = rec.cur, "embeddings"
            try:
                y = el(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps, dropout_p=dropout_p)
            finally:
                rec.cur = prev
            drop = None
            if len(rec.draws) > n0:
                rec.draws[n0][3] = "embeddings"
                drop = tuple(rec.draws[n0][:3])
            r = dict(ids=_c(ids).reshape(-1), pos_ids=_c(pos_ids).reshape(-1), seg_ids=_c(seg_ids).reshape(-1),
                     tabs=[t.detach().to(torch.bfloat16) for t in (word, pos, seg)], gamma=_c(gamma), beta=_c(beta),
                     eps=eps, y=_c(y), drop=drop, dy=None)
            y.register_hook(lambda g: r.__setitem__("dy", _c(g)))
            rec.emb = r
            return y
        ops.embedding_layernorm_trainable = embedding_layernorm_trainable
        return self

    def detach(self):
        for f in reversed(self._undo):
            f()
        self._undo = []

    def __enter__(self):
        return self.attach()

    def __exit__(self, *exc):
        self.detach()

    def _fwd(self, name, role, a, b, out, shift, add, draw, **extra):
        r = dict(a=_c(a), b=_c(b), out=_c(out), shift=_c(shift), add=_c(add), draw=draw, **extra)
        self.fwd[(name, role)] = r
        self.aptr[a.data_ptr()] = (name, role)
        self.wptr[b.data_ptr()] = (name, role)

    def _bwd(self, name, pas, **r):
        if (name, pas) in self.bwd:
            raise AssertionError("%s %s: recorded twice in one step" % (name, pas))
        self.bwd[(name, pas)] = r
        self.order.append((name, pas))

    def _attn(self, r, qkv, heads, drop, out, lse):
        name = self.cur
        r.update(qkv=_c(qkv), heads=heads, drop=self._draw_of(drop, None if drop is None else name + " probabilities"),
                 out=_c(out), lse=_c(lse))
        self.fwd[(name, "attention")] = r
        self.qptr[qkv.data_ptr()] = name

    def _attn_bwd(self, qkv, out, lse, dout, drop, d, tag):
        name = self.qptr[qkv.data_ptr()]
        self._bwd(name, "attention backward" + tag, qkv=_c(qkv), o=_c(out), lse=_c(lse), dout=_c(dout),
                  draw=self._draw_of(drop), out=_c(d))

    # ----------------------------------------------------------------------------------------------------- checks
    def _ratio(self, kind, r):
        c1, c2 = r if isinstance(r, tuple) else (r, None)
        w = self.ratios.setdefault(kind, [0.0, 0.0])
        w[0] = max(w[0], c1 or 0.0)
        w[1] = max(w[1], c2 or 0.0)

    def _grad_of(self, name):
        """The gradient of parameter ``name``: its bucket window or ``.grad``; counted for the coverage check."""
        p = self.params[name]
        self._seen[name] = self._seen.get(name, 0) + 1
        sink = getattr(p, "_edl_grad_sink", None)
        if sink is not None:
            torch.cuda.synchronize()
            return sink.view(p.shape), "(bucket)", True
        if p.grad is None:
            raise AssertionError("%s: no gradient (neither a bucket window nor .grad)" % name)
        return p.grad, "(grad)", False

    def _b(self, name, pas):
        r = self.bwd.get((name, pas))
        if r is None:
            raise AssertionError("%s %s: never ran in the backward" % (name, pas))
        return r

    def _weight(self, pname, rec_w, what):
        """A weight's gradient: numerically against the recorded wgrad operands, and (outside a bucket) bitwise the
        recorded bf16 result in the parameter's dtype."""
        g, where, _ = self._grad_of(pname)
        rows = g.shape[0]
        self._ratio("weight gradients", check_wgrad(g, rec_w["dy"][:, :rows] if rec_w["dy"].shape[1] != rows
                                                    else rec_w["dy"], rec_w["x"], rec_w["split"],
                                                    "%s %s" % (what, where)))
        if rec_w["out"] is not None:                 # returned to autograd: .grad is that bf16 result, cast
            check_same(g, rec_w["out"].reshape(-1, g.shape[1])[:rows].to(g.dtype), "%s %s" % (what, where))

    def _bias(self, pname, dy, what):
        g, where, _ = self._grad_of(pname)
        self._ratio("bias gradients", check_bias(g, dy[:, :g.numel()], "%s %s" % (what, where)))

    def check(self, labels):
        """Every check; raises AssertionError naming the layer and the pass.  ``labels``: the class indices of the
        step's mean cross-entropy loss.  Returns ``{kind: [c1, c2]}``, the worst ratios."""
        self._seen, self.ratios = {}, {}
        m = self.model
        nl = len(m.layers)
        # 1 + 2: every kernel call
        self._check_embeddings()
        for i in range(nl):
            self._check_attention_block("layers.%d" % i)
            self._check_ffn("layers.%d" % i)
        for r in self.ln:
            self._check_ln(r)
        self._check_head(labels)
        # 3: wiring and coverage
        self._check_wiring(nl)
        expect = ["embeddings"]
        for i in range(nl):
            expect += ["layers.%d.attention probabilities" % i, "layers.%d.attention branch" % i,
                       "layers.%d.ffn branch" % i]
        expect.append("pooled")
        drawn = [tuple(d[:4]) for d in self.draws]
        if drawn:
            check_draw_order(drawn, expect)
        check_coverage([n for n, p in m.named_parameters() if p.requires_grad], self._seen)
        return self.ratios

    def _check_embeddings(self):
        r = self.emb
        ids, pid, sid = r["ids"], r["pos_ids"], r["seg_ids"]
        terms = [r["tabs"][0].double()[ids], r["tabs"][1].double()[pid], r["tabs"][2].double()[sid]]
        rows, c = ids.numel(), r["y"].shape[1]
        z = rowwise_z(r["drop"], rows, c, ids.device)
        self._ratio("LayerNorm y", check_layernorm(None, r["gamma"], r["beta"], r["eps"], r["y"], "embeddings forward",
                                                   z=z, terms=terms))
        dy = r["dy"].double() if z is None else r["dy"].double() * z
        _, dE, mag, rg, mg, rb, mb = ln_f64(sum(terms), dy, r["gamma"], r["eps"])
        for n, idx, tab in (("word_emb", ids, r["tabs"][0]), ("pos_emb", pid, r["tabs"][1]),
                            ("seg_emb", sid, r["tabs"][2])):
            g, where, _ = self._grad_of(n)
            ref = torch.zeros(tab.shape, device=g.device, dtype=torch.float64).index_add_(0, idx, dE)
            mm = torch.zeros(tab.shape, device=g.device, dtype=torch.float64).index_add_(0, idx, mag + dE.abs())
            self._ratio("LayerNorm backward", check_bound(g, ref, 2.0 ** -12 * mm,
                                                          "embeddings backward %s %s" % (n, where)))
        for n, ref, mg_ in (("emb_ln_g", rg, mg), ("emb_ln_b", rb, mb)):
            g, where, _ = self._grad_of(n)
            self._ratio("LayerNorm backward", check_bound(g, ref, 2.0 ** -12 * mg_,
                                                          "embeddings backward %s %s" % (n, where)))

    def _check_attention_block(self, layer):
        name = layer + ".attention"
        q, a, o = self.fwd[(name, "qkv")], self.fwd[(name, "attention")], self.fwd[(name, "out")]
        packed = a["layout"] == "packed"
        tag = " (packed)" if packed else ""
        self._ratio("GEMM forward", check_gemm(q["out"], q["a"], q["b"], name + " qkv forward", shift=q["shift"]))
        ro, rl = check_attention_forward(a, name + " forward" + tag)
        self._ratio("attention O", ro)
        self._ratio("lse", rl)
        if a["drop"] is not None:
            again = (self.orig["attention_varlen_forward_saved"](a["qkv"], a["cu_t"], a["max_len"], a["heads"],
                                                                 a["key_mask"], None) if packed else
                     self.orig["attention_forward_saved"](a["qkv"], a["mask"], a["b"], a["l"], a["heads"], None))
            check_same(a["lse"], again[1], name + " forward" + tag + " lse (p > 0 against p = 0)")
        self._check_out_gemm(o, name + " out forward")
        # backward
        bo = self._b(name, "dgrad dctx")
        self._ratio("GEMM dgrad", check_gemm(bo["out"], bo["a"], bo["b"], name + " dgrad dctx", b_mn_major=True))
        ba = self._b(name, "attention backward" + tag)
        self._ratio("attention dQ / dK / dV", check_attention_backward(a, ba["out"], ba["dout"],
                                                                       name + " backward" + tag))
        bx = self._b(name, "dgrad dx")
        self._ratio("GEMM dgrad", check_gemm(bx["out"], bx["a"], bx["b"], name + " dgrad dx", b_mn_major=True,
                                             add=bx["add"]))
        if o["draw"] is not None:
            bd = self._b(name + " branch", "dropout backward")
            check_dropout_apply(bd["out"], bd["x"], bd["draw"], name + " branch dropout backward")
        self._weight(layer + ".qkv_w", self._b(name, "qkv wgrad"), name + " qkv wgrad")
        self._bias(layer + ".qkv_b", ba["out"], name + " qkv bias gradient")
        self._weight(layer + ".out_w", self._b(name, "out wgrad"), name + " out wgrad")
        self._bias(layer + ".out_b", bo["a"], name + " out bias gradient")

    def _check_out_gemm(self, r, what):
        if r["draw"] is None:
            self._ratio("GEMM forward", check_gemm(r["out"], r["a"], r["b"], what, add=r["add"], shift=r["shift"]))
        else:
            z = rowwise_z(r["draw"], r["out"].shape[0], r["out"].shape[1], r["out"].device)
            self._ratio("residual dropout", check_residual_dropout(r["out"], r["a"], r["b"], r["shift"], r["add"], z,
                                                                   what + " (dropout)"))

    def _check_ffn(self, layer):
        name = layer + ".ffn"
        f1, f2 = self.fwd[(name, "ffn1")], self.fwd[(name, "ffn2")]
        self._ratio("GEMM forward", check_gemm(f1["out"], f1["a"], f1["b"], name + " ffn1 forward u",
                                               shift=f1["shift"]))
        y = self.orig["gemm_bf16"](f1["a"], f1["b"], col_shift=f1["shift"].float(), gelu=True)
        check_same(f1["y"], y, name + " ffn1 forward y (the inference GELU epilogue)")
        self._check_out_gemm(f2, name + " ffn2 forward")
        bg = self._b(name, "gelu dgrad")
        self._ratio("GELU dgrad", check_gelu_grad(bg["out"], bg["a"], bg["b"], bg["u"], name + " gelu dgrad"))
        bx = self._b(name, "dgrad dx")
        self._ratio("GEMM dgrad", check_gemm(bx["out"], bx["a"], bx["b"], name + " dgrad dx", b_mn_major=True,
                                             add=bx["add"]))
        if f2["draw"] is not None:
            bd = self._b(name + " branch", "dropout backward")
            check_dropout_apply(bd["out"], bd["x"], bd["draw"], name + " branch dropout backward")
        self._weight(layer + ".ffn1_w", self._b(name, "ffn1 wgrad"), name + " ffn1 wgrad")
        self._bias(layer + ".ffn1_b", bg["out"], name + " ffn1 bias gradient")
        self._weight(layer + ".ffn2_w", self._b(name, "ffn2 wgrad"), name + " ffn2 wgrad")
        self._bias(layer + ".ffn2_b", bg["a"], name + " ffn2 bias gradient")

    def _check_ln(self, r):
        name = r["name"]
        self._ratio("LayerNorm y", check_layernorm(r["x"], r["gamma"], r["beta"], r["eps"], r["y"], name + " forward"))
        if r["dy"] is None:
            raise AssertionError("%s: its output gradient was never produced" % name)
        dg, where, _ = self._grad_of(name + "_g")
        db, _, _ = self._grad_of(name + "_b")
        self._ratio("LayerNorm backward", check_layernorm_backward(r["x"], r["dy"], r["gamma"], r["eps"], r["dx"], dg,
                                                                   db, "%s backward %s" % (name, where)))

    def _check_head(self, labels):
        p, c = self.fwd[("pooler", "fc")], self.fwd[("classifier", "fc")]
        self._ratio("GEMM forward", check_gemm(p["out"], p["a"], p["b"], "pooler forward", shift=p["shift"]))
        self._ratio("GEMM forward", check_gemm(c["out"], c["a"], c["b"], "classifier forward", shift=c["shift"]))
        n = self.model.num_labels
        bc = self._b("classifier", "dgrad")
        z = c["out"][:, :n].float()
        dz = bc["a"][:, :n]
        self._ratio("logits gradient", so.check_logits_grad(dz, so.ref_soft_ce_grad(z, labels.to(z.device), "labels"),
                                                            "classifier backward (logits gradient)"))
        check_same(bc["a"][:, n:], torch.zeros_like(bc["a"][:, n:]), "classifier backward (padded logit columns)")
        self._ratio("GEMM dgrad", check_gemm(bc["out"], bc["a"], bc["b"], "classifier dgrad", b_mn_major=True))
        self._weight("cls_w", self._b("classifier", "fc wgrad"), "classifier wgrad")
        self._bias("cls_b", bc["a"], "classifier bias gradient")
        pd = self.fwd.get(("pooled", "dropout"))
        if pd is not None:
            check_dropout_apply(pd["y"], pd["x"], pd["draw"], "pooled dropout forward")
            check_same(pd["y"], c["a"], "classifier forward input (the pooled dropout's output)")
            bd = self._b("pooled", "dropout backward")
            check_dropout_apply(bd["out"], bd["x"], bd["draw"], "pooled dropout backward")
            check_same(bd["x"], bc["out"], "pooled dropout backward input (the classifier dgrad)")
        bp = self._b("pooler", "dgrad")
        self._ratio("GEMM dgrad", check_gemm(bp["out"], bp["a"], bp["b"], "pooler dgrad", b_mn_major=True))
        self._weight("pool_w", self._b("pooler", "fc wgrad"), "pooler wgrad")
        self._bias("pool_b", bp["a"], "pooler bias gradient")

    def _check_wiring(self, nl):
        """The bitwise links between producers and consumers, forward and backward."""
        ln = {r["name"]: r for r in self.ln}
        x = self.emb["y"]
        dx_prev = ("embeddings", self.emb)
        for i in range(nl):
            layer = "layers.%d" % i
            an, fn = layer + ".attention", layer + ".ffn"
            q, a, o = self.fwd[(an, "qkv")], self.fwd[(an, "attention")], self.fwd[(an, "out")]
            l1, l2 = ln[layer + ".ln1"], ln[layer + ".ln2"]
            f1, f2 = self.fwd[(fn, "ffn1")], self.fwd[(fn, "ffn2")]
            check_same(q["a"], x, an + " qkv forward input (the previous LayerNorm's output)")
            check_same(a["qkv"], q["out"], an + " forward qkv (the QKV GEMM's output)")
            check_same(o["a"], a["out"], an + " out forward input (the attention output)")
            check_same(o["add"], x, an + " out forward addend (the block input)")
            check_same(l1["x"], o["out"], layer + ".ln1 forward input")
            check_same(f1["a"], l1["y"], fn + " ffn1 forward input")
            check_same(f2["a"], f1["y"], fn + " ffn2 forward input (gelu y)")
            check_same(f2["add"], l1["y"], fn + " ffn2 forward addend (the block input)")
            check_same(l2["x"], f2["out"], layer + ".ln2 forward input")
            # backward of the attention block
            bo, ba, bx = self._b(an, "dgrad dctx"), self._b(an, "attention backward" + (
                " (packed)" if a["layout"] == "packed" else "")), self._b(an, "dgrad dx")
            check_same(bx["add"], l1["dx"], an + " dgrad dx addend (grad h, the LayerNorm's dx)")
            if o["draw"] is None:
                check_same(bo["a"], bx["add"], an + " dgrad dctx input (dh)")
            else:
                bd = self._b(an + " branch", "dropout backward")
                check_same(bd["x"], bx["add"], an + " branch dropout backward input (dh)")
                check_same(bo["a"], bd["out"], an + " dgrad dctx input (Z o dh)")
            check_same(ba["dout"], bo["out"], an + " backward dout (dctx)")
            for k in ("qkv", "lse"):
                check_same(ba[k], a[k], an + " backward " + k + " (the forward's)")
            check_same(ba["o"], a["out"], an + " backward out (the forward's)")
            if ba["draw"] != a["drop"]:
                raise AssertionError("%s backward: draw %s, forward drew %s" % (an, ba["draw"], a["drop"]))
            check_same(bx["a"], ba["out"], an + " dgrad dx input (dqkv)")
            wq, wo = self._b(an, "qkv wgrad"), self._b(an, "out wgrad")
            check_same(wq["dy"], ba["out"], an + " qkv wgrad dy (dqkv)")
            check_same(wq["x"], q["a"], an + " qkv wgrad x (the block input)")
            check_same(wo["dy"], bo["a"], an + " out wgrad dy")
            check_same(wo["x"], a["out"], an + " out wgrad x (the attention output)")
            self._link_dx(dx_prev, bx["out"], an + " dgrad dx")
            # backward of the FFN block
            bg, fx = self._b(fn, "gelu dgrad"), self._b(fn, "dgrad dx")
            check_same(fx["add"], l2["dx"], fn + " dgrad dx addend (grad h, the LayerNorm's dx)")
            if f2["draw"] is None:
                check_same(bg["a"], fx["add"], fn + " gelu dgrad input (dh)")
            else:
                bd = self._b(fn + " branch", "dropout backward")
                check_same(bd["x"], fx["add"], fn + " branch dropout backward input (dh)")
                check_same(bg["a"], bd["out"], fn + " gelu dgrad input (Z o dh)")
            check_same(bg["u"], f1["out"], fn + " gelu dgrad u (the forward's)")
            check_same(fx["a"], bg["out"], fn + " dgrad dx input (dU)")
            w1, w2 = self._b(fn, "ffn1 wgrad"), self._b(fn, "ffn2 wgrad")
            check_same(w1["dy"], bg["out"], fn + " ffn1 wgrad dy (dU)")
            check_same(w1["x"], f1["a"], fn + " ffn1 wgrad x")
            check_same(w2["dy"], bg["a"], fn + " ffn2 wgrad dy")
            check_same(w2["x"], f1["y"], fn + " ffn2 wgrad x (gelu y)")
            self._link_dx(("ln1", l1), fx["out"], fn + " dgrad dx")
            x, dx_prev = l2["y"], ("ln2", l2)
        # the head: the last LayerNorm's output gradient is the pooler's dgrad on the [CLS] rows and 0 elsewhere
        last = dx_prev[1]
        bp = self._b("pooler", "dgrad")
        a = self.fwd[(("layers.0.attention"), "attention")]
        if a["layout"] == "padded":
            b, l = a["b"], a["l"]
            cls = torch.arange(b, device=x.device) * l
        else:
            cls = torch.tensor(a["cu"][:-1], device=x.device, dtype=torch.long)
        check_same(self.fwd[("pooler", "fc")]["a"], x.index_select(0, cls), "pooler forward input (the [CLS] rows)")
        dy = last["dy"]
        rest = torch.ones(dy.shape[0], dtype=torch.bool, device=dy.device)
        rest[cls] = False
        check_same(dy[rest], torch.zeros_like(dy[rest]), "%s output gradient outside the [CLS] rows" % last["name"])
        check_same(dy.index_select(0, cls), bp["out"], "%s output gradient on the [CLS] rows (pooler dgrad)"
                   % last["name"])
        wp, wc = self._b("pooler", "fc wgrad"), self._b("classifier", "fc wgrad")
        check_same(wp["dy"], bp["a"], "pooler wgrad dy")
        check_same(wp["x"], self.fwd[("pooler", "fc")]["a"], "pooler wgrad x")
        check_same(wc["dy"], self._b("classifier", "dgrad")["a"], "classifier wgrad dy")
        check_same(wc["x"], self.fwd[("classifier", "fc")]["a"], "classifier wgrad x")

    def _link_dx(self, prev, dx, what):
        """A block's dx is the output gradient of the LayerNorm (or embedding-LayerNorm) that produced its input."""
        kind, r = prev
        name = "embeddings" if kind == "embeddings" else r["name"]
        if r["dy"] is None:
            raise AssertionError("%s: its output gradient was never produced" % name)
        check_same(r["dy"], dx, "%s output gradient (%s)" % (name, what))
