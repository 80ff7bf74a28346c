"""Float64 oracle of the ResNeXt teacher's inference forward, layer by layer (tests/f64_bounds.py criteria).

``TeacherRecorder`` is attached to a ``models.resnext.ResNeXt`` (or the teacher zoo's softmax wrapper around one) and
records, per layer, the tensors that layer read and wrote in one forward: every ``FoldedConv``'s input, residual,
output and folded-BN ``scale`` / ``shift``, the global average pool, the classifier and the softmax.  It also wraps the
ops a ``FoldedConv`` calls, so it knows which path ran -- fused 1x1, two-kernel residual, widened groups,
``conv3x3_s2_infer``, stride 1 then subsample, ``stem7_infer``, FP8 per-tensor or FP8 block -- and keeps the
intermediate bf16 GEMM output of the two-step residual paths.  Everything is cloned inside the hooks, so under CUDA-graph
capture the clones become part of the graph and hold each replay's values.

``check()`` judges every layer against float64 built from its recorded input (teacher-forced):

* a convolution that ran on the library (ResNeXt_tiny's narrow groups): criterion 2 on its stored output, then
  ``scale_shift_act`` on that output;
* bf16 1x1 (stride 1 or 2), grouped 3x3 (every route, against the ORIGINAL grouped weight and ``groups``: this checks
  the block-diagonal widening and the stride-2 kernel against plain grouped-convolution semantics), the 7x7 stem and the
  classifier: criteria 1 and 2;
* the fused residual 1x1 against the bf16 weight the kernel reads, ``bf16(W scale)``; the two-kernel residual path as
  its GEMM and then ``scale_shift_act`` on the GEMM's stored output;
* max-pool exactly (its output is the first block's recorded input), the global pool with ``gap_tau``, the softmax within
  fp32 rounding of float64 softmax of the recorded logits;
* FP8 layers from the quantised operand recomputed with the torch references (and checked bit for bit against the one
  the kernel read): float64 of the dequantised operands times the stored scales, then the epilogue, by criterion 1 with
  ``fp8_tau`` (block) or ``fp8_tensor_tau`` (per-tensor); FP8 residual layers as GEMM, then ``scale_shift_act``.

Failure messages name the module path and the path, e.g. ``blocks.12.c2 (widened, s2)``."""
import math
from collections import defaultdict

import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.models import resnext
from edl_b200.ops import fp8

SSA_TAU = 2 * fb.EPS32          # scale_shift_act: one fmaf, then the residual add
SOFTMAX_TAU = 64 * fb.EPS32     # fp32 softmax of fp32 logits: exp, the row sum and the quotient, relative


def _c(t):
    return None if t is None else t.detach().clone()


def check_bf16(out, ref, mag, *args, **kw):
    """``fb.check_bf16``; an output of fewer than ``fb.E2E_MIN_ROWS`` rows (the pooled features, the logits, the last
    stage's maps of a small image) is judged on its transpose, per pixel over the channels, as tests/step_oracle.py."""
    o, r, g = fb.rows(out), fb.rows(ref), fb.rows(mag)
    if o.shape[0] < fb.E2E_MIN_ROWS <= o.shape[1]:
        o, r, g = o.t(), r.t(), g.t()
    return fb.check_bf16(o, r, g, *args, **kw)


def classify(calls, conv):
    """The path a ``FoldedConv`` forward took, from the ops it called (``calls``: (op name, info) in call order)."""
    names = [c[0] for c in calls]
    if "gemm_fp8_blockscaled" in names:
        return "fp8 block" + (", residual" if "scale_shift_act" in names else "")
    if "gemm_fp8" in names:
        return "fp8 tensor" + (", residual" if "scale_shift_act" in names else "")
    if "stem7_infer" in names:
        return "stem7"
    for op, tag in (("conv3x3_s2_infer", "s2"), ("conv3x3_infer", "subsample" if conv.stride == 2 else "s1")):
        if op in names:
            widened = dict(calls)[op]["widened"]
            return ("widened, " if widened else "") + tag
    if "gemm_bf16" in names:
        if dict(calls)["gemm_bf16"].get("add"):
            return "fused residual"
        return "two-kernel residual" if "scale_shift_act" in names else "1x1"
    return "library"


class _Conv:
    def __init__(self, name, mod):
        self.name, self.mod = name, mod
        self.x = self.res = self.out = None
        self.calls = []
        self.inter = None        # the bf16 GEMM output of a two-step residual path
        self.x8 = None           # the quantised operand the FP8 kernel read (per-tensor: bytes; block: (bytes, sa))
        self.runs = 0

    @property
    def path(self):
        return classify(self.calls, self.mod)

    @property
    def label(self):
        return "%s (%s)" % (self.name, self.path)


class TeacherRecorder:
    """Records one forward of ``model`` (a ResNeXt, or a module with ``.net`` = ResNeXt whose output is the softmax)."""

    def __init__(self, model):
        self.top = model
        self.net = getattr(model, "net", model)
        self.names = {m: n for n, m in self.net.named_modules()}
        self._hooks, self._patched = [], []
        self._current = None
        self.reset()

    def reset(self):
        self.convs = {m: _Conv(n, m) for m, n in self.names.items() if isinstance(m, resnext.FoldedConv)}
        self.gap = None
        self.logits = self.probs = None

    # ------------------------------------------------------------------------------------------------------ capture
    def __enter__(self):
        for m, rec in self.convs.items():
            self._hooks.append(m.register_forward_pre_hook(self._pre, with_kwargs=True))
            self._hooks.append(m.register_forward_hook(self._post, with_kwargs=True))
        self._hooks.append(self.net.register_forward_hook(self._net_post))
        if self.top is not self.net:
            self._hooks.append(self.top.register_forward_hook(self._top_post))
        for mod, name in ((ops, "gemm_bf16"), (ops, "scale_shift_act"), (ops, "conv3x3_s2_infer"), (ops, "conv3x3_infer"),
                          (ops, "stem7_infer"), (ops, "global_avg_pool"), (fp8, "gemm_fp8"), (fp8, "gemm_fp8_blockscaled"),
                          (fp8, "quantize_e4m3"), (fp8, "quantize_e4m3_blocks")):
            orig = getattr(mod, name)
            setattr(mod, name, self._wrap(name, orig))
            self._patched.append((mod, name, orig))
        return self

    def __exit__(self, *exc):
        for h in self._hooks:
            h.remove()
        for mod, name, orig in self._patched:
            setattr(mod, name, orig)
        self._hooks, self._patched = [], []

    def _pre(self, m, args, kwargs):
        rec = self.convs[m]
        rec.runs += 1
        rec.calls = []
        rec.inter = rec.x8 = None
        rec.x = _c(args[0])
        rec.res = _c(kwargs.get("residual", args[1] if len(args) > 1 else None))
        rec.scale, rec.shift = _c(m.scale), _c(m.shift)
        self._current = rec

    def _post(self, m, args, kwargs, out):
        rec = self.convs[m]
        rec.out = _c(out)
        rec.act_scale = _c(getattr(m, "act_scale", None)) if m._fp8 == "tensor" else None
        rec.w8 = None
        if m._fp8 is not None:
            w8, ws, _, _ = m._fp8_weights()
            rec.w8, rec.ws = _c(w8), _c(ws)
        self._current = None

    def _net_post(self, m, args, out):
        self.logits = _c(out)

    def _top_post(self, m, args, out):
        self.probs = _c(out)

    def _wrap(self, name, fn):
        rec_of = self

        def wrapped(*args, **kwargs):
            out = fn(*args, **kwargs)
            rec = rec_of._current
            if name == "global_avg_pool":
                rec_of.gap = (_c(args[0]), _c(out))
            elif rec is not None:
                info = {}
                if name in ("conv3x3_s2_infer", "conv3x3_infer"):
                    info["widened"] = args[1].shape[3] != rec.mod.weight.shape[3]
                elif name == "gemm_bf16":
                    info["add"] = kwargs.get("add") is not None
                    rec.inter = _c(kwargs.get("out", out))
                elif name in ("gemm_fp8", "gemm_fp8_blockscaled"):
                    rec.inter = _c(kwargs.get("out", out))
                elif name == "scale_shift_act" and rec.inter is None:
                    rec.inter = _c(args[0])             # the library convolution's stored output
                elif name == "quantize_e4m3":
                    rec.x8 = _c(out)
                elif name == "quantize_e4m3_blocks":
                    rec.x8 = tuple(_c(t) for t in out)
                rec.calls.append((name, info))
            return out

        return wrapped

    # ------------------------------------------------------------------------------------------------------- checks
    def paths(self):
        """{module path: path taken} of the recorded forward."""
        return {r.name: r.path for r in self.convs.values()}

    def check(self, log=print):
        """Judge every recorded layer; returns {category: (worst criterion-1 ratio, worst criterion-2 ratio)}."""
        worst = defaultdict(lambda: [0.0, 0.0])

        def note(cat, c1, c2=None):
            w = worst[cat]
            w[0] = max(w[0], c1 or 0.0)
            w[1] = max(w[1], c2 or 0.0)

        not_once = [r.name for r in self.convs.values() if r.runs != 1]
        assert not not_once, "layers that did not run exactly once: %s" % not_once
        for rec in self.convs.values():
            cat, ratios = self._check_conv(rec, log)
            note(cat, *ratios)
        pooled = self.convs[self.net.blocks[0].c1].x
        fb.check_exact(pooled.double(), fb.maxpool_ref(self.convs[self.net.stem].out)[0], what="max-pool (blocks.0 input)")
        if self.gap is not None:
            x, out = self.gap
            last = self.convs[self.net.blocks[-1].c3].out
            fb.check_exact(x, last, what="global pool input (last block output)")
            note("pools", check_bf16(out, *fb.gap_ref(x), tau=fb.gap_tau(x.shape[2] * x.shape[3]),
                                     what="global pool")[0])
            feats = out
            ref, mag = fb.gemm_ref(feats, self.net.fc_weight, shift=self.net.fc_bias)
            note("classifier", *check_bf16(self.logits, ref, mag, feats.shape[1], what="classifier"))
        if self.probs is not None:
            p64 = torch.softmax(self.logits.double(), -1)
            err = (self.probs.double() - p64).abs()
            bound = SOFTMAX_TAU * p64 + 2.0 ** -149
            ratio = float((err / bound).max())
            assert ratio <= 1, "softmax: worst |p - p64| / bound %.3g" % ratio
            note("softmax", ratio)
        return dict(worst)

    def _check_conv(self, rec, log):
        m, path = rec.mod, rec.path
        what = rec.label
        s = m.stride
        sc4, sh4 = rec.scale.view(1, -1, 1, 1), rec.shift.view(1, -1, 1, 1)     # per channel of NCHW references
        if path.startswith("fp8"):
            return ("fp8 block" if path.startswith("fp8 block") else "fp8 tensor"), self._check_fp8(rec, log)
        w = m.weight
        if path == "fused residual":
            # the weight the kernel reads is bf16(W scale), built here from the weight and the recorded scale
            w1 = (w.view(m.cout, m.cin).float() * rec.scale.float()[:, None]).to(w.dtype)
            fb.check_exact(m._scaled_weight(), w1, what=what + " scaled weight")
            w1 = w1.view(m.cout, 1, 1, m.cin)
            ref, mag = fb.conv_ref(rec.x, w1, stride=s, padding=0, add=rec.res, shift=sh4, relu=m.relu)
            return "bf16", check_bf16(rec.out, ref, mag, m.cin, what=what)
        if path == "two-kernel residual":
            ref, mag = fb.conv_ref(rec.x, w, stride=s, padding=0)
            r1 = check_bf16(rec.inter, ref, mag, m.cin, what=what + " GEMM")
            y1 = rec.inter.view(rec.out.shape[0], rec.out.shape[2], rec.out.shape[3], -1).permute(0, 3, 1, 2)
            ref, mag = fb.scale_shift_ref(y1, rec.scale, rec.shift, rec.res, m.relu)
            r2 = check_bf16(rec.out, ref, mag, tau=SSA_TAU, what=what + " scale_shift_act")
            return "bf16", (max(r1[0], r2[0]), max(r1[1], r2[1]))
        if path == "1x1":
            ref, mag = fb.conv_ref(rec.x, w, stride=s, padding=0, scale=sc4, shift=sh4, relu=m.relu)
            return "bf16", check_bf16(rec.out, ref, mag, m.cin, what=what)
        if path == "stem7":
            ref, mag = fb.conv_ref(rec.x, w, stride=2, padding=3, scale=sc4, shift=sh4, relu=m.relu)
            return "bf16", check_bf16(rec.out, ref, mag, 160, what=what)
        if path in ("s1", "s2", "subsample") or path.startswith("widened"):
            k = 9 * (64 if path.startswith("widened") else w.shape[3])
            ref, mag = fb.conv_ref(rec.x, w, stride=s, padding=1, groups=m.groups, scale=sc4, shift=sh4,
                                   relu=m.relu)
            return "bf16", check_bf16(rec.out, ref, mag, k, what=what)
        # library convolution (not this project's kernel: criterion 2 alone), then scale_shift_act on its stored output
        ref, mag = fb.conv_ref(rec.x, w, stride=s, padding=(m.k - 1) // 2, groups=m.groups)
        r1 = check_bf16(rec.inter, ref, mag, w.shape[1] * w.shape[2] * w.shape[3], criteria=(2,), what=what + " conv")
        ref, mag = fb.scale_shift_ref(rec.inter, rec.scale, rec.shift, rec.res, m.relu)
        r2 = check_bf16(rec.out, ref, mag, tau=SSA_TAU, what=what + " scale_shift_act")
        return "library", (r2[0], max(r1[1], r2[1]))

    def _check_fp8(self, rec, log):
        m, what = rec.mod, rec.label
        s = m.stride
        x = rec.x[:, :, ::s, ::s] if s != 1 else rec.x
        x2 = fb.rows(x)
        k = m.cin
        w2 = m.weight.detach().view(m.cout, m.cin)
        if rec.path.startswith("fp8 block"):
            q, sa = fp8.quantize_e4m3_blocks_reference(x2)
            fb.check_exact(rec.x8[0], q, what=what + " quantised operand")
            fb.check_exact(rec.x8[1], sa, what=what + " operand block scales")
            # the weights and their block scales from the current weight, not from the layer's cache
            w8, sb = fp8.quantize_weight_blocks(w2)
            fb.check_exact(rec.w8, w8, what=what + " e4m3 weights")
            fb.check_exact(rec.ws, sb, what=what + " weight block scales")
            a64, w64 = fb.dequant_a(q, sa), fb.dequant_w(w8, sb)
            acc, mag = a64 @ w64.t(), a64.abs() @ w64.abs().t()
            scale, tau = rec.scale.double(), fb.fp8_tau(k)
        else:
            q = (x2.float() / rec.act_scale).clamp(-fp8.E4M3_MAX, fp8.E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)
            fb.check_exact(rec.x8, q, what=what + " quantised operand")
            # the column scale the epilogue must use: activation scale x weight-row scale x folded-BN scale, in fp32,
            # built from the recorded activation and BN scales and the current weight
            w8, ws = fp8.quantize_weight_rows(w2)
            deq = (rec.act_scale * ws * rec.scale).contiguous()
            fb.check_exact(rec.w8, w8, what=what + " e4m3 weights")
            fb.check_exact(rec.ws, deq, what=what + " dequantisation scale")
            a64, w64 = q.view(torch.float8_e4m3fn).double(), w8.view(torch.float8_e4m3fn).double()
            acc, mag = a64 @ w64.t(), a64.abs() @ w64.abs().t()
            scale, tau = deq.double(), fb.fp8_tensor_tau(k)
        shift = rec.shift.double()
        res = rec.res is not None
        ref = acc * scale + shift
        mag = mag * scale.abs() + shift.abs()
        if m.relu and not res:
            ref = ref.relu()
        gemm_out = rec.inter if res else fb.rows(rec.out)
        c1, _ = fb.check_bf16(gemm_out, ref, mag, tau=tau, criteria=(1,), what=what + (" GEMM" if res else ""))
        log("%s: worst criterion-1 ratio %.3f (tau %.3g)" % (what, c1, tau))
        if res:
            y1 = rec.inter.view(rec.out.shape[0], rec.out.shape[2], rec.out.shape[3], -1).permute(0, 3, 1, 2)
            ones = torch.ones_like(rec.scale)
            r, g = fb.scale_shift_ref(y1, ones, torch.zeros_like(rec.shift), rec.res, m.relu)
            c1b, c2 = check_bf16(rec.out, r, g, tau=SSA_TAU, what=what + " scale_shift_act")
            return max(c1, c1b), c2
        return c1, None


def random_bn(model, seed, device=None):
    """Random folded BatchNorm in every ``FoldedConv`` (``load_bn``) and a nonzero classifier bias: gamma in
    [0.5, 1.5] / sqrt(depth) for the layers that end a residual block, so the sum over ~30 blocks stays in range; beta and
    the mean ~ N(0, 0.1); var in [0.5, 1.5]."""
    gen = torch.Generator().manual_seed(seed)
    depth = len(model.blocks)
    for name, m in model.named_modules():
        if isinstance(m, resnext.FoldedConv):
            c = m.cout
            g = torch.rand(c, generator=gen) + 0.5
            if name.endswith(".c3") or name.endswith(".ds"):
                g = g / math.sqrt(depth)
            args = (g, torch.randn(c, generator=gen) * 0.1, torch.randn(c, generator=gen) * 0.1,
                    torch.rand(c, generator=gen) + 0.5)
            m.load_bn(*[a.to(m.scale.device) for a in args])
    with torch.no_grad():
        model.fc_bias.copy_((torch.randn(model.fc_bias.shape, generator=gen) * 0.5).to(model.fc_bias.device))


def stage_rms(rec, model):
    """RMS of the stem's output and of each stage's output (its last block) from a recorder's records."""
    out = {"stem": rec.convs[model.stem].out}
    ends = [i - 1 for i, b in enumerate(model.blocks) if i > 0 and b.ds is not None] + [len(model.blocks) - 1]
    for st, i in enumerate(ends):
        out["stage %d" % (st + 1)] = rec.convs[model.blocks[i].c3].out
    return {k: float(v.double().square().mean().sqrt()) for k, v in out.items()}
