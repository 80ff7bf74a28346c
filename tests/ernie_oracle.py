"""Float64 oracle of the ERNIE teacher's inference forward (``models.ernie.ErnieEncoder``), layer by layer, in bf16 and
block-scaled FP8, padded, packed and request-batched (tests/f64_bounds.py criteria).

``ErnieRecorder`` patches the entry points the forward calls through module attributes -- ``ops.embedding_layernorm``
[``_e4m3``], ``ops.gemm_bf16``, ``ops.attention``, ``ops.attention_varlen``, ``ops.layer_norm`` [``_e4m3``],
``ops.linear_bf16``, ``fp8.gemm_fp8_blockscaled``, ``fp8.gemm_fp8_gelu_e4m3``, ``fp8.quantize_e4m3_blocks`` and
``torch.tanh`` (the pooler's) -- and records every call of one forward with its arguments and outputs.  Everything is
cloned inside the wrappers, so under CUDA-graph capture the clones are part of the graph and hold each replay's values.
Exit undoes the patches.

``check(logits)`` assigns the calls to ``embeddings``, ``layers.<i>.{qkv, attention, attention quant, out, ln1, ffn1,
ffn2, ln2}``, ``pooler`` and ``classifier`` by call order, asserting the sequence of the mode that ran, and judges each
call against float64 built from exactly what that call read (teacher-forced, so per-kernel bounds hold inside the model
without compounding).  Only bounds the suite already runs are used:

* embedding-LayerNorm and LayerNorm y: ``ln_ref`` (tests/test_ernie_gpu.py's docstring), ``check_bf16`` with tau 1;
  the e4m3 variants' (q, sa) bit for bit ``fp8.quantize_e4m3_blocks_reference(y)``;
* bf16 GEMMs (QKV, out-projection and FFN2 with their addend, pooler, classifier): ``check_bf16`` at tau(K), on the
  transpose below ``E2E_MIN_ROWS`` rows (tests/teacher_oracle.py); FFN1's GELU epilogue by tests/test_ernie_gpu.py's
  ``gemm_tau(K) 1.13 mag + 6 2^-23 |pre|``;
* FP8 QKV, out-projection and FFN2: float64 of ``dequant_a`` / ``dequant_w`` plus the epilogue, criterion 1 with
  ``fp8_tau(K)``; FFN1 -> e4m3 by ``f64_bounds.check_gelu_e4m3``;
* attention, padded or packed (with ``key_mask``), head dim 64 or 32: ``student_oracle.attention_ref``, criterion 1
  with tau 1; its slack is 0 for a row without a valid key, which must therefore be exactly 0;
* ``quantize_e4m3_blocks`` of the attention output bit for bit the reference; the pooler's ``tanh`` bit for bit
  ``torch.tanh`` of its recorded input (a library op: this checks the wiring).

Wiring and weights, bit for bit: each call's operand is its producer's output (the QKV GEMM reads the layer input, the
out-projection the attention output and the layer input as addend, ...), the pooler reads rows ``b L`` (padded) or
``cu_seqlens[:-1]`` (packed) of the last LayerNorm, the returned logits are the classifier's ``[:, :num_labels]`` as
fp32, and every weight a call read equals the one rebuilt at check time from the module's current parameters
(``param.to(bf16)``, ``fp8.quantize_weight_blocks(param)``, ``param.float()``).  No call may be left unjudged, and on
CUDA ``ops.fallbacks()`` must be empty.

On CPU an FP8-enabled model emulates the pipeline through the same entry points, except that the pooler and classifier
run as float32 ``F.linear``: the recorded head is then ``tanh`` alone.  The oracle judges that form by the pooler's
pre-activation (the ``tanh`` input) and the returned logits against float64 of the recorded rows, within fp32
rounding: a sum of K products in any order in fp32, then the bias, is within K 2^-23 of the magnitude, so
``check_bf16`` with tau = K 2^-23.

A failure names the site and the mode, e.g. ``layers.7.ffn2 (fp8)``; with ``EDL_F64_BOUNDS_LOG`` set every bound check
appends its worst ratios to that file.

Worst ratios observed over tests/test_ernie_oracle_gpu.py (ernie_base, MiniLM-L12-H384 and ernie_tiny, bf16 and FP8,
padded, packed with and without ``key_mask``, L up to 512, ``forward_requests``, a graph replay; one NVIDIA H100 80GB
HBM3, 700 W power limit), read from ``EDL_F64_BOUNDS_LOG`` with the two negative controls left out (criterion 1 /
criterion 2 where it applies):

    call                                      bf16                  fp8
    embedding-LayerNorm                       c1 0.989   c2 1.00    c1 0.995   c2 1.00
    QKV                                       c1 0.997   c2 1.00    c1 0.684
    attention (head dims 64 and 32)           c1 0.519              c1 0.495
    out-projection + residual                 c1 0.999   c2 1.00    c1 0.797
    LayerNorm 1 / 2                           c1 0.992   c2 1.00    c1 0.996   c2 1.00
    FFN1 (GELU; FP8: -> e4m3)                 c1 0.996   c2 1.00    c1 0.872
    FFN2 + residual                           c1 0.994   c2 1.00    c1 0.750
    pooler                                    c1 0.993   c2 1.00    c1 0.996   c2 1.00
    classifier                                c1 0.981   c2 1.00    c1 0.966   c2 1.00
The attention quantisation, the e4m3 LayerNorm outputs, the tanh, the wiring and the weights matched bit for bit."""
import inspect
import math

import torch

import f64_bounds as fb
import student_oracle as so
import teacher_oracle as to
from edl_b200 import ops
from edl_b200.models import ernie
from edl_b200.ops import fp8

BF = torch.bfloat16
GELU_LIP = 1.13                  # max |gelu'|
_PATCHED = ((ops, "embedding_layernorm"), (ops, "embedding_layernorm_e4m3"), (ops, "gemm_bf16"), (ops, "attention"),
            (ops, "attention_varlen"), (ops, "layer_norm"), (ops, "layer_norm_e4m3"), (ops, "linear_bf16"),
            (fp8, "gemm_fp8_blockscaled"), (fp8, "gemm_fp8_gelu_e4m3"), (fp8, "quantize_e4m3_blocks"), (torch, "tanh"))


def _c(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, (tuple, list)):
        return type(v)(_c(t) for t in v)
    return v


class Call:
    """One recorded call: ``name``, its bound arguments ``a`` (defaults filled in) and its output ``out``."""

    def __init__(self, name, a, out):
        self.name, self.a, self.out = name, a, out

    def __repr__(self):
        return "Call(%s)" % self.name


def random_vectors(model, seed, cls_scale=20.0):
    """Random biases and LayerNorm parameters (gamma in [0.5, 1.5], beta and biases ~ N(0, 0.1)) in every layer, the
    embeddings, pooler and classifier, and ``cls_w`` scaled so the logits are decisive."""
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.dim() != 1:
                continue
            if name.endswith("_g"):
                v = torch.rand(p.shape, generator=gen) + 0.5
            else:
                v = torch.randn(p.shape, generator=gen) * 0.1
            p.copy_(v.to(p.device))
        model.cls_w.mul_(cls_scale)


class ErnieRecorder:
    """Records one forward of ``model`` (an ``ErnieEncoder``) inside ``with ErnieRecorder(model) as rec:``."""

    def __init__(self, model):
        self.model = model
        self.calls = []
        self._patched = []

    def __enter__(self):
        self.calls = []
        for mod, name in _PATCHED:
            orig = getattr(mod, name)
            setattr(mod, name, self._wrap(name, orig))
            self._patched.append((mod, name, orig))
        return self

    def __exit__(self, *exc):
        for mod, name, orig in reversed(self._patched):
            setattr(mod, name, orig)
        self._patched = []

    def _wrap(self, name, fn):
        sig = None if name == "tanh" else inspect.signature(fn)
        calls = self.calls

        def wrapped(*args, **kwargs):
            out = fn(*args, **kwargs)
            if sig is None:
                a = {"x": _c(args[0])}
            else:
                b = sig.bind(*args, **kwargs)
                b.apply_defaults()
                a = {k: _c(v) for k, v in b.arguments.items()}
            calls.append(Call(name, a, _c(out)))
            return out

        return wrapped

    # ------------------------------------------------------------------------------------------------------- checks
    def sites(self):
        """[(site, call)] in call order, after asserting the per-layer sequence of the mode that ran."""
        m = self.model
        q = m._fp8
        cuda = m.word_emb.is_cuda
        att = [c.name for c in self.calls if c.name in ("attention", "attention_varlen")]
        att = att[0] if att else "attention"
        want = [("embeddings", "embedding_layernorm_e4m3" if q else "embedding_layernorm")]
        for i in range(m.num_layers):
            p = "layers.%d." % i
            if q:
                want += [(p + "qkv", "gemm_fp8_blockscaled"), (p + "attention", att),
                         (p + "attention quant", "quantize_e4m3_blocks"), (p + "out", "gemm_fp8_blockscaled"),
                         (p + "ln1", "layer_norm_e4m3"), (p + "ffn1", "gemm_fp8_gelu_e4m3"),
                         (p + "ffn2", "gemm_fp8_blockscaled"),
                         (p + "ln2", "layer_norm_e4m3" if i < m.num_layers - 1 else "layer_norm")]
            else:
                want += [(p + "qkv", "gemm_bf16"), (p + "attention", att), (p + "out", "gemm_bf16"), (p + "ln1", "layer_norm"),
                         (p + "ffn1", "gemm_bf16"), (p + "ffn2", "gemm_bf16"), (p + "ln2", "layer_norm")]
        if cuda:
            want += [("pooler", "linear_bf16"), ("pooler tanh", "tanh"), ("classifier", "gemm_bf16")]
        else:
            want += [("pooler tanh", "tanh")]          # the CPU head: float32 F.linear around the tanh
        got = [c.name for c in self.calls]
        for k, ((site, name), g) in enumerate(zip(want, got)):
            if name != g:
                raise AssertionError("%s (%s): call %d is %s, expected %s" % (site, self.mode, k, g, name))
        if len(got) != len(want):
            raise AssertionError("%d calls recorded, %d expected in %s mode (%s)" % (
                len(got), len(want), self.mode, "missing " + want[len(got)][0] if len(got) < len(want)
                else "unjudged " + ", ".join(got[len(want):])))
        return list(zip([s for s, _ in want], self.calls))

    @property
    def mode(self):
        return "fp8" if self.model._fp8 else "bf16"

    def check(self, logits, log=print):
        """Judge every recorded call and the returned ``logits``; returns {call kind: (worst c1, worst c2)}."""
        m = self.model
        if m.word_emb.is_cuda:
            assert ops.fallbacks() == {}, ops.fallbacks()
        worst = {}

        def note(kind, r):
            c1, c2 = (r if isinstance(r, tuple) else (r, None))
            w = worst.setdefault(kind, [0.0, 0.0])
            w[0] = max(w[0], c1 or 0.0)
            w[1] = max(w[1], c2 or 0.0)

        sites = dict(self.sites())
        lab = lambda s: "%s (%s)" % (s, self.mode)                               # noqa: E731
        same = lambda got, want, what: so.check_same(got, want.to(got.device), what)   # noqa: E731
        q = bool(m._fp8)
        c = m.hidden

        def wmat(p):
            return p.detach().to(BF)

        def wvec(p):
            return p.detach().float()

        def check_q(y, qs, what):
            rq, rs = fp8.quantize_e4m3_blocks_reference(y)
            same(qs[0], rq, what + " e4m3 operand")
            same(qs[1], rs, what + " e4m3 block scales")

        # ---- embeddings
        e = sites["embeddings"]
        what = lab("embeddings")
        for k, p in (("word", m.word_emb), ("pos", m.pos_emb), ("seg", m.seg_emb)):
            same(e.a[k], wmat(p), what + " " + k + " table")
        same(e.a["gamma"], wvec(m.emb_ln_g), what + " gamma")
        same(e.a["beta"], wvec(m.emb_ln_b), what + " beta")
        assert e.a["eps"] == m.eps, what + " eps"
        terms = [e.a["word"].double()[e.a["ids"].reshape(-1)], e.a["pos"].double()[e.a["pos_ids"].reshape(-1)],
                 e.a["seg"].double()[e.a["seg_ids"].reshape(-1)]]
        y = e.out[0] if q else e.out
        ref, slack = so.ln_ref(sum(terms), e.a["gamma"], e.a["beta"], m.eps, dx=2 * fb.EPS32 * sum(t.abs() for t in terms))
        note("LayerNorm, embedding-LayerNorm", fb.check_bf16(y, ref, slack, tau=1.0, what=what))
        if q:
            check_q(y, e.out[1:], what)
        x, xq = y, (e.out[1:] if q else None)            # the layer input and its e4m3 copy

        att_call = None
        for i, lyr in enumerate(m.layers):
            p = "layers.%d." % i
            # ---- QKV
            s = sites[p + "qkv"]
            what = lab(p + "qkv")
            qkv = self._gemm(s, what, x, xq, None, lyr.qkv_w, lyr.qkv_b, note)
            # ---- attention
            s = att_call = sites[p + "attention"]
            what = lab(p + "attention")
            same(s.a["qkv"], qkv, what + " operand (the QKV output)")
            note("attention", self._attention(s, what))
            ctx = s.out
            ctxq = None
            if q:
                s = sites[p + "attention quant"]
                what = lab(p + "attention quant")
                same(s.a["x"], ctx, what + " operand (the attention output)")
                check_q(ctx, s.out, what)
                ctxq = s.out
            # ---- out-projection + residual
            h1 = self._gemm(sites[p + "out"], lab(p + "out"), ctx, ctxq, x, lyr.out_w, lyr.out_b, note)
            # ---- LayerNorm 1
            x1, x1q = self._ln(sites[p + "ln1"], lab(p + "ln1"), h1, lyr.ln1_g, lyr.ln1_b, q, note, check_q)
            # ---- FFN1 (GELU)
            s = sites[p + "ffn1"]
            what = lab(p + "ffn1")
            fq = None
            if q:
                same(s.a["a8"], x1q[0], what + " e4m3 operand (ln1's)")
                same(s.a["sa"], x1q[1], what + " operand block scales (ln1's)")
                w8, sw = fp8.quantize_weight_blocks(lyr.ffn1_w.detach())
                same(s.a["b8"], w8, what + " e4m3 weight")
                same(s.a["sb"], sw, what + " weight block scales")
                same(s.a["bias"], wvec(lyr.ffn1_b), what + " bias")
                a64, w64 = fb.dequant_a(s.a["a8"], s.a["sa"]), fb.dequant_w(w8, sw)
                pre, mag = fb.epilogue(a64 @ w64.t(), a64.abs() @ w64.abs().t(), shift=s.a["bias"])
                note("FP8 FFN1 -> e4m3", fb.check_gelu_e4m3(s.out[0], s.out[1], pre, mag, a64.shape[1], what=what))
                fq, f = s.out, None
            else:
                same(s.a["a"], x1, what + " operand (ln1's output)")
                same(s.a["b"], wmat(lyr.ffn1_w), what + " weight")
                same(s.a["col_shift"], wvec(lyr.ffn1_b), what + " bias")
                assert s.a["gelu"] and s.a["add"] is None and s.a["col_scale"] is None, what + " epilogue flags"
                pre, mag = fb.gemm_ref(s.a["a"], s.a["b"], shift=s.a["col_shift"])
                ref = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
                k = s.a["a"].shape[1]
                note("bf16 FFN1 (GELU)", fb.check_bf16(s.out, ref, fb.tau(k) * GELU_LIP * mag + 6 * fb.EPS32 * pre.abs(),
                                                       tau=1.0, what=what))
                f = s.out
            # ---- FFN2 + residual
            h2 = self._gemm(sites[p + "ffn2"], lab(p + "ffn2"), f, fq, x1, lyr.ffn2_w, lyr.ffn2_b, note)
            # ---- LayerNorm 2
            last = i == m.num_layers - 1
            x, xq = self._ln(sites[p + "ln2"], lab(p + "ln2"), h2, lyr.ln2_g, lyr.ln2_b, q and not last, note, check_q)

        # ---- head: the [CLS] rows of the last LayerNorm
        if att_call.name == "attention":
            b, l = att_call.a["batch"], att_call.a["seq_len"]
            first = torch.arange(b, device=x.device) * l
        else:
            first = att_call.a["cu_seqlens"][:-1].long().to(x.device)
        cls = x.index_select(0, first)
        t = sites["pooler tanh"]
        n = m.num_labels
        if m.word_emb.is_cuda:
            s = sites["pooler"]
            what = lab("pooler")
            same(s.a["x"], cls, what + " operand (the [CLS] rows of the last LayerNorm)")
            same(s.a["weight"], wmat(m.pool_w), what + " weight")
            same(s.a["bias"], wvec(m.pool_b), what + " bias")
            assert not s.a["relu"] and not s.a["gelu"], what + " epilogue flags"
            note("bf16 GEMM", to.check_bf16(s.out, *fb.gemm_ref(cls, s.a["weight"], shift=s.a["bias"]), c, what=what))
            same(t.a["x"], s.out, lab("pooler tanh") + " operand (the pooler output)")
        else:
            pw = wmat(m.pool_w)
            note("CPU head (fp32)", to.check_bf16(t.a["x"], *fb.gemm_ref(cls, pw, shift=wvec(m.pool_b)),
                                                  tau=c * fb.EPS32, what=lab("pooler") + " (float32 head)"))
        same(t.out, torch.tanh(t.a["x"]), lab("pooler tanh"))
        pooled = t.out
        rows = m.cls_w.shape[0]
        pad = max(ernie.CLS_PAD, -(-rows // ernie.CLS_PAD) * ernie.CLS_PAD)
        cls_w = torch.zeros(pad, c, device=m.cls_w.device)
        cls_w[:rows] = m.cls_w.detach().float()
        cls_b = torch.zeros(pad, device=m.cls_w.device)
        cls_b[:rows] = m.cls_b.detach().float()
        if m.word_emb.is_cuda:
            s = sites["classifier"]
            what = lab("classifier")
            same(s.a["a"], pooled, what + " operand (the tanh output)")
            same(s.a["b"], cls_w.to(BF), what + " weight")
            same(s.a["col_shift"], cls_b, what + " bias")
            assert s.a["add"] is None and not s.a["gelu"] and s.a["col_scale"] is None, what + " epilogue flags"
            note("bf16 GEMM", to.check_bf16(s.out, *fb.gemm_ref(pooled, s.a["b"], shift=cls_b), c, what=what))
            same(logits, s.out[:, :n].float(), lab("logits") + " (the classifier's first num_labels columns)")
        else:
            ref, mag = fb.gemm_ref(pooled, cls_w[:n].to(BF), shift=cls_b[:n])
            note("CPU head (fp32)", to.check_bf16(logits.to(BF), ref, mag, tau=c * fb.EPS32,
                                                  what=lab("classifier") + " (float32 head)"))
            same(logits, logits.to(BF).float(), lab("logits") + " (bf16 values)")
        for kind, (c1, c2) in sorted(worst.items()):
            log("ernie oracle %s: worst c1 %.3f, c2 %.3f" % (kind, c1, c2))
        return {k: tuple(v) for k, v in worst.items()}

    # ------------------------------------------------------------------------------------------------------ helpers
    def _gemm(self, s, what, a, aq, add, w, bias, note):
        """A QKV, out-projection or FFN2 call: operand ``a`` (bf16) or ``aq`` (e4m3 bytes and scales), the residual
        ``add`` (None for QKV)."""
        same = lambda got, want, w_: so.check_same(got, want.to(got.device), w_)   # noqa: E731
        if self.model._fp8:
            same(s.a["a8"], aq[0], what + " e4m3 operand (its producer's)")
            same(s.a["sa"], aq[1], what + " operand block scales (its producer's)")
            w8, sw = fp8.quantize_weight_blocks(w.detach())
            same(s.a["b8"], w8, what + " e4m3 weight")
            same(s.a["sb"], sw, what + " weight block scales")
            same(s.a["col_shift"], bias.detach().float(), what + " bias")
            assert s.a["col_scale"] is None and not s.a["relu"], what + " epilogue flags"
            if add is None:
                assert s.a["add"] is None, what + ": an addend where none is expected"
            else:
                same(s.a["add"], add, what + " addend (the layer's residual input)")
            a64, w64 = fb.dequant_a(s.a["a8"], s.a["sa"]), fb.dequant_w(w8, sw)
            ref, mag = fb.epilogue(a64 @ w64.t(), a64.abs() @ w64.abs().t(), add=s.a["add"], shift=s.a["col_shift"])
            k = a64.shape[1]
            note("FP8 GEMM (QKV, out, FFN2)", fb.check_bf16(s.out, ref, mag, tau=fb.fp8_tau(k), criteria=(1,), what=what))
            return s.out
        same(s.a["a"], a, what + " operand (its producer's output)")
        same(s.a["b"], w.detach().to(BF), what + " weight")
        same(s.a["col_shift"], bias.detach().float(), what + " bias")
        assert not s.a["gelu"] and s.a["col_scale"] is None and not s.a["relu"], what + " epilogue flags"
        if add is None:
            assert s.a["add"] is None, what + ": an addend where none is expected"
        else:
            same(s.a["add"], add, what + " addend (the layer's residual input)")
        ref, mag = fb.gemm_ref(s.a["a"], s.a["b"], add=s.a["add"], shift=s.a["col_shift"])
        note("bf16 GEMM", to.check_bf16(s.out, ref, mag, s.a["a"].shape[1], what=what))
        return s.out

    def _ln(self, s, what, h, g, b, quant, note, check_q):
        same = lambda got, want, w_: so.check_same(got, want.to(got.device), w_)   # noqa: E731
        same(s.a["x"], h, what + " operand (the residual GEMM's output)")
        same(s.a["gamma"], g.detach().float(), what + " gamma")
        same(s.a["beta"], b.detach().float(), what + " beta")
        assert s.a["eps"] == self.model.eps, what + " eps"
        y = s.out[0] if quant else s.out
        note("LayerNorm, embedding-LayerNorm", fb.check_bf16(y, *so.ln_ref(h.double(), s.a["gamma"], s.a["beta"],
                                                                           self.model.eps), tau=1.0, what=what))
        if quant:
            check_q(y, s.out[1:], what)
            return y, s.out[1:]
        return y, None

    def _attention(self, s, what):
        m = self.model
        qkv, out, d = s.a["qkv"], s.out, m.head_dim
        if s.name == "attention":
            assert (s.a["heads"], s.a["head_dim"]) == (m.heads, d), what + " heads / head dim"
            b, l = s.a["batch"], s.a["seq_len"]
            ref, slack = so.attention_ref(qkv, s.a["mask"], b, l, m.heads, d)
            return fb.check_bf16(out, ref, slack, tau=1.0, criteria=(1,), what=what)[0]
        assert s.a["heads"] == m.heads and qkv.shape[1] == 3 * m.heads * d, what + " heads / head dim"
        cu = [int(v) for v in s.a["cu_seqlens"].tolist()]
        assert cu[0] == 0 and cu[-1] == qkv.shape[0] and max(e - s_ for s_, e in zip(cu[:-1], cu[1:])) <= s.a["max_len"], \
            what + " cu_seqlens / max_len"
        km = s.a["key_mask"]
        refs, slacks = [], []
        for s_, e in zip(cu[:-1], cu[1:]):
            mk = None if km is None else km[s_:e].view(1, e - s_)
            r, sl = so.attention_ref(qkv[s_:e], mk, 1, e - s_, m.heads, d)
            refs.append(r)
            slacks.append(sl)
        return fb.check_bf16(out, torch.cat(refs), torch.cat(slacks), tau=1.0, criteria=(1,), what=what)[0]
