"""Float64 oracle of a whole training step, layer by layer (tests/f64_bounds.py criteria).

``StepRecorder`` is attached to a ResNet-vd or plain ResNet before a step and records, per layer, the tensors that layer
actually read and wrote in that step: each convolution's input, weight, output and epilogue statistics; each
BatchNorm's input, residual, output, saved ``mean`` / ``rstd`` / ReLU mask bits, the running statistics before the
update and the parameters it read; the pools, the classifier and the loss; and, through tensor hooks, the gradient of
every activation.  Everything is cloned inside the hooks: ``dres`` aliases ``dy`` and autograd may add into it in place,
and under CUDA-graph capture the clones become part of the graph, so after a replay they hold that replay's values.

``check()`` then judges every layer against a float64 reference built from those recorded inputs (teacher-forced:
rounding errors do not compound through the network, so the per-kernel bounds also hold inside the model), every
activation gradient against the sum of its consumers' contributions, and every element of every trainable parameter's
gradient -- in its flat-bucket window (``p._edl_grad_sink``) or in ``p.grad`` -- exactly once.  A layer that ran on the
library (``ops.fallbacks()``) is judged by criterion 2 alone and named in the report.  Failure messages name the module
path and the pass, e.g. ``blocks.7.c dgrad`` or ``blocks.3.short wgrad (bucket)``."""
import math
from collections import defaultdict

import torch

import f64_bounds as fb
from edl_b200 import ops
from edl_b200.models.resnet_vd import ConvBNAct
from edl_b200.ops import gemm as G

EPS = fb.EPS32


def _c(t):
    return None if t is None else t.detach().clone()


def bn_tau(m, c):
    """fp32 bound of whichever BatchNorm reduction kernel ran (register, streaming or SM-resident): the largest."""
    return max(fb.bn_reduce_tau(p, m, c) for p in ("regs", "stream", "fused"))


def ref_soft_ce_grad(z, target, kind):
    """d(loss)/dz of ``ops.soft_cross_entropy`` (default temperatures, no smoothing) in float64."""
    z64 = z.double()
    n, c = z64.shape
    if kind == "labels":
        p = torch.zeros_like(z64)
        p[torch.arange(n, device=z.device), target] = 1.0
    elif kind == "probs":
        p = target.double()
    else:
        p = torch.softmax(target.double(), -1)
    return (torch.softmax(z64, -1) * p.sum(-1, keepdim=True) - p) / n


def check_logits_grad(got, ref, what):
    """|got - ref| <= 1e-4 |ref| + 1e-6 max_row |ref| (+ one bf16 ulp of ref for a bf16 gradient), as the loss tests."""
    ref = ref.to(got.device)
    bound = 1e-4 * ref.abs() + 1e-6 * ref.abs().amax(-1, keepdim=True)
    if got.dtype == torch.bfloat16:
        bound = bound + fb.ulp(ref, 8)
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("%s: %d elements out of bounds, first at %s: got %r, ref %r" % (
            what, int(bad.sum()), i, got[i].item(), ref[i].item()))
    return float((err / bound.clamp_min(1e-300)).max())


def ref_sgd(w, v, g, lr, mu, wd):
    """One SGD-momentum step in float64 with its bounds, as tests/test_optim_gpu.py."""
    w, v, g = w.double(), v.double(), g.double()
    gg = g + wd * w
    v1 = mu * v + gg
    mag_v = mu * v.abs() + g.abs() + (wd * w).abs()
    return w - lr * v1, v1, 1e-6 * (w.abs() + lr * mag_v), 1e-6 * mag_v


def _assert_close(got, ref, tol, what):
    bad = ~((got.double() - ref.to(got.device)).abs() <= tol.to(got.device))
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError("%s: %d of %d elements out of bounds, first at %d: got %r, ref %r, tol %r" % (
            what, int(bad.sum()), bad.numel(), i, got[i].item(), ref[i].item(), tol[i].item()))


def check_sgd_step(flat, opt, snap, lr, mu, wd, what="optimizer"):
    """Master weights, momentum and low-precision parameters after one ``FlatSGDMomentum`` step against the float64
    rule applied to the gradient the step left in the bucket, from ``snap = {dtype: (master, momentum)}`` taken before
    the step."""
    for dt, g in flat.groups.items():
        master = g.master if g.master is not None else g.param
        w, v, tw, tv = ref_sgd(*snap[dt], g.grad, lr, mu, wd)
        _assert_close(master, w, tw, "%s master %s" % (what, dt))
        _assert_close(opt.state[dt]["mom"], v, tv, "%s momentum %s" % (what, dt))
        if g.master is not None:
            fb.check_exact(g.param, master.to(g.param.dtype), what="%s parameters %s" % (what, dt))


def check_bf16(out, ref, mag, *args, terms=None, **kw):
    """``fb.check_bf16`` on [rows, channels]; an output of fewer than ``fb.E2E_MIN_ROWS`` rows (the 2 x 2 maps of the
    last stage at 64 x 64, the classifier) is judged on its transpose, per pixel over the channels: over fewer rows the
    per-column yardstick of criterion 2 depends on where a few values fall on the bf16 grid.  Criterion 1 is unchanged;
    row and column indices in messages are then swapped."""
    o, r, g = fb.rows(out), fb.rows(ref), fb.rows(mag)
    if o.shape[0] < fb.E2E_MIN_ROWS <= o.shape[1]:
        o, r, g = o.t(), r.t(), g.t()
        terms = terms and [(fb.rows(a).t(), fb.rows(b).t()) for a, b in terms]
    return fb.check_bf16(o, r, g, *args, terms=terms, **kw)


class _Act:
    """An activation of the step: its recorded gradient and the float64 contributions of its consumers."""

    def __init__(self, name, t):
        self.name, self.t, self.grad = name, t, None
        self.terms = []          # (description, fn() -> (ref, mag, tau, criteria))
        self.keep = None         # callable -> bool mask when the producing BatchNorm stored its gradient premasked

    def hook(self, g):
        self.grad = g.detach().clone()


class StepRecorder:
    def __init__(self, model):
        self.model = model
        self.names = {m: n for n, m in model.named_modules()}
        self.units = [m for m in model.modules() if isinstance(m, ConvBNAct)]
        self._undo = []
        self.reset()

    # ------------------------------------------------------------------------------------------------------ capture
    def reset(self):
        self.acts = {}
        self.convs, self.bns, self.pools = [], [], []
        self.fc = self.loss = None
        self.lib = defaultdict(set)          # weight data_ptr -> passes that ran on the library

    def act(self, t, name):
        """The record of activation ``t`` (created, with its gradient hook, on first sight)."""
        a = self.acts.get(id(t))
        if a is None or a.t is not t:
            a = self.acts[id(t)] = _Act(name, t)
            if t.requires_grad:
                t.register_hook(a.hook)
        return a

    def _patch(self, obj, attr, new):
        old = getattr(obj, attr)
        setattr(obj, attr, new)
        self._undo.append(lambda: setattr(obj, attr, old))
        return old

    def attach(self):
        for u in self.units:
            self._wrap_unit(u)
        rec = self
        orig_lib = self._patch(G, "_count_lib_conv", None)

        def count_lib(x, what, w, stride, groups):
            if x.is_cuda:
                rec.lib[w.data_ptr()].add(what)
            return orig_lib(x, what, w, stride, groups)
        G._count_lib_conv = count_lib
        for name, ref, back, tau_f, tau_b in (
                ("max_pool_3x3_s2", None, None, 0.0, 3 * EPS), ("avg_pool_2x2", fb.avgpool_ref, fb.avgpool_bwd_ref,
                                                               3 * EPS, EPS),
                ("global_avg_pool", fb.gap_ref, fb.gap_bwd_ref, None, 2 * EPS)):
            self._wrap_pool(name, ref, back, tau_f, tau_b)
        orig_ce = self._patch(ops, "soft_cross_entropy", None)

        def ce(logits, target, target_kind="probs", **kw):
            assert not kw, "the oracle's loss reference has default temperatures and no smoothing"
            rec.loss = (rec.act(logits, "logits"), _c(logits), _c(target), target_kind)
            return orig_ce(logits, target, target_kind=target_kind)
        ops.soft_cross_entropy = ce
        h = self.model.register_forward_hook(self._fc_hook)
        self._undo.append(h.remove)
        return self

    def detach(self):
        for f in reversed(self._undo):
            f()
        self._undo = []

    def __enter__(self):
        return self.attach()

    def __exit__(self, *exc):
        self.detach()

    def _wrap_unit(self, u):
        rec, name = self, self.names[u]
        conv = u.conv

        def wrapped(x, want_stats, fork=False):
            out, stats = conv(x, want_stats, fork)
            y, xa = out if fork else (out, None)
            r = dict(name=name, unit=u, x=_c(x), w=_c(u.weight), y=_c(y), stats=_c(stats), ynode=y,
                     kind=type(y.grad_fn).__name__ if y.grad_fn is not None else "", fork=None, dy=rec.act(y, name + " conv"),
                     wptr=u.weight.data_ptr())
            if xa is not None:
                r["fork"] = rec.act(xa, name + " input (forked alias)")
            if x.requires_grad:
                rec.act(x, name + " input").terms.append((name + " dgrad", lambda: rec._dgrad_term(r)))
            rec.convs.append(r)
            return out, stats
        u.conv = wrapped
        self._undo.append(lambda: delattr(u, "conv"))

        def pre(bn, args, kwargs):
            bn._oracle_pre = (_c(bn.running_mean), _c(bn.running_var), _c(bn.weight), _c(bn.bias))

        def post(bn, args, kwargs, out):
            res = kwargs.get("residual")
            sums = kwargs.get("sums")
            if sums is None and bn.ws is not None and bn.ws[0] is not None:
                sums = bn.ws[0]
            rm0, rv0, gamma, beta = bn._oracle_pre
            saved = out.grad_fn.saved_tensors
            b = dict(name=name, bn=bn, x=_c(args[0]), res=_c(res), out=_c(out), ctx=out.grad_fn, sums=_c(sums),
                     conv_sums=kwargs.get("sums") is not None, mean=_c(saved[3]), rstd=_c(saved[4]),
                     saved_y=_c(saved[1]), rm0=rm0, rv0=rv0, gamma=gamma, beta=beta, oact=rec.act(out, name))
            b["oact"].keep = lambda: rec._premasked(b)
            if res is not None:
                rec.act(res, name + " residual").terms.append((name + " bn dres", lambda: rec._dres_term(b)))
            rec.bns.append(b)
        for h in (u.bn.register_forward_pre_hook(pre, with_kwargs=True),
                  u.bn.register_forward_hook(post, with_kwargs=True)):
            self._undo.append(h.remove)

    def _wrap_pool(self, attr, ref, back, tau_f, tau_b):
        rec = self
        orig = self._patch(ops, attr, None)

        def pool(x):
            y = orig(x)
            p = dict(name=attr, x=_c(x), y=_c(y), slots=None, oact=rec.act(y, attr))
            if attr == "max_pool_3x3_s2" and y.grad_fn is not None and y.is_cuda:
                p["slots"] = _c(y.grad_fn.saved_tensors[0]).permute(0, 3, 1, 2)
            p["ref"], p["back"], p["tau_f"], p["tau_b"] = ref, back, tau_f, tau_b
            if x.requires_grad:
                rec.act(x, attr + " input").terms.append((attr + " backward", lambda: rec._pool_term(p)))
            rec.pools.append(p)
            return y
        setattr(ops, attr, pool)

    def _fc_hook(self, model, args, logits):
        fc = model.fc
        gap = self.pools[-1]
        f = dict(name=self.names[fc], x=gap["y"], w=_c(fc.weight), b=_c(fc.bias), logits=_c(logits),
                 oact=self.act(logits, "logits"))
        gap["oact"].terms.append((f["name"] + " dgrad", lambda: self._fc_dgrad_term(f)))
        self.fc = f

    # ------------------------------------------------------------------------------------------- gradient terms
    def _premasked(self, b):
        """The bool keep-mask when the consumer's dgrad epilogue stored this BatchNorm's gradient already masked."""
        ctx = b["ctx"]
        hook = getattr(ctx, "hook", None)
        if b["saved_y"] is not None and b["saved_y"].dtype == torch.uint8 and hook is not None and hook.done:
            return fb.rows(b["out"]) > 0
        return None

    def _dgrad_term(self, r):
        u, w, dy = r["unit"], r["w"], r["dy"].grad
        taps = w.shape[1] * w.shape[2]
        add = r["fork"].grad if r["fork"] is not None else None
        ref, mag = fb.dgrad_ref(dy, w, r["x"].shape, u.stride, (u.k - 1) // 2, add=add)
        k = u.cout * taps * (2 if r["kind"].startswith("_Conv3x3Pair") else 1)
        lib = "dgrad" in self.lib.get(r["wptr"], ())
        return ref, mag, fb.tau(k), (2,) if lib else (1, 2)

    def _dres_term(self, b):
        d = b["oact"].grad
        if b["bn"].relu and self._premasked(b) is None:
            d = d * (b["out"] > 0)
        d = d.double()
        return d, d.abs(), 0.0, (1, 2)

    def _pool_term(self, p):
        dy = p["oact"].grad
        if p["name"] == "max_pool_3x3_s2":
            _, idx = fb.maxpool_ref(p["x"])
            ref, mag = fb.maxpool_bwd_ref(dy, idx, p["x"].shape)
        else:
            ref, mag = p["back"](dy, p["x"].shape)
        return ref, mag, p["tau_b"], (1, 2)

    def _fc_dgrad_term(self, f):
        dy = f["oact"].grad
        ref, mag = fb.gemm_ref(dy, f["w"], b_mn_major=True)
        return ref, mag, fb.tau(f["w"].shape[0]), (1, 2)

    # ---------------------------------------------------------------------------------------------------- checks
    def _grad_of(self, p, name):
        """(gradient, label) of parameter ``p``: its bucket window or ``p.grad``; counted for the coverage check."""
        self._seen[id(p)] = self._seen.get(id(p), 0) + 1
        sink = getattr(p, "_edl_grad_sink", None)
        if sink is not None:
            return sink.view(p.shape), "(bucket)"
        if p.grad is None:
            raise AssertionError("%s: no gradient (neither a bucket window nor .grad)" % name)
        return p.grad, "(grad)"

    def _ratio(self, kind, r):
        c1, c2 = r if isinstance(r, tuple) else (r, None)
        w = self.ratios.setdefault(kind, [0.0, 0.0])
        w[0] = max(w[0], c1 or 0.0)
        w[1] = max(w[1], c2 or 0.0)

    def check(self):
        """Every check; raises AssertionError naming the layer and pass.  Returns ``{"library": [...], "ratios":
        {kind: [c1, c2]}}``."""
        self._seen, self.ratios, library = {}, {}, []
        assert [r["name"] for r in self.convs] == [b["name"] for b in self.bns], "one BatchNorm per convolution"
        # activation gradients first and in the order backward produced them: a wrong one is named where it was
        # produced, not where a later check reads it
        for a in reversed(list(self.acts.values())):
            self._check_act(a)
        for r, b in zip(self.convs, self.bns):
            lib = sorted(self.lib.get(r["wptr"], ()))
            if lib:
                library.append("%s (%s)" % (r["name"], ", ".join(lib)))
            self._check_conv(r, lib)
            self._check_bn(b, r)
        for p in self.pools:
            self._check_pool(p)
        self._check_fc()
        for n, p in self.model.named_parameters():
            if p.requires_grad and self._seen.get(id(p), 0) != 1:
                raise AssertionError("%s: gradient checked %d times (every element exactly once expected)" % (
                    n, self._seen.get(id(p), 0)))
        return {"library": library, "ratios": self.ratios}

    def _check_conv(self, r, lib):
        u, x, w, y, name = r["unit"], r["x"], r["w"], r["y"], r["name"]
        stride, pad = u.stride, (u.k - 1) // 2
        kind = r["kind"]
        cin = w.shape[3]
        k = {"_Conv3x3PairFnBackward": 9 * 64, "_Stem7FnBackward": 160}.get(kind, w.shape[1] * w.shape[2] * cin)
        crit = (2,) if "fprop" in lib else (1, 2)
        self._ratio("conv fprop", check_bf16(y, *fb.conv_ref(x, w, stride, pad), k, what=name + " fprop",
                                                criteria=crit))
        if r["stats"] is not None:
            self._ratio("conv statistics", fb.check_sums(r["stats"], *fb.stats_ref(y), y.numel() // u.cout,
                                                        what=name + " fprop statistics"))
        # weight gradient
        g, where = self._grad_of(u.weight, name + " wgrad")
        dy = r["dy"].grad
        if dy is None:
            raise AssertionError("%s: the convolution's output gradient was never produced" % name)
        n, _, ho, wo = dy.shape
        cout = u.cout
        m = n * ho * wo
        what = "%s wgrad %s" % (name, where)
        if "wgrad" in lib:
            split, crit = 1, (2,)
        else:
            crit = (1, 2)
            if kind == "_Conv1x1FnBackward":
                split = G._split_k_for(cout, cin, m)
            elif kind == "_Conv3x3FnBackward":
                split = G.conv3x3_wgrad_split(n, ho, wo, cin, cout)
            elif kind == "_Conv3x3S2FnBackward":
                split = G.conv3x3_wgrad_split(n, ho, wo, cin, cout, s2=True)
            elif kind == "_Conv1x1S2FnBackward":
                split = G.conv1x1_s2_wgrad_split(n, ho, wo, cin, cout)
            elif kind == "_Stem7FnBackward":
                split = G._split_k_for(cout, 160, m)
            elif kind == "_StemConvFnBackward":
                split = 132
            elif kind in ("_Conv3x3PairFnBackward", "_ConvLibFnBackward") and x.is_cuda:
                # pixel-pair weight gradient (also under a library fprop / dgrad: _pair_wgrad_ok)
                split = G.conv3x3_wgrad_split(n, ho, wo // 2, 64, 2 * cout) + 1
                self._ratio("pair wgrad", fb.check_pair_wgrad(g, x, dy, tuple(w.shape), m // 2, split, what=what))
                return
            else:                            # the CPU paths: fp32 library kernels, held to the bf16 bounds
                split = 1
        ref, mag = fb.wgrad_ref(x, dy, tuple(w.shape), stride, pad)
        self._ratio("wgrad", check_bf16(g.reshape(cout, -1), ref.reshape(cout, -1), mag.reshape(cout, -1), m, split,
                                           what=what, criteria=crit))

    def _check_bn(self, b, r):
        bn, x, out, name = b["bn"], b["x"], b["out"], b["name"] + " bn"
        c = bn.num_features
        m = x.numel() // c
        mean, rstd, gamma, beta = b["mean"], b["rstd"], b["gamma"], b["beta"]
        self._ratio("bn y", check_bf16(out, *fb.bn_y_ref(x, mean, rstd, gamma, beta, b["res"], bn.relu),
                                          tau=fb.BN_Y_TAU, what=name + " y"))
        running = (b["rm0"], b["rv0"], bn.running_mean, bn.running_var, bn.momentum)
        if b["sums"] is not None:
            if not b["conv_sums"]:
                self._ratio("bn statistics", fb.check_sums(b["sums"], *fb.stats_ref(x), m, tau_s=bn_tau(m, c),
                                                           what=name + " statistics"))
            fb.check_bn_saved_stats(b["sums"], mean, rstd, m, bn.eps, what=name, running=running)
        else:
            fb.check_bn_stats_e2e(x, mean, rstd, bn.eps, bn_tau(m, c), what=name)
            fb.check_bn_running_e2e(x, *running, bn_tau(m, c), what=name)
        sv = b["saved_y"]
        if sv is not None and sv.dtype == torch.uint8:
            fb.check_exact(sv, fb.mask_bits(fb.rows(out) > 0), what=name + " ReLU mask bits")
        # backward: the reduction (fused into the consumer's dgrad epilogue or the BatchNorm's own kernel)
        d = b["oact"].grad
        if d is None:
            raise AssertionError("%s: its output gradient was never produced" % name)
        keep = self._premasked(b)
        ctx = b["ctx"]
        hook = getattr(ctx, "hook", None)
        fused_epi = hook is not None and hook.done
        ref, mag, extra = fb.bn_dsums_ref(d, x, mean, rstd, gamma, beta, bn.relu,
                                          y=out if (bn.relu and keep is None) else None,
                                          mask=keep if keep is not None else None)
        tau_s = (128 + math.ceil(m / fb.TILE)) * EPS if fused_epi else bn_tau(m, c)
        gg, where = self._grad_of(bn.weight, name + " dgamma")
        gb, _ = self._grad_of(bn.bias, name + " dbeta")
        self._ratio("bn dgamma / dbeta", fb.check_sums(gg, ref[c:], mag[c:], m, extra=extra[c:], tau_s=tau_s,
                                                       what="%s dgamma %s" % (name, where)))
        self._ratio("bn dgamma / dbeta", fb.check_sums(gb, ref[:c], mag[:c], m, extra=extra[:c], tau_s=tau_s,
                                                       what="%s dbeta %s" % (name, where)))
        dx = r["dy"].grad
        kx = (fb.rows(out) > 0) if (bn.relu and keep is None) else None
        dref, dmag = fb.bn_dx_ref(d, x, mean, rstd, gamma, ref, m, keep=kx, dsums_err=tau_s * mag + extra)
        self._ratio("bn dx", check_bf16(fb.rows(dx), dref, dmag, tau=fb.BN_DX_TAU, what=name + " dx"))

    def _check_pool(self, p):
        x, y, name = p["x"], p["y"], p["name"]
        if name == "max_pool_3x3_s2":
            if p["slots"] is not None:
                fb.check_maxpool(y, p["slots"], x, what=name)
            else:
                fb.check_exact(y.double(), fb.maxpool_ref(x)[0], what=name + " y")
            return
        tau = p["tau_f"] if p["tau_f"] is not None else fb.gap_tau(x.shape[2] * x.shape[3])
        ref, mag = p["ref"](x)
        self._ratio("pools", check_bf16(y, ref, mag, tau=tau, what=name + " forward"))

    def _check_fc(self):
        f = self.fc
        name = f["name"]
        x, w, b = f["x"], f["w"], f["b"]
        self._ratio("fc", check_bf16(f["logits"], *fb.gemm_ref(x, w, shift=b.float()), w.shape[1],
                                        what=name + " forward"))
        _, z, t, kind = self.loss
        dz = f["oact"].grad
        self._ratio("logits gradient", (check_logits_grad(dz, ref_soft_ce_grad(z, t, kind), "loss backward (logits "
                                                                                            "gradient)"), None))
        gw, where = self._grad_of(self.model.fc.weight, name + " wgrad")
        n = dz.shape[0]
        split = G._split_k_for(w.shape[0], w.shape[1], n) if dz.is_cuda else 1
        self._ratio("wgrad", check_bf16(gw, *fb.gemm_ref(dz, x, a_mn_major=True, b_mn_major=True), n, split,
                                           what="%s wgrad %s" % (name, where)))
        gb, where = self._grad_of(self.model.fc.bias, name + " bias gradient")
        d64 = dz.double()
        self._ratio("fc bias gradient", fb.check_sums(gb, d64.sum(0), d64.abs().sum(0), n,
                                                      what="%s bias gradient %s" % (name, where)))

    def _check_act(self, a):
        if not a.terms:
            return
        if a.grad is None:
            raise AssertionError("%s: its gradient was never produced" % a.name)
        parts = [(desc, *fn()) for desc, fn in a.terms]
        ref = sum(p[1] for p in parts)
        mag = sum(p[2] for p in parts)
        tau = max(p[3] for p in parts)
        crit = (2,) if any(p[4] == (2,) for p in parts) else (1, 2)
        keep = a.keep() if a.keep is not None else None
        if keep is not None:
            ref, mag = [torch.where(keep, fb.rows(t), torch.zeros_like(fb.rows(t))) for t in (ref, mag)]
        what = parts[0][0] if len(parts) == 1 else "%s gradient (%s)" % (a.name, " + ".join(p[0] for p in parts))
        if len(parts) == 1 and tau == 0.0:
            fb.check_exact(fb.rows(a.grad).double(), fb.rows(ref), what=what)
            return
        terms = [(p[1], p[2]) for p in parts] if len(parts) > 1 else None
        kind = "dgrad" if all(p[0].endswith("dgrad") for p in parts) else "activation gradients (sums, pools)"
        self._ratio(kind, check_bf16(fb.rows(a.grad), fb.rows(ref), fb.rows(mag), tau=tau, what=what,
                                        terms=terms and [(fb.rows(r), fb.rows(g)) for r, g in terms], criteria=crit))
