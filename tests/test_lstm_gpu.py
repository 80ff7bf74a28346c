"""The bidirectional LSTM recurrence kernels (csrc/lstm.cu) and the BiLSTM student on the GPU.

Per-step exact-operand bounds: every saved c_t, h_t and gate of the forward, and every dgates_t of the backward, is
checked against float64 recomputed from the kernel's own inputs to that step (the stored bf16 h_{t-1}, the saved
fp32 c_{t-1}, the bf16 xproj row and W_hh, the kernel's bf16 dgates_{t+1}), so the bound does not compound over time.
The bound is derived, not fitted:

* fp32 accumulation of the wgmma: ``tau(K) * mag`` (tests/f64_bounds.py), K = H = 128 forward, K = 4H = 512 backward;
* the activation intrinsics: sigma(x) = __fdividef(1, 1 + __expf(-x)).  The CUDA C Programming Guide gives __expf
  within 2 + floor(|1.173 x|) ulp and __fdividef within 2 ulp; with the fp32 add that is an absolute error of at most
  ``eps_sig(x) = (2 + 1.173 |x|) 2^-23 + 2^-24 + 2^-22`` (sigma <= 1).  tanh(x) = 2 sigma(2x) - 1 adds one rounding
  of a value <= 1: ``eps_tanh(x) = 2 eps_sig(2x) + 2^-24``;
* propagation through the gate derivatives: |sigma'| <= 1/4, |tanh'| <= 1;
* fp32 rounding of the few products and sums of the cell update (2^-23 per operation on the magnitudes), and one
  bf16 rounding (1/2 ulp) of every stored bf16 value.
End to end, outputs and gradients are compared with float64 nn.LSTM on the same bf16-rounded inputs and weights."""
import os
import re
import subprocess
import sys

import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from edl_b200 import ops  # noqa: E402
from edl_b200.models.small import BiLSTM  # noqa: E402
from edl_b200.ops import rnn  # noqa: E402
from f64_bounds import guarded, tau, ulp  # noqa: E402

DEV = torch.device("cuda", 0)
H = 128
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E23, E24 = 2.0 ** -23, 2.0 ** -24


def _log(line):
    """Append a measured error / bound line to the file named by EDL_F64_BOUNDS_LOG (as tests/f64_bounds.py does)."""
    path = os.environ.get("EDL_F64_BOUNDS_LOG")
    if path:
        with open(path, "a") as f:
            f.write(line + "\n")


def _params(seed, e, dtype=torch.float32, scale=1.0):
    torch.manual_seed(seed)
    m = torch.nn.LSTM(e, H, batch_first=True, bidirectional=True)
    ps = [p.detach().to(torch.bfloat16).to(dtype) * scale for p in m.parameters()]
    return ps


def _lengths(b, L, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, L + 1, (b,), generator=g)
    for i, v in enumerate((L, 0, 1)):                            # a batch of one gets L
        if i < b:
            lens[(i * 7) % b] = v
    return lens


def eps_sig(x):
    return (2 + 1.173 * x.abs()) * E23 + E24 + 2 * E23


def eps_tanh(x):
    return 2 * eps_sig(2 * x) + E24


def hb(x):
    """1/2 ulp of bf16 at |x| (float64)"""
    return 0.5 * ulp(x.abs(), 8)


# ------------------------------------------------------------------------------------------- per-step exact operands
def _run_guarded(x, lengths, params, dy, dhn):
    """Both kernels on operands copied into NaN-guarded buffers and outputs inside sentinel-filled buffers."""
    b, L, e = x.shape
    hs0, hn0, g0, cs0, xt, len32, whh0, xproj0 = rnn.lstm_forward_saved(x, lengths, params)
    gx = guarded((L * b, 8 * H), pad_rows=8, values=xproj0)
    gw = guarded((2 * 4 * H, H), pad_rows=8, values=whh0.view(-1, H))
    gl = guarded((b,), pad_rows=8, fill=-5, dtype=torch.int32, values=len32)
    ghs = guarded(((L + 2) * b, 2 * H), pad_rows=8, fill=3.0)
    ghn = guarded((2 * b, H), pad_rows=8, fill=3.0)
    gg = guarded((L * b, 8 * H), pad_rows=8, fill=3.0)
    gc = guarded((L * b, 2 * H), pad_rows=8, fill=3.0, dtype=torch.float32)
    whh = gw.t.view(2, 4 * H, H)
    C = ops.native()
    C.lstm_fwd(gx.t, whh, gl.t, ghs.t, ghn.t.view(2, b, H), gg.t.view(L * b, 2, H, 4), gc.t.view(L * b, 2, H), L)
    gdy = guarded((b * L, 2 * H), pad_rows=8, values=dy.reshape(b * L, 2 * H))
    gdh = guarded((2 * b, H), pad_rows=8, values=dhn.reshape(2 * b, H))
    gdg = guarded((L * b, 8 * H), pad_rows=8, fill=3.0)
    C.lstm_bwd(whh, gl.t, gg.t.view(L * b, 2, H, 4), gc.t.view(L * b, 2, H), gdy.t.view(b, L, 2 * H),
               gdh.t.view(2, b, H), gdg.t, L)
    torch.cuda.synchronize()
    for g, what in ((gx, "xproj"), (gw, "whh"), (gl, "lengths"), (ghs, "hs"), (ghn, "hn"), (gg, "gates"), (gc, "cs"),
                    (gdy, "dy"), (gdh, "dhn"), (gdg, "dgates")):
        g.assert_untouched(what)
    # the guarded run computes what the op's own buffers hold
    assert torch.equal(ghs.t, hs0) and torch.equal(ghn.t.view(2, b, H), hn0)
    return dict(xproj=gx.t, whh=whh, hs=ghs.t, hn=ghn.t.view(2, b, H), gates=gg.t.view(L * b, 2, H, 4),
                cs=gc.t.view(L * b, 2, H), dgates=gdg.t)


def _check(got, want, bound, what):
    err = (got.double() - want).abs()
    bad = ~(err <= bound)
    _log("%s: max err %.3e, max err / bound %.3f" % (what, float(err.max()), float((err / bound).max())))
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError("%s: %d elements outside the bound, first at %s: got %r, want %r, bound %r" % (
            what, int(bad.sum()), i, float(got.double()[tuple(i)]), float(want[tuple(i)]), float(bound[tuple(i)])))


@pytest.mark.parametrize("B,L,E", [(65, 23, 64), (3, 9, 200)])
def test_per_step_exact_operand_bounds(B, L, E):
    torch.manual_seed(B + L)
    params = [p.to(DEV) for p in _params(11, E, scale=2.0)]     # larger weights: saturating gates are exercised too
    x = torch.randn(B, L, E, device=DEV).to(torch.bfloat16)
    lengths = _lengths(B, L, B * L).to(DEV)
    dy = (torch.randn(B, L, 2 * H, device=DEV) * 0.5).to(torch.bfloat16)
    dhn = torch.randn(2, B, H, device=DEV).to(torch.bfloat16)
    o = _run_guarded(x, lengths, params, dy, dhn)
    perm = rnn._thread_order(H, DEV)
    lens = lengths.clamp(0, L).long()
    xp = o["xproj"].double().view(L, B, 8 * H)
    hs = o["hs"].double().view(L + 2, B, 2 * H)
    cs = o["cs"].double().view(L, B, 2, H)
    gates = o["gates"].double().view(L, B, 2, H, 4)
    dg = o["dgates"].double().view(L, B, 8 * H)
    ar = torch.arange(B, device=DEV)
    for d in range(2):
        W = o["whh"][d].double()                                  # [4H, H] nn.LSTM order
        xnat = torch.empty(L, B, 4 * H, dtype=torch.float64, device=DEV)
        xnat[:, :, perm] = xp[:, :, 4 * H * d:4 * H * (d + 1)]
        # ---- forward, step by step from the kernel's own operands
        for s in range(L):
            act = s < lens
            if not act.any():
                break
            t = (torch.full_like(lens, s) if d == 0 else (lens - 1 - s)).clamp(0, L - 1)
            tp = t - 1 if d == 0 else t + 1                       # the previous step's time
            hprev = hs[tp + 1, ar, H * d:H * (d + 1)]             # zero blocks at 0 and L + 1
            cprev = cs[tp.clamp(0, L - 1), ar, d] if s > 0 else torch.zeros(B, H, dtype=torch.float64, device=DEV)
            xr = xnat[t, ar]
            pre = xr + hprev @ W.t()
            dpre = tau(H) * (xr.abs() + hprev.abs() @ W.abs().t())
            pi, pf, pg, po = pre.split(H, 1)
            qi, qf, qg, qo = dpre.split(H, 1)
            i, f, g, og = torch.sigmoid(pi), torch.sigmoid(pf), torch.tanh(pg), torch.sigmoid(po)
            di, df, dgg, do = (qi / 4 + eps_sig(pi), qf / 4 + eps_sig(pf), qg + eps_tanh(pg), qo / 4 + eps_sig(po))
            c = f * cprev + i * g
            dc = df * cprev.abs() + di * g.abs() + dgg * i.abs() + df * di + di * dgg \
                + 3 * E23 * (f.abs() * cprev.abs() + i.abs() * g.abs())
            kc = cs[t, ar, d]
            a = act.unsqueeze(1)
            sel = lambda v: v[a.expand_as(v)]                      # noqa: E731
            _check(sel(kc), sel(c), sel(dc * (1 + 2 ** -10)), "c_t d%d s%d" % (d, s))
            kg = gates[t, ar, d]
            for k, (want, dw) in enumerate(((i, di), (f, df), (g, dgg), (og, do))):
                _check(sel(kg[..., k]), sel(want), sel(dw * (1 + 2 ** -10) + hb(want + dw)), "gate%d d%d s%d" % (k, d, s))
            # h_t from the kernel's own c_t: o * tanh(c_t), one fp32 product, one bf16 rounding
            hw = og * torch.tanh(kc)
            dh = do + og * eps_tanh(kc) + E23 * hw.abs()
            kh = hs[t + 1, ar, H * d:H * (d + 1)]
            _check(sel(kh), sel(hw), sel(dh * (1 + 2 ** -10) + hb(hw.abs() + dh)), "h_t d%d s%d" % (d, s))
            last = a & (s == lens - 1).unsqueeze(1)
            if last.any():
                assert torch.equal(o["hn"][d][last.expand(-1, H)], o["hs"].view(L + 2, B, 2 * H)[t + 1, ar, H * d:H * (d + 1)][last.expand(-1, H)])
        # ---- backward, from the kernel's dgates_{t+1}; the carried dc is propagated in float64 with its bound
        dcc = torch.zeros(B, H, dtype=torch.float64, device=DEV)
        ddcc = torch.zeros_like(dcc)
        for s in range(L - 1, -1, -1):
            act = s < lens
            a = act.unsqueeze(1)
            t = (torch.full_like(lens, s) if d == 0 else (lens - 1 - s)).clamp(0, L - 1)
            tn = t + 1 if d == 0 else t - 1                       # time of step s + 1
            nxt = (s + 1 < lens).unsqueeze(1)
            dgn = torch.where(nxt, dg[tn.clamp(0, L - 1), ar, 4 * H * d:4 * H * (d + 1)], torch.zeros(B, 4 * H, dtype=torch.float64, device=DEV))
            ext = dy.double()[ar, t, H * d:H * (d + 1)] + torch.where((s == lens - 1).unsqueeze(1), dhn.double()[d], torch.zeros_like(dcc))
            dh = ext + dgn @ W
            ddh = tau(4 * H) * (dgn.abs() @ W.abs()) + 2 * E23 * (ext.abs() + (dgn.abs() @ W.abs()))
            gv = gates[t, ar, d]
            i, f, g, og = gv[..., 0], gv[..., 1], gv[..., 2], gv[..., 3]
            kc = cs[t, ar, d]
            cprev = cs[(t - 1 if d == 0 else t + 1).clamp(0, L - 1), ar, d] if s > 0 else torch.zeros_like(kc)
            tc = torch.tanh(kc)
            etc = eps_tanh(kc)
            dct = dh * og * (1 - tc * tc)
            dc = dct + dcc
            ddc = (ddh * og * (1 - tc * tc) + dh.abs() * og * (2 * tc.abs() * etc + etc * etc) + ddcc
                   + 4 * E23 * (dct.abs() + dcc.abs()) + 2 * E23 * (dh * og).abs())      # (1 - tc^2): 2^-23 absolute
            want = [dc * g * i * (1 - i), dc * cprev * f * (1 - f), dc * i * (1 - g * g), dh * tc * og * (1 - og)]
            dwant = [ddc * (g * i * (1 - i)).abs() + 4 * E23 * want[0].abs(),
                     ddc * (cprev * f * (1 - f)).abs() + 4 * E23 * want[1].abs(),
                     ddc * (i * (1 - g * g)).abs() + 4 * E23 * want[2].abs() + 2 * E23 * (dc * i).abs(),
                     ddh * (og * (1 - og)).abs() * tc.abs() + dh.abs() * etc * (og * (1 - og)).abs() + 4 * E23 * want[3].abs()]
            kd = dg[t, ar, 4 * H * d:4 * H * (d + 1)].view(B, 4, H)
            sel = lambda v: v[a.expand_as(v)]                      # noqa: E731
            for k in range(4):
                _check(sel(kd[:, k]), sel(want[k]), sel(dwant[k] * (1 + 2 ** -10) + hb(want[k].abs() + dwant[k])),
                       "dgates%d d%d s%d" % (k, d, s))
            dcc = torch.where(a, dc * f, torch.zeros_like(dc))
            ddcc = torch.where(a, ddc * f + E23 * (dc * f).abs(), torch.zeros_like(dc))
    # padded positions: zero h and dgates
    tt = torch.arange(L, device=DEV).unsqueeze(1)
    pad = (tt >= lens.unsqueeze(0))                               # [L, B]
    assert (hs[1:L + 1][pad] == 0).all() and (hs[0] == 0).all() and (hs[L + 1] == 0).all()
    assert (dg[pad] == 0).all()
    z = lens == 0
    assert (o["hn"][:, z] == 0).all()


# ---------------------------------------------------------------------------------------------------------- end to end
def _torch_f64(x, lengths, params):
    """float64 nn.LSTM over pack_padded_sequence on the samples with length >= 1; zeros for the others."""
    b, L, e = x.shape
    m = torch.nn.LSTM(e, H, batch_first=True, bidirectional=True).to(DEV, torch.float64)
    with torch.no_grad():
        for p, v in zip(m.parameters(), params):
            p.copy_(v.double())
    x64 = x.double().requires_grad_(True)
    nz = (lengths > 0).nonzero().flatten()
    y = torch.zeros(b, L, 2 * H, dtype=torch.float64, device=DEV)
    hn = torch.zeros(2, b, H, dtype=torch.float64, device=DEV)
    if nz.numel():
        packed = pack_padded_sequence(x64[nz], lengths[nz].cpu(), batch_first=True, enforce_sorted=False)
        out, (h, _) = m(packed)
        yy, _ = pad_packed_sequence(out, batch_first=True, total_length=L)
        y = y.index_copy(0, nz, yy)
        hn = hn.index_copy(1, nz, h)
    return m, x64, y, hn


E2E = [(1, 1, 64), (63, 2, 128), (64, 64, 200), (65, 129, 64), (200, 64, 128), (1, 129, 200), (200, 2, 64),
       (64, 1, 128), (65, 64, 200)]


@pytest.mark.parametrize("B,L,E", E2E)
def test_end_to_end_vs_float64_nn_lstm(B, L, E):
    ops.reset_fallbacks()
    params = [p.to(DEV) for p in _params(B + L + E, E)]
    x = torch.randn(B, L, E, device=DEV).to(torch.bfloat16)
    lengths = _lengths(B, L, B * 1000 + L).to(DEV)
    m, x64, y_ref, hn_ref = _torch_f64(x, lengths, params)
    wy = torch.randn(B, L, 2 * H, device=DEV, dtype=torch.float64).to(torch.bfloat16).double()
    wh = torch.randn(2, B, H, device=DEV, dtype=torch.float64).to(torch.bfloat16).double()
    ((y_ref * wy).sum() + (hn_ref * wh).sum()).backward()

    xk = x.clone().requires_grad_(True)
    pk = [p.clone().requires_grad_(True) for p in params]
    y, hn = ops.lstm(xk, lengths, pk)
    torch.autograd.backward([y, hn], [wy.to(torch.bfloat16).expand_as(y), wh.to(torch.bfloat16)])
    assert ops.fallbacks() == {}
    # Tolerance.  Every step rounds h to bf16 (2^-9 relative) before it re-enters the recurrence, and the saved gates
    # and dgates are bf16: one step contributes a few bf16 roundings of values of magnitude <= 1.  With nn.LSTM's
    # initialisation (|w| <= 1/sqrt(H)) the recurrence is contractive, so these do not grow with L: outputs within
    # 8 bf16 half-ulps of 1 (2^-6) element-wise; gradients, sums over B * L of such products, within 2^-6 of their
    # norm (normwise) and element-wise within 2^-6 of the largest entry of the tensor.
    _log("e2e B%d L%d E%d: y %.3e hn %.3e" % (B, L, E, float((y.double() - y_ref).abs().max()),
                                             float((hn.double() - hn_ref).abs().max())))
    assert (y.double() - y_ref).abs().max() <= 2 ** -6
    assert (hn.double() - hn_ref).abs().max() <= 2 ** -6
    grads = [(xk.grad, x64.grad, "dX")] + [(p.grad, q.grad, n) for p, (n, q) in zip(pk, m.named_parameters())]
    for got, want, what in grads:
        assert got.dtype == torch.float32 or what == "dX"
        err = (got.double() - want)
        rel = float(err.norm() / want.norm().clamp_min(1e-30))
        mx = float(err.abs().max() / want.abs().max().clamp_min(1e-30))
        _log("e2e B%d L%d E%d %s: normwise %.3e, max/max %.3e" % (B, L, E, what, rel, mx))
        assert rel <= 2 ** -6 and mx <= 2 ** -6, (what, rel, mx)
    # zero-length samples: zero outputs, zero input gradient; padded rows of dX are zero
    tt = torch.arange(L, device=DEV)
    pad = tt.unsqueeze(0) >= lengths.unsqueeze(1)
    assert (y[pad] == 0).all() and (xk.grad[pad] == 0).all()
    assert (hn[:, lengths == 0] == 0).all()


# ------------------------------------------------------------------------------------------------ isolation, determinism
def _fwd_bwd(x, lengths, params, wy, wh):
    xk = x.clone().requires_grad_(True)
    pk = [p.clone().requires_grad_(True) for p in params]
    y, hn = ops.lstm(xk, lengths, pk)
    torch.autograd.backward([y, hn], [wy, wh])
    return y.detach().clone(), hn.detach().clone(), xk.grad, [p.grad for p in pk]


def test_isolation_and_determinism():
    B, L, E = 70, 40, 128
    params = [p.to(DEV) for p in _params(5, E)]
    x = torch.randn(B, L, E, device=DEV).to(torch.bfloat16)
    lengths = _lengths(B, L, 77).to(DEV)
    wy = torch.randn(B, L, 2 * H, device=DEV).to(torch.bfloat16)
    wh = torch.randn(2, B, H, device=DEV).to(torch.bfloat16)
    pad = torch.arange(L, device=DEV).unsqueeze(0) >= lengths.unsqueeze(1)
    wy = wy.masked_fill(pad.unsqueeze(2), 0)
    base = _fwd_bwd(x, lengths, params, wy, wh)
    again = _fwd_bwd(x, lengths, params, wy, wh)
    for a, b in zip(base[:3] + tuple(base[3]), again[:3] + tuple(again[3])):
        assert torch.equal(a, b)                                  # bitwise deterministic
    # NaN in padded rows and in every row of sample 5: no forward output bit of another sample changes
    xn = x.clone()
    xn[pad] = float("nan")
    xn[5] = float("nan")
    with torch.no_grad():
        y, hn = ops.lstm(xn, lengths, params)
    keep = torch.ones(B, dtype=torch.bool, device=DEV)
    keep[5] = False
    assert torch.equal(y[keep], base[0][keep]) and torch.equal(hn[:, keep], base[1][:, keep])
    # arbitrary finite values in padded rows: every gradient bit unchanged; padded rows of dX are zero
    xf = x.clone()
    xf[pad] = torch.randn(int(pad.sum()), E, device=DEV).to(torch.bfloat16) * 100
    other = _fwd_bwd(xf, lengths, params, wy, wh)
    assert torch.equal(other[2], base[2])
    for a, b in zip(other[3], base[3]):
        assert torch.equal(a, b)
    assert (base[2][pad] == 0).all()


def test_bilstm_train_step_cuda_graph_matches_eager():
    torch.manual_seed(0)
    model = BiLSTM(vocab_size=1000).to(DEV)
    opt = torch.optim.Adam(model.parameters(), 1e-3, capturable=True)
    ids = torch.randint(1, 1000, (96, 48), device=DEV)
    ids[torch.arange(48, device=DEV).unsqueeze(0) >= torch.randint(1, 49, (96, 1), device=DEV)] = 0
    label = torch.randint(0, 2, (96,), device=DEV)

    def step():
        opt.zero_grad(set_to_none=False)
        loss = torch.nn.functional.cross_entropy(model(ids), label)
        loss.backward()
        opt.step()
        return loss

    ops.reset_fallbacks()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    state = ({k: v.clone() for k, v in model.state_dict().items()},
             [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in s.items()} for s in opt.state.values()])

    def restore():
        with torch.no_grad():
            for k, v in model.state_dict().items():
                v.copy_(state[0][k])
            for s, s0 in zip(opt.state.values(), state[1]):
                for k, v in s.items():
                    if torch.is_tensor(v):
                        v.copy_(s0[k])

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gl = step()
    restore()
    el = step().clone()
    eager = {k: v.clone() for k, v in model.state_dict().items()}
    restore()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gl, el)
    for k, v in model.state_dict().items():
        assert torch.equal(v, eager[k]), k
    assert ops.fallbacks() == {}


def test_distill_example_lstm_on_gpu():
    p = subprocess.run([sys.executable, "examples/distill/nlp/distill.py", "--model", "lstm", "--epochs", "2",
                        "--vocab", "400"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600,
                       text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", p.stdout)]
    assert len(losses) >= 4 and min(losses[-2:]) < losses[0], p.stdout
