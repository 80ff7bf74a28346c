"""Transformer student on the GPU: float64 bounds for the new kernels (attention backward, LayerNorm and
embedding-LayerNorm backward, both GELU training epilogues), unchanged inference, and whole training steps of
ErnieStudent (against float32 torch, bitwise reproducible, CUDA-graph replay, no library fallback).

Every float64 reference is built from exactly the bf16 / fp32 tensors the kernel read.  ``mag`` is the same expression
over absolute values, the scale of the rounding errors.  The bounds:
  attention dQ / dK / dV   |out - ref| <= 2^-8 |ref| + 2^-6 mag: the recomputed P carries the forward's row sum over
                           bf16-rounded probabilities (relative 2^-9 per term), P and dS are rounded to bf16 before their
                           second products (2^-9 each), D is formed from the stored bf16 O, and the result is stored bf16;
                           2^-6 covers those four relative errors with a factor of two to spare
  LayerNorm dx, dE         |out - ref| <= 2^-8 |ref| (bf16 store; 0 for fp32 dE) + 2^-16 mag (fp32 row sums of <= 1024)
  dgamma / dbeta, tables   |out - ref| <= 2^-12 sum |terms|: fp32 chains of up to a few thousand terms (rows of a warp,
                           warps, CTA partials; the library's segment sum over repeated ids)
  GELU epilogues           u: 2^-8 |ref| + 2^-20 mag; y: bitwise the inference epilogue's; dU: 2^-8 |ref| + 2^-16 mag
                           with mag = sum |dy w| (|gelu'(u)| + 1)."""
import os
import re
import subprocess
import sys

import pytest
import torch

from edl_b200 import ops
from edl_b200.models.ernie import ErnieStudent
from student_oracle import attention_f64, ln_f64
from test_ernie_student_cpu import _functional_encoder

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _check(out, ref, bound, what):
    out = out.double()
    assert torch.isfinite(out).all(), what + ": non-finite output"
    err = (out - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    assert (err <= bound).all(), "%s: worst error / bound %.3f" % (what, ratio)
    return ratio


@pytest.mark.parametrize("L", [1, 63, 64, 65, 128, 200, 512])
def test_attention_backward_f64_bounds(L):
    torch.manual_seed(L)
    b, h = 4, 2
    qkv = (torch.randn(b * L, 3 * h * 64, device=DEV) * 1.5).to(torch.bfloat16)
    mask = (torch.rand(b, L, device=DEV) > 0.3).to(torch.uint8)
    mask[0] = 0                                                       # a fully masked sample
    mask[1, 0] = 0                                                    # token 0 masked
    mask[2] = 1
    do = torch.randn(b * L, h * 64, device=DEV).to(torch.bfloat16)
    out, lse = ops.transformer.attention_forward_saved(qkv, mask, b, L, h)
    assert torch.equal(out, ops.attention(qkv, mask, b, L, h))        # O bitwise unchanged by the saved statistics
    dqkv = ops.transformer.attention_backward(qkv, mask, out, lse, do, b, L, h)
    _, _, ref, mag = attention_f64(qkv, mask, do, b, L, h)
    _check(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, "attention dqkv L=%d" % L)
    has = (mask != 0).any(1)                                               # at L = 1 sample 1 has no valid key either
    assert (dqkv.view(b, L, -1)[~has] == 0).all()                     # no valid key: exactly zero gradients
    assert torch.isinf(lse[~has]).all() and torch.isfinite(lse[has]).all()
    again = ops.transformer.attention_backward(qkv, mask, out, lse, do, b, L, h)
    assert torch.equal(again, dqkv)


def test_attention_backward_negative_control():
    """A swapped key pair in the input the reference sees must break the bound."""
    torch.manual_seed(1)
    b, L, h = 2, 96, 2
    qkv = torch.randn(b * L, 3 * h * 64, device=DEV).to(torch.bfloat16)
    mask = torch.ones(b, L, device=DEV, dtype=torch.uint8)
    do = torch.randn(b * L, h * 64, device=DEV).to(torch.bfloat16)
    out, lse = ops.transformer.attention_forward_saved(qkv, mask, b, L, h)
    dqkv = ops.transformer.attention_backward(qkv, mask, out, lse, do, b, L, h)
    bad = qkv.clone()
    bad[[3, 70]] = bad[[70, 3]]
    _, _, ref, mag = attention_f64(bad, mask, do, b, L, h)
    with pytest.raises(AssertionError):
        _check(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, "control")


@pytest.mark.parametrize("rows,C", [(1, 384), (77, 384), (4096, 384), (300, 1024), (33, 8), (2000, 136)])
def test_layernorm_backward_f64_bounds(rows, C):
    torch.manual_seed(rows + C)
    x = (torch.randn(rows, C, device=DEV) * 2 + 0.5).to(torch.bfloat16)
    dy = torch.randn(rows, C, device=DEV).to(torch.bfloat16)
    gamma = torch.randn(C, device=DEV)
    beta = torch.randn(C, device=DEV)
    xr = x.clone().requires_grad_(True)
    g, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    y = ops.layer_norm_trainable(xr, g, bt, 1e-12)
    assert torch.equal(y, ops.layer_norm(x, gamma, beta, 1e-12))
    y.backward(dy)
    _, dx, mag, dg, mg, db, mb = ln_f64(x, dy, gamma, 1e-12)
    _check(xr.grad, dx, 2.0 ** -8 * dx.abs() + 2.0 ** -16 * mag, "LayerNorm dx")
    _check(g.grad, dg, 2.0 ** -12 * mg, "dgamma")
    _check(bt.grad, db, 2.0 ** -12 * mb, "dbeta")


@pytest.mark.parametrize("rows,C", [(5, 384), (4096, 384), (700, 768)])
def test_embedding_layernorm_backward_f64_bounds(rows, C):
    torch.manual_seed(rows)
    word = torch.randn(500, C, device=DEV) * 0.5
    pos = torch.randn(130, C, device=DEV) * 0.5
    seg = torch.randn(2, C, device=DEV) * 0.5
    gamma, beta = torch.randn(C, device=DEV), torch.randn(C, device=DEV)
    ids = torch.randint(0, 500, (rows,), device=DEV)
    ids[: rows // 2] = 7                                              # a repeated row: summed table gradient
    pid, sid = torch.randint(0, 130, (rows,), device=DEV), torch.randint(0, 2, (rows,), device=DEV)
    ps = [t.clone().requires_grad_(True) for t in (word, pos, seg, gamma, beta)]
    y = ops.embedding_layernorm_trainable(ids, pid, sid, *ps, 1e-12)
    dy = torch.randn_like(y.float()).to(torch.bfloat16)
    y.backward(dy)
    tb = [t.to(torch.bfloat16) for t in (word, pos, seg)]
    x = tb[0].double()[ids] + tb[1].double()[pid] + tb[2].double()[sid]
    _, dE, mag, dg, mg, db, mb = ln_f64(x, dy, gamma, 1e-12)
    for t, idx, n, what in ((ps[0], ids, 500, "word"), (ps[1], pid, 130, "pos"), (ps[2], sid, 2, "seg")):
        ref = torch.zeros(n, C, device=DEV, dtype=torch.float64).index_add_(0, idx, dE)
        m = torch.zeros(n, C, device=DEV, dtype=torch.float64).index_add_(0, idx, mag + dE.abs())
        _check(t.grad, ref, 2.0 ** -12 * m, "embedding table " + what)
    _check(ps[3].grad, dg, 2.0 ** -12 * mg, "dgamma")
    _check(ps[4].grad, db, 2.0 ** -12 * mb, "dbeta")


@pytest.mark.parametrize("M,N,K", [(1, 64, 64), (129, 1536, 384), (4096, 1536, 384), (300, 200, 136)])
def test_gelu_epilogues_f64_bounds(M, N, K):
    torch.manual_seed(M + N)
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, device=DEV) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV)
    y, u = ops.gemm_bf16_gelu_train(x, w, bias)
    assert torch.equal(y, ops.gemm_bf16(x, w, col_shift=bias, gelu=True))   # y is the inference epilogue's
    ref = x.double() @ w.double().t() + bias.double()
    _check(u, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -20 * (x.double().abs() @ w.double().abs().t() + bias.double().abs()),
           "u")
    # FFN2's dgrad through gelu': dU = (dY W2) * gelu'(u), W2 [N2, N]
    n2 = 256
    dy = torch.randn(M, n2, device=DEV).to(torch.bfloat16)
    w2 = (torch.randn(n2, N, device=DEV) / n2 ** 0.5).to(torch.bfloat16)
    du = ops.gemm_bf16_gelu_grad(dy, w2, u)
    ud = u.double()
    gp = 0.5 * (1 + torch.erf(ud / 2 ** 0.5)) + ud * torch.exp(-0.5 * ud * ud) / (2 * torch.pi) ** 0.5
    ref = (dy.double() @ w2.double()) * gp
    mag = (dy.double().abs() @ w2.double().abs()) * (gp.abs() + 1)
    _check(du, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -16 * mag, "dU")


def _student(seed=0):
    torch.manual_seed(seed)
    m = ErnieStudent(vocab=1000, hidden=384, layers=4, heads=6, ffn=1536, max_pos=513, num_labels=2)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return m.to(DEV)


def _batch(b=32, l=128, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(1, 1000, (b, l), device=DEV, generator=g)
    lens = torch.randint(1, l + 1, (b, 1), device=DEV, generator=g)
    ids[torch.arange(l, device=DEV).unsqueeze(0) >= lens] = 0
    ids[1] = torch.randint(1, 1000, (l,), device=DEV, generator=g)
    ids[1, 0] = 0                                                     # a sample whose token 0 is masked
    return ids, torch.randint(0, 2, (b,), device=DEV, generator=g)


def test_student_gradients_match_float32_torch():
    """Every parameter gradient of one bf16 step within 3 % (relative L2) of the float32 torch encoder's."""
    m = _student()
    ids, label = _batch(16, 128)
    ops.reset_fallbacks()
    torch.nn.functional.cross_entropy(m(ids), label).backward()
    assert ops.fallbacks() == {}
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    b, l = ids.shape
    pos = torch.arange(l, device=DEV).expand(b, l)
    ref = _functional_encoder(m, ids, pos, torch.zeros_like(ids), ids != 0)
    torch.nn.functional.cross_entropy(ref, label).backward()
    worst = 0.0
    for n, p in m.named_parameters():
        r = float((got[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30))
        worst = max(worst, r)
        assert r < 0.03, "%s: relative L2 error %.4f" % (n, r)
    print("worst relative gradient error %.4f" % worst)


def _train(m, opt, ids, label):
    opt.zero_grad(set_to_none=False)
    loss = torch.nn.functional.cross_entropy(m(ids), label)
    loss.backward()
    opt.step()
    return loss


def test_student_step_deterministic_and_graph_replay():
    ids, label = _batch()
    runs = []
    for _ in range(2):
        m = _student()
        opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)
        for _ in range(2):
            _train(m, opt, ids, label)
        runs.append({k: v.clone() for k, v in m.state_dict().items()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k                   # bitwise reproducible
    m = _student()
    opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)
    ops.reset_fallbacks()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _train(m, opt, ids, label)
    torch.cuda.current_stream().wait_stream(side)
    assert ops.fallbacks() == {}
    state = ({k: v.clone() for k, v in m.state_dict().items()},
             [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in s.items()} for s in opt.state.values()])

    def restore():
        with torch.no_grad():
            for k, v in m.state_dict().items():
                v.copy_(state[0][k])
            for s, s0 in zip(opt.state.values(), state[1]):
                for k, v in s.items():
                    if torch.is_tensor(v):
                        v.copy_(s0[k])

    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        gl = _train(m, opt, ids, label)
    restore()
    el = _train(m, opt, ids, label).clone()
    eager = {k: v.clone() for k, v in m.state_dict().items()}
    restore()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gl, el)
    for k, v in m.state_dict().items():
        assert torch.equal(v, eager[k]), k


def test_distill_example_ernie_on_gpu():
    p = subprocess.run([sys.executable, "examples/distill/nlp/distill.py", "--model", "ernie", "--epochs", "2",
                        "--vocab", "400"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600,
                       text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", p.stdout)]
    assert len(losses) >= 4 and min(losses[-2:]) < losses[0], p.stdout
