"""Dropout on the GPU: every kernel against float64 references built from ops.transformer.dropout_keep_reference at the
generator state the call drew (ops.dropout bit for bit; the residual-dropout GEMM epilogue, the attention forward and
backward and embedding-LayerNorm within float64 bounds), and whole ErnieStudent steps with dropout: against a float32
functional encoder that applies the reference masks at the documented sites and offsets, bitwise reproducible, in a
CUDA graph, and unchanged at p = 0 and in eval().

Bounds (``mag``: the same expression over absolute values):
  residual-dropout epilogue  kept: |out - ref| <= 2^-8 |ref| + 2^-16 mag (bf16 store; fp32 sums over K <= 384);
                             dropped: the addend bit for bit
  attention O                2^-8 |ref| + 2^-6 mag: the bf16 P (relative 2^-9) and the row sum over rounded values, as
                             the backward bound of tests/test_ernie_student_gpu.py
  attention dQ / dK / dV     2^-8 |ref| + 2^-6 mag, the existing backward bound, with Z in the reference
  embedding-LayerNorm        y: 2^-8 |ref| + 2^-16 mag; dE, dgamma, dbeta: the LayerNorm backward bounds on Z o dy
With EDL_F64_BOUNDS_LOG set, each check appends its worst error / bound ratio to that file."""
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models.ernie import ErnieStudent
from edl_b200.ops.transformer import _draw
from student_oracle import attention_f64 as _attention_f64, ln_f64 as _ln_f64

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 0.1


def _gen():
    return torch.cuda.default_generators[0]


def _scale(p):
    return torch.tensor(1.0 / (1.0 - p), dtype=torch.float32).item()


def _z(seed, offset, shape, p=P):
    """float64 Z = keep * fp32(1 / (1 - p)) over the flat indices of ``shape``."""
    n = 1
    for d in shape:
        n *= d
    keep = ops.dropout_keep_reference(seed, offset, torch.arange(n, device=DEV), p).view(shape)
    return keep.double() * _scale(p)


def _check(out, ref, bound, what):
    out = out.double()
    assert torch.isfinite(out).all(), what + ": non-finite output"
    err = (out - ref).abs()
    ratio = float((err / bound.clamp_min(1e-300)).max())
    path = os.environ.get("EDL_F64_BOUNDS_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"what": what, "c1": ratio}) + "\n")
    assert (err <= bound).all(), "%s: worst error / bound %.3f" % (what, ratio)
    return ratio


@pytest.mark.parametrize("n", [1, 7, 8, 1001, 4099, (1 << 20) + 3])
def test_dropout_op_exact(n):
    torch.cuda.manual_seed(n)
    seed = torch.cuda.initial_seed()
    buf = torch.ones(n + 1, device=DEV, dtype=torch.bfloat16)
    for x in (buf[:n], buf[1:]):                                       # 16-byte aligned and not
        x = x.clone().requires_grad_(True) if x.data_ptr() % 16 == 0 else x.detach().requires_grad_(True)
        off = _gen().get_offset()
        y = ops.dropout(x, P)
        assert _gen().get_offset() == off + 4
        keep = ops.dropout_keep_reference(seed, off, torch.arange(n, device=DEV), P)
        s = torch.tensor(_scale(P)).to(torch.bfloat16).to(DEV)
        assert torch.equal(y, torch.where(keep, s, torch.zeros_like(s)))
        g = torch.randn(n, device=DEV).to(torch.bfloat16)
        y.backward(g)
        assert torch.equal(x.grad, torch.where(keep, (g.float() * _scale(P)).to(torch.bfloat16), torch.zeros_like(g)))
    assert ops.dropout(buf, 0.0) is buf and ops.dropout(buf, P, training=False) is buf


@pytest.mark.parametrize("M", [1, 129, 4096])
@pytest.mark.parametrize("N", [384, 1536, 200])
def test_residual_dropout_epilogue(M, N):
    torch.manual_seed(M * N)
    K = 384
    x = torch.randn(M, K, device=DEV).to(torch.bfloat16)
    w = (torch.randn(N, K, device=DEV) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV)
    add = torch.randn(M, N, device=DEV).to(torch.bfloat16)
    drop = _draw(DEV, P)
    ops.reset_fallbacks()
    out = ops.gemm_bf16_residual_dropout(x, w, bias, add, drop)
    assert ops.fallbacks() == {}
    z = _z(drop.seed, drop.offset, (M, N))
    kept = z != 0
    branch = x.double() @ w.double().t() + bias.double()
    ref = add.double() + z * branch
    mag = add.double().abs() + z * (x.double().abs() @ w.double().abs().t() + bias.double().abs())
    bound = 2.0 ** -8 * ref.abs() + 2.0 ** -16 * mag
    _check(out[kept], ref[kept], bound[kept], "residual dropout M=%d N=%d" % (M, N))
    assert torch.equal(out[~kept], add[~kept])                         # a dropped element stores the residual


@pytest.mark.parametrize("L", [1, 63, 64, 65, 128, 200, 512])
def test_attention_dropout_f64_bounds(L):
    torch.manual_seed(L)
    b, h = 4, 2
    qkv = (torch.randn(b * L, 3 * h * 64, device=DEV) * 1.5).to(torch.bfloat16)
    mask = (torch.rand(b, L, device=DEV) > 0.3).to(torch.uint8)
    mask[0] = 0                                                       # a fully masked sample
    mask[1, 0] = 0                                                    # token 0 masked
    mask[2] = 1
    do = torch.randn(b * L, h * 64, device=DEV).to(torch.bfloat16)
    _, lse0 = ops.transformer.attention_forward_saved(qkv, mask, b, L, h)
    drop = _draw(DEV, P)
    out, lse = ops.transformer.attention_forward_saved(qkv, mask, b, L, h, drop)
    assert torch.equal(lse, lse0)                                     # lse of the undropped softmax
    dqkv = ops.transformer.attention_backward(qkv, mask, out, lse, do, b, L, h, drop)
    z = _z(drop.seed, drop.offset, (b, h, L, L))
    o, mo, ref, mag = _attention_f64(qkv, mask, do, b, L, h, z)
    _check(out, o, 2.0 ** -8 * o.abs() + 2.0 ** -6 * mo, "attention dropout O L=%d" % L)
    _check(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, "attention dropout dqkv L=%d" % L)
    has = (mask != 0).any(1)
    assert (dqkv.view(b, L, -1)[~has] == 0).all()                     # no valid key: exactly zero gradients
    assert torch.equal(ops.transformer.attention_backward(qkv, mask, out, lse, do, b, L, h, drop), dqkv)
    if L >= 63:
        # negative control: the mask of the next site's offset breaks the bound
        zb = _z(drop.seed, drop.offset + 4, (b, h, L, L))
        o2, mo2, _, _ = _attention_f64(qkv, mask, do, b, L, h, zb)
        with pytest.raises(AssertionError):
            _check(out, o2, 2.0 ** -8 * o2.abs() + 2.0 ** -6 * mo2, "control")


@pytest.mark.parametrize("rows,C", [(5, 384), (4096, 384), (700, 768)])
def test_embedding_layernorm_dropout_f64_bounds(rows, C):
    torch.manual_seed(rows)
    word = torch.randn(500, C, device=DEV) * 0.5
    pos = torch.randn(130, C, device=DEV) * 0.5
    seg = torch.randn(2, C, device=DEV) * 0.5
    gamma, beta = torch.randn(C, device=DEV), torch.randn(C, device=DEV)
    ids = torch.randint(0, 500, (rows,), device=DEV)
    ids[: rows // 2] = 7
    pid, sid = torch.randint(0, 130, (rows,), device=DEV), torch.randint(0, 2, (rows,), device=DEV)
    ps = [t.clone().requires_grad_(True) for t in (word, pos, seg, gamma, beta)]
    seed, off = torch.cuda.initial_seed(), _gen().get_offset()
    y = ops.embedding_layernorm_trainable(ids, pid, sid, *ps, 1e-12, dropout_p=P)
    assert _gen().get_offset() == off + 4
    dy = torch.randn_like(y.float()).to(torch.bfloat16)
    y.backward(dy)
    z = _z(seed, off, (rows, C))
    tb = [t.to(torch.bfloat16) for t in (word, pos, seg)]
    x = tb[0].double()[ids] + tb[1].double()[pid] + tb[2].double()[sid]
    xh, dE, mag, dg, mg, db, mb = _ln_f64(x, dy.double() * z, gamma, 1e-12)
    yref = z * (xh * gamma.double() + beta.double())
    _check(y, yref, 2.0 ** -8 * yref.abs() + 2.0 ** -16 * z * (xh.abs() * gamma.double().abs() + beta.double().abs()),
           "embedding LayerNorm dropout y")
    for t, idx, n, what in ((ps[0], ids, 500, "word"), (ps[1], pid, 130, "pos"), (ps[2], sid, 2, "seg")):
        ref = torch.zeros(n, C, device=DEV, dtype=torch.float64).index_add_(0, idx, dE)
        m = torch.zeros(n, C, device=DEV, dtype=torch.float64).index_add_(0, idx, mag + dE.abs())
        _check(t.grad, ref, 2.0 ** -12 * m, "embedding table dropout " + what)
    _check(ps[3].grad, dg, 2.0 ** -12 * mg, "dgamma dropout")
    _check(ps[4].grad, db, 2.0 ** -12 * mb, "dbeta dropout")


def _student(seed=0, **kw):
    torch.manual_seed(seed)
    m = ErnieStudent(vocab=1000, hidden=384, layers=4, heads=6, ffn=1536, max_pos=513, num_labels=2, **kw)
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
    ids[1, 0] = 0
    return ids, torch.randint(0, 2, (b,), device=DEV, generator=g)


def _functional_encoder_dropout(m, ids, keep, seed, off, p):
    """Float32 post-LN encoder from nn.functional with the reference masks at the sites and offsets ErnieStudent
    documents: embedding output, then per layer the probabilities, the attention branch and the FFN branch, then the
    pooled [CLS] features; 4 offset units per site."""
    b, l = ids.shape
    c, nh = m.hidden, m.heads
    z = lambda o, shape: _z(seed, o, shape, p).float()   # noqa: E731
    pos = torch.arange(l, device=DEV).expand(b, l)
    x = F.embedding(ids, m.word_emb) + F.embedding(pos, m.pos_emb) + F.embedding(torch.zeros_like(ids), m.seg_emb)
    x = F.layer_norm(x, (c,), m.emb_ln_g, m.emb_ln_b, m.eps) * z(off, (b, l, c))
    bias = torch.zeros(b, 1, 1, l, device=DEV).masked_fill(~keep.view(b, 1, 1, l), float("-inf"))
    for i, lyr in enumerate(m.layers):
        o0 = off + 4 + 12 * i
        q, k, v = (t.transpose(1, 2) for t in F.linear(x, lyr.qkv_w, lyr.qkv_b).view(b, l, 3, nh, 64).unbind(2))
        pr = torch.softmax(q @ k.transpose(-1, -2) / 8 + bias, -1) * z(o0, (b, nh, l, l))
        o = (pr @ v).transpose(1, 2).reshape(b, l, c)
        x = F.layer_norm(z(o0 + 4, (b, l, c)) * F.linear(o, lyr.out_w, lyr.out_b) + x, (c,), lyr.ln1_g, lyr.ln1_b, m.eps)
        f = F.linear(F.gelu(F.linear(x, lyr.ffn1_w, lyr.ffn1_b)), lyr.ffn2_w, lyr.ffn2_b)
        x = F.layer_norm(z(o0 + 8, (b, l, c)) * f + x, (c,), lyr.ln2_g, lyr.ln2_b, m.eps)
    pooled = torch.tanh(F.linear(x[:, 0], m.pool_w, m.pool_b)) * z(off + 4 + 12 * len(m.layers), (b, c))
    return F.linear(pooled, m.cls_w, m.cls_b)


def test_student_dropout_gradients_match_float32_torch():
    m = _student(hidden_dropout=P, attention_dropout=P)
    ids, label = _batch()
    seed, off = torch.cuda.initial_seed(), _gen().get_offset()
    ops.reset_fallbacks()
    F.cross_entropy(m(ids), label).backward()
    assert ops.fallbacks() == {}
    assert _gen().get_offset() == off + 4 * (2 + 3 * len(m.layers))
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    F.cross_entropy(_functional_encoder_dropout(m, ids, ids != 0, seed, off, P), label).backward()
    worst = 0.0
    for n, p in m.named_parameters():
        r = float((got[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30))
        worst = max(worst, r)
        assert r < 0.03, "%s: relative L2 error %.4f" % (n, r)
    print("worst relative gradient error with dropout %.4f" % worst)


def _train(m, opt, ids, label):
    opt.zero_grad(set_to_none=False)
    loss = F.cross_entropy(m(ids), label)
    loss.backward()
    opt.step()
    return loss


def test_student_dropout_deterministic_and_graph_replay():
    ids, label = _batch()
    runs = []
    for _ in range(2):
        m = _student(hidden_dropout=P, attention_dropout=P)
        opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)
        for _ in range(2):
            _train(m, opt, ids, label)
        runs.append({k: v.clone() for k, v in m.state_dict().items()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k                   # same generator state: bitwise equal
    m = _student(hidden_dropout=P, attention_dropout=P)
    opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)
    ops.reset_fallbacks()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _train(m, opt, ids, label)
    torch.cuda.current_stream().wait_stream(side)
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
    assert ops.fallbacks() == {}
    restore()
    off = _gen().get_offset()
    el = _train(m, opt, ids, label).clone()
    eager = {k: v.clone() for k, v in m.state_dict().items()}
    per_step = 4 * (2 + 3 * len(m.layers))
    assert _gen().get_offset() == off + per_step
    restore()
    _gen().set_offset(off)
    g.replay()
    torch.cuda.synchronize()
    assert _gen().get_offset() == off + per_step
    assert torch.equal(gl, el)                                        # the replay drew the eager step's masks
    for k, v in m.state_dict().items():
        assert torch.equal(v, eager[k]), k
    restore()
    g.replay()                                                        # the next offsets: different masks
    torch.cuda.synchronize()
    assert _gen().get_offset() == off + 2 * per_step
    assert not torch.equal(gl, el)


def test_student_p0_and_eval_unchanged():
    ids, _ = _batch()
    base = _student()
    for kw, train in (({"hidden_dropout": 0.0, "attention_dropout": 0.0}, True),
                      ({"hidden_dropout": P, "attention_dropout": P}, False)):
        m = _student(**kw)
        base.train(train)
        m.train(train)
        with torch.no_grad():
            ops.reset_launches()
            ref = base(ids)
            n_ref = ops.launches()
            off = _gen().get_offset()
            ops.reset_launches()
            got = m(ids)
            assert ops.launches() == n_ref
            assert _gen().get_offset() == off                        # nothing drawn
        assert torch.equal(got, ref)


def test_distill_example_ernie_dropout_on_gpu():
    p = subprocess.run([sys.executable, "examples/distill/nlp/distill.py", "--model", "ernie", "--dropout", "0.1",
                        "--epochs", "2", "--vocab", "400"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=600, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", p.stdout)]
    assert len(losses) >= 4 and all(v == v for v in losses), p.stdout
