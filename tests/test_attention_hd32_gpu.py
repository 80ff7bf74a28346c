"""Head dim 32 on the GPU: the D = 32 instantiations of the attention kernels against float64, padded and packed, with
and without dropout, and the MiniLM-shaped encoder and the 12-head student end to end on the kernels.

The float64 references here are those of tests/student_oracle.py with the head dim as a parameter; the bounds are the
oracle's with their D-dependent terms taken at D = 32: scores accumulate D / 16 + 1 fp32 roundings, and the exponent
scale is c = log2(e) / sqrt(D).
  O          the eps / tau_acc bound of tests/test_ernie_gpu.py (``check_bf16`` criterion 1, tau = 1)
  lse        |lse~ - lse| <= 1.45 (eps + tau_acc) + 2^-23 |lse|, +inf exactly for a row without a valid key
  dQ, dK, dV |out - ref| <= 2^-8 |ref| + 2^-6 mag, exactly 0 for a row without a valid key
  O with Z   2^-8 |ref| + 2^-6 mag (dropout: the bf16 P carries the kept elements' scale)"""
import math

import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models import teacher_zoo
from edl_b200.models.ernie import ErnieStudent, pack_sequences
from f64_bounds import EPS32, check_bf16
from test_ernie_student_cpu import _functional_encoder

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
T = ops.transformer
D = 32
P = 0.1
LOG2E = math.log2(math.e)


def _heads(qkv, b, l, h, d):
    x = qkv.double().view(b, l, 3, h, d)
    return [x[:, :, i].transpose(1, 2) for i in range(3)]                        # [B, H, L, d]


def _flat(t):
    b, h, l, d = t.shape
    return t.transpose(1, 2).reshape(b * l, h * d)


def _eps(q, k, keep, d):
    """Per row: the relative error eps of the kernel's rounded probabilities, and c s with masked keys at -inf."""
    s = q @ k.transpose(-1, -2)
    smag = q.abs() @ k.abs().transpose(-1, -2)
    c = LOG2E / math.sqrt(d)
    cs = (s * c).masked_fill(~keep, float("-inf"))
    m = cs.amax(-1, keepdim=True)
    mf = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    delta = c * (d / 16 + 1) * EPS32 * smag + EPS32 * (cs.abs() + (cs - mf).abs())
    eps = (2.0 ** -8 + 2.0 ** -21 + 1.01 * math.log(2) * delta).masked_fill(~keep, 0.0).amax(-1, keepdim=True)
    return eps, cs, mf


def attention_f64(qkv, mask, b, l, h, d, do=None, z=None):
    """Float64 attention of head dim d with its bounds: dict of o, o_slack (p = 0 bound), lse, lse_bound and, with
    ``do``, dqkv and mag; ``z`` [B, H, L, L] dropout on the probabilities (then o_mag for the 2^-6 bound)."""
    q, k, v = _heads(qkv, b, l, h, d)
    keep = (torch.ones(b, l, dtype=torch.bool, device=qkv.device) if mask is None else mask != 0).view(b, 1, 1, l)
    eps, cs, mf = _eps(q, k, keep, d)
    tau_acc = (8 * -(-l // 64) + 32) * EPS32
    tot = torch.exp2(cs - mf).sum(-1, keepdim=True)
    lse = torch.where(tot > 0, mf + torch.log2(tot.clamp_min(1e-300)), torch.full_like(tot, float("inf")))
    p = (torch.exp2(cs - mf) / torch.where(tot > 0, tot, torch.ones_like(tot))).masked_fill(~keep, 0.0)
    zz = torch.ones_like(p) if z is None else z.double()
    pz = p * zz
    o = pz @ v
    r = {"o": _flat(o), "o_slack": _flat((2 * eps / (1 - eps) + tau_acc) * (p @ v.abs())), "o_mag": _flat(pz @ v.abs()),
         "lse": lse.squeeze(-1),
         "lse_bound": (1.45 * (eps + tau_acc) + EPS32 * lse.abs().nan_to_num(0.0, posinf=0.0)).squeeze(-1)}
    if do is not None:
        sc = 1 / math.sqrt(d)
        dO = do.double().view(b, l, h, d).transpose(1, 2)
        dp = dO @ v.transpose(-1, -2)
        ds = p * (zz * dp - (dO * o).sum(-1, keepdim=True))
        mds = p * (zz * (dO.abs() @ v.abs().transpose(-1, -2)) + (dO.abs() * o.abs()).sum(-1, keepdim=True))
        r["dqkv"] = torch.cat([_flat(ds @ k * sc), _flat(ds.transpose(-1, -2) @ q * sc),
                               _flat(pz.transpose(-1, -2) @ dO)], 1)
        r["mag"] = torch.cat([_flat(mds @ k.abs() * sc), _flat(mds.transpose(-1, -2) @ q.abs() * sc),
                              _flat(pz.transpose(-1, -2) @ dO.abs())], 1)
    return r


def _check(out, ref, bound, what):
    out = out.double()
    assert torch.isfinite(out).all(), what + ": non-finite output"
    err = (out - ref).abs()
    assert (err <= bound).all(), "%s: worst error / bound %.3f" % (what, float((err / bound.clamp_min(1e-300)).max()))


def _check_lse(lse, ref, bound, what):
    inf = torch.isinf(ref)
    assert torch.equal(torch.isinf(lse), inf) and (lse[inf] > 0).all(), what + ": +inf rows"
    _check(lse[~inf], ref[~inf], bound[~inf], what)


def _dqkv_bound(r):
    return 2.0 ** -8 * r["dqkv"].abs() + 2.0 ** -6 * r["mag"]


def _padded_inputs(b, l, h, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = (torch.randn(b * l, 3 * h * D, device=DEV, generator=g) * 2).to(torch.bfloat16)
    mask = (torch.rand(b, l, device=DEV, generator=g) > 0.3).to(torch.uint8)
    mask[0] = 0                                                       # a sample without any valid key
    mask[1, 0] = 0                                                    # token 0 masked
    mask[2] = 1
    do = torch.randn(b * l, h * D, device=DEV, generator=g).to(torch.bfloat16)
    return qkv, mask, do


def _drop_z(drop, b, h, l):
    idx = torch.arange(b * h * l * l, device=DEV)
    return (ops.dropout_keep_reference(drop.seed, drop.offset, idx, P).double() * drop.scale).view(b, h, l, l)


@pytest.mark.parametrize("L", [1, 63, 64, 65, 128, 200, 512])
def test_forward_backward_padded(L):
    b, h = 4, 3
    qkv, mask, do = _padded_inputs(b, L, h, L)
    ops.reset_fallbacks()
    out, lse = T.attention_forward_saved(qkv, mask, b, L, h)
    assert torch.equal(out, ops.attention(qkv, mask, b, L, h, D))    # the inference instantiation, the same bits
    dqkv = T.attention_backward(qkv, mask, out, lse, do, b, L, h)
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    r = attention_f64(qkv, mask, b, L, h, D, do)
    check_bf16(out, r["o"], r["o_slack"], tau=1.0, criteria=(1,), what="attention O hd32 L %d" % L)
    _check_lse(lse, r["lse"], r["lse_bound"], "lse hd32 L %d" % L)
    _check(dqkv, r["dqkv"], _dqkv_bound(r), "dqkv hd32 L %d" % L)
    has = (mask != 0).any(1)
    assert (out.view(b, L, -1)[~has] == 0).all() and (dqkv.view(b, L, -1)[~has] == 0).all()
    assert torch.equal(T.attention_backward(qkv, mask, out, lse, do, b, L, h), dqkv)


def test_backward_negative_control():
    """One bf16 ulp added to a dQ element of a row without a valid key (reference 0, bound 0) fails the check."""
    b, L, h = 3, 96, 2
    qkv, mask, do = _padded_inputs(b, L, h, 5)
    out, lse = T.attention_forward_saved(qkv, mask, b, L, h)
    dqkv = T.attention_backward(qkv, mask, out, lse, do, b, L, h)
    r = attention_f64(qkv, mask, b, L, h, D, do)
    _check(dqkv, r["dqkv"], _dqkv_bound(r), "control baseline")
    bad = dqkv.clone()
    bits = bad.view(torch.int16)
    bits[3, 5] += 1                                                   # row 3 is in sample 0: no valid key
    with pytest.raises(AssertionError):
        _check(bad, r["dqkv"], _dqkv_bound(r), "control")


def test_dropout_padded():
    b, L, h = 3, 130, 4
    qkv, mask, do = _padded_inputs(b, L, h, 11)
    _, lse0 = T.attention_forward_saved(qkv, mask, b, L, h)
    gen = torch.cuda.default_generators[0]
    off = gen.get_offset()
    drop = T._draw(DEV, P)
    assert gen.get_offset() == off + 4
    out, lse = T.attention_forward_saved(qkv, mask, b, L, h, drop)
    dqkv = T.attention_backward(qkv, mask, out, lse, do, b, L, h, drop)
    assert torch.equal(lse, lse0)                                     # lse is the undropped softmax's
    r = attention_f64(qkv, mask, b, L, h, D, do, z=_drop_z(drop, b, h, L))
    _check(out, r["o"], 2.0 ** -8 * r["o"].abs() + 2.0 ** -6 * r["o_mag"], "O with dropout")
    _check(dqkv, r["dqkv"], _dqkv_bound(r), "dqkv with dropout")


# ---------------------------------------------------------------------------------------------------------- packed
LENS = [1, 63, 64, 65, 128, 38]                                       # T = 359, odd


def _packed_inputs(seed, masked=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h, t = 4, sum(LENS)
    cu = torch.tensor([0] + LENS, dtype=torch.int32).cumsum(0).to(torch.int32).to(DEV)
    qkv = (torch.randn(t, 3 * h * D, device=DEV, generator=g) * 2).to(torch.bfloat16)
    do = torch.randn(t, h * D, device=DEV, generator=g).to(torch.bfloat16)
    km = None
    if masked:
        km = (torch.rand(t, device=DEV, generator=g) > 0.2).to(torch.uint8)
        km[cu[:-1].long()] = 1
        km[int(cu[3])] = 0                                            # sequence 3: token 0 is not a key
    return qkv, cu, km, do, h


def _seq(cu, i):
    return int(cu[i]), int(cu[i + 1])


def test_packed_bitwise_padded_b1_and_isolated():
    qkv, cu, km, do, h = _packed_inputs(3)
    mx = max(LENS)
    ops.reset_fallbacks()
    out, lse = T.attention_varlen_forward_saved(qkv, cu, mx, h, km)
    dqkv = T.attention_varlen_backward(qkv, cu, mx, h, km, out, lse, do)
    assert torch.equal(out, ops.attention_varlen(qkv, cu, mx, h, km))   # inference instantiation, the same bits
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    for i in range(len(LENS)):
        s, e = _seq(cu, i)
        n = e - s
        m = km[s:e].view(1, n).contiguous()
        o1, l1 = T.attention_forward_saved(qkv[s:e].contiguous(), m, 1, n, h)
        d1 = T.attention_backward(qkv[s:e].contiguous(), m, o1, l1, do[s:e].contiguous(), 1, n, h)
        assert torch.equal(out[s:e], o1) and torch.equal(lse[:, s:e], l1.view(h, n)) and torch.equal(dqkv[s:e], d1), i
        r = attention_f64(qkv[s:e], m, 1, n, h, D, do[s:e])
        check_bf16(out[s:e], r["o"], r["o_slack"], tau=1.0, criteria=(1,), what="packed O seq %d" % i)
        _check_lse(lse[:, s:e], r["lse"].view(h, n), r["lse_bound"].view(h, n), "packed lse seq %d" % i)
        _check(dqkv[s:e], r["dqkv"], _dqkv_bound(r), "packed dqkv seq %d" % i)
    # refilling every other sequence with NaN leaves a sequence's bits unchanged
    for i in (0, 3, 4):
        s, e = _seq(cu, i)
        q2, d2 = torch.full_like(qkv, float("nan")), torch.full_like(do, float("nan"))
        q2[s:e], d2[s:e] = qkv[s:e], do[s:e]
        o2, l2 = T.attention_varlen_forward_saved(q2, cu, mx, h, km)
        g2 = T.attention_varlen_backward(q2, cu, mx, h, km, o2, l2, d2)
        assert torch.equal(o2[s:e], out[s:e]) and torch.equal(l2[:, s:e], lse[:, s:e]), i
        assert torch.equal(g2[s:e], dqkv[s:e]), i


def test_dropout_packed():
    qkv, cu, km, do, h = _packed_inputs(7)
    mx = max(LENS)
    _, lse0 = T.attention_varlen_forward_saved(qkv, cu, mx, h, km)
    drop = T._draw(DEV, P)
    out, lse = T.attention_varlen_forward_saved(qkv, cu, mx, h, km, drop)
    dqkv = T.attention_varlen_backward(qkv, cu, mx, h, km, out, lse, do, drop)
    assert torch.equal(lse, lse0)
    for b, n in enumerate(LENS):
        s, e = _seq(cu, b)
        i = torch.arange(n, device=DEV)
        hh = torch.arange(h, device=DEV)
        idx = ((b * h + hh).view(-1, 1, 1) * 512 + i.view(1, -1, 1)) * 512 + i.view(1, 1, -1)
        z = ops.dropout_keep_reference(drop.seed, drop.offset, idx, P).double().unsqueeze(0) * drop.scale
        r = attention_f64(qkv[s:e], km[s:e].view(1, n), 1, n, h, D, do[s:e], z=z)
        _check(out[s:e], r["o"], 2.0 ** -8 * r["o"].abs() + 2.0 ** -6 * r["o_mag"], "packed O with dropout %d" % b)
        _check(dqkv[s:e], r["dqkv"], _dqkv_bound(r), "packed dqkv with dropout %d" % b)


def test_unsupported_head_dims_are_counted():
    """Head dims the kernels do not take (TinyBERT's 26, 128) run the float32 reference, counted as fallbacks."""
    for d, h in ((26, 12), (128, 2)):
        qkv = torch.randn(2 * 16, 3 * h * d, device=DEV).to(torch.bfloat16)
        ops.reset_fallbacks()
        out = ops.attention(qkv, None, 2, 16, h, d)
        assert out.shape == (32, h * d) and ops.fallbacks() != {}, d
        with pytest.raises(RuntimeError, match="head dim D = 64 or 32"):
            ops.native().attention_fwd(qkv, None, torch.empty_like(out), 2, 16, h, None, None)


# ------------------------------------------------------------------------------------------------------ models
def _inputs(b, l, seed, vocab):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(l // 4, l + 1, (b,), generator=g)
    lens[0] = l
    mask = (torch.arange(l)[None] < lens[:, None]).float()
    ids = torch.randint(0, vocab, (b, l), generator=g)
    seg = torch.randint(0, 2, (b, l), generator=g)
    pos = torch.arange(l).expand(b, l).contiguous()
    return [t.to(DEV) for t in (ids, pos, seg, mask)]


def _torch_forward32(model, ids, pos, seg, mask):
    """fp32 torch forward of any head dim with the bf16-rounded weights of the kernel path."""
    r = lambda t: t.detach().to(torch.bfloat16).float()                               # noqa: E731
    b, l = ids.shape
    c, h = model.hidden, model.heads
    x = r(model.word_emb)[ids] + r(model.pos_emb)[pos] + r(model.seg_emb)[seg]
    x = F.layer_norm(x, (c,), model.emb_ln_g.float(), model.emb_ln_b.float(), model.eps)
    keep = (mask != 0).view(b, 1, 1, l)
    for lyr in model.layers:
        q, k, v = F.linear(x, r(lyr.qkv_w), lyr.qkv_b.float()).view(b, l, 3, h, c // h).permute(2, 0, 3, 1, 4)
        ctx = F.scaled_dot_product_attention(q, k, v, attn_mask=keep).transpose(1, 2).reshape(b, l, c)
        x = F.layer_norm(F.linear(ctx, r(lyr.out_w), lyr.out_b.float()) + x, (c,), lyr.ln1_g.float(), lyr.ln1_b.float(),
                         model.eps)
        f = F.gelu(F.linear(x, r(lyr.ffn1_w), lyr.ffn1_b.float()))
        x = F.layer_norm(F.linear(f, r(lyr.ffn2_w), lyr.ffn2_b.float()) + x, (c,), lyr.ln2_g.float(), lyr.ln2_b.float(),
                         model.eps)
    pooled = torch.tanh(F.linear(x[:, 0], r(model.pool_w), model.pool_b.float()))
    return F.linear(pooled, r(model.cls_w), model.cls_b.float())


def _agree(got, other):
    cos = F.cosine_similarity(got.flatten()[None].double(), other.flatten()[None].double()).item()
    return cos, (got.argmax(1) == other.argmax(1)).float().mean().item()


def _replay_equals(fn, want):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = fn()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, want)


def test_minilm_encoder_forward_packed_fp8():
    torch.manual_seed(0)
    model = teacher_zoo.build("minilm_l12_h384")[0].to(DEV).eval()
    with torch.no_grad():
        model.cls_w.mul_(20)                  # decisive logits for the top-1 comparison
    b, l = 16, 128
    ids, pos, seg, mask = _inputs(b, l, 1, 30522)
    mask[3, 0] = 0                            # a sample whose token 0 is masked: the packed path's key_mask
    packed = [p.to(DEV) if torch.is_tensor(p) else p for p in pack_sequences(ids.cpu(), pos.cpu(), seg.cpu(),
                                                                               mask.cpu(), model.pos_emb.shape[0])]
    assert packed[5] is not None
    ops.reset_fallbacks()
    padded = model(ids, pos, seg, mask)
    got = model.forward_packed(*packed)
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    want = _torch_forward32(model, ids, pos, seg, mask)
    for name, x, other in (("padded", padded, want), ("packed", got, want), ("packed vs padded", got, padded)):
        cos, agree = _agree(x, other)
        assert cos > 0.999 and agree >= 15 / 16, (name, cos, agree)
    _replay_equals(lambda: model.forward_packed(*packed), got)
    reqs = [[t[i:i + 4].cpu() for t in (ids, pos, seg, mask)] for i in (0, 4, 8, 12)]
    assert torch.equal(model.forward_requests(reqs), got)
    assert model.enable_fp8() == 48
    ops.reset_fallbacks()
    fp8 = model.forward_packed(*packed)
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    cos, agree = _agree(fp8, got)             # the bar of tests/test_ernie_fp8_gpu.py
    assert cos >= 0.995 and agree >= 15 / 16, (cos, agree)
    _replay_equals(lambda: model.forward_packed(*packed), fp8)


def _student(**kw):
    torch.manual_seed(0)
    m = ErnieStudent(vocab=1000, hidden=384, layers=4, heads=12, ffn=1536, max_pos=513, num_labels=2, **kw)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.05)
    return m.to(DEV)


def _batch(b=16, l=128, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(1, 1000, (b, l), device=DEV, generator=g)
    lens = torch.randint(1, l + 1, (b, 1), device=DEV, generator=g)
    ids[torch.arange(l, device=DEV).unsqueeze(0) >= lens] = 0
    ids[1] = torch.randint(1, 1000, (l,), device=DEV, generator=g)
    ids[1, 0] = 0                                                     # a sample whose token 0 is masked
    return ids, torch.randint(0, 2, (b,), device=DEV, generator=g)


def _packed(ids):
    b, l = ids.shape
    pk = pack_sequences(ids, torch.arange(l).expand(b, l), torch.zeros_like(ids), ids != 0)
    return tuple(t.to(DEV) if torch.is_tensor(t) else t for t in pk)


def _compare_grads(m, got, what):
    worst = 0.0
    for n, p in m.named_parameters():
        r = float((got[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30))
        worst = max(worst, r)
        assert r < 0.03, "%s %s: relative L2 error %.4f" % (what, n, r)
    print("worst relative gradient error (%s) %.4f" % (what, worst))


def _functional_dropout(m, ids, keep, seed, off, p):
    """``_functional_encoder`` with the reference masks at ErnieStudent's documented sites and offsets (padded)."""
    b, l = ids.shape
    c, nh = m.hidden, m.heads
    d = c // nh

    def z(o, shape):
        n = math.prod(shape)
        keep_ = ops.dropout_keep_reference(seed, o, torch.arange(n, device=DEV), p).view(shape)
        return keep_.float() * torch.tensor(1.0 / (1.0 - p), dtype=torch.float32).item()

    pos = torch.arange(l, device=DEV).expand(b, l)
    x = F.embedding(ids, m.word_emb) + F.embedding(pos, m.pos_emb) + F.embedding(torch.zeros_like(ids), m.seg_emb)
    x = F.layer_norm(x, (c,), m.emb_ln_g, m.emb_ln_b, m.eps) * z(off, (b, l, c))
    bias = torch.zeros(b, 1, 1, l, device=DEV).masked_fill(~keep.view(b, 1, 1, l), float("-inf"))
    for i, lyr in enumerate(m.layers):
        o0 = off + 4 + 12 * i
        q, k, v = (t.transpose(1, 2) for t in F.linear(x, lyr.qkv_w, lyr.qkv_b).view(b, l, 3, nh, d).unbind(2))
        pr = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d) + bias, -1) * z(o0, (b, nh, l, l))
        o = (pr @ v).transpose(1, 2).reshape(b, l, c)
        x = F.layer_norm(z(o0 + 4, (b, l, c)) * F.linear(o, lyr.out_w, lyr.out_b) + x, (c,), lyr.ln1_g, lyr.ln1_b,
                         m.eps)
        f = F.linear(F.gelu(F.linear(x, lyr.ffn1_w, lyr.ffn1_b)), lyr.ffn2_w, lyr.ffn2_b)
        x = F.layer_norm(z(o0 + 8, (b, l, c)) * f + x, (c,), lyr.ln2_g, lyr.ln2_b, m.eps)
    pooled = torch.tanh(F.linear(x[:, 0], m.pool_w, m.pool_b)) * z(off + 4 + 12 * len(m.layers), (b, c))
    return F.linear(pooled, m.cls_w, m.cls_b)


@pytest.mark.parametrize("layout", ["padded", "packed", "dropout"])
def test_student_heads12_gradients_match_float32_torch(layout):
    m = _student(**({"hidden_dropout": P, "attention_dropout": P} if layout == "dropout" else {}))
    assert m.head_dim == 32
    ids, label = _batch()
    gen = torch.cuda.default_generators[0]
    seed, off = torch.cuda.initial_seed(), gen.get_offset()
    ops.reset_fallbacks()
    logits = m.forward_packed(*_packed(ids)) if layout == "packed" else m(ids)
    F.cross_entropy(logits, label).backward()
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    assert gen.get_offset() == off + (4 * (2 + 3 * len(m.layers)) if layout == "dropout" else 0)
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    b, l = ids.shape
    if layout == "dropout":
        ref = _functional_dropout(m, ids, ids != 0, seed, off, P)
    else:
        ref = _functional_encoder(m, ids, torch.arange(l, device=DEV).expand(b, l), torch.zeros_like(ids), ids != 0)
    F.cross_entropy(ref, label).backward()
    _compare_grads(m, got, layout)


def test_student_heads12_graph_replay():
    """A padded and a packed step captured in one CUDA graph replay the eager bits."""
    ids, label = _batch(32, 128, seed=2)
    pk = _packed(ids)
    m = _student()
    opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)

    def step():
        opt.zero_grad(set_to_none=False)
        loss = F.cross_entropy(m(ids), label) + F.cross_entropy(m.forward_packed(*pk), label)
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
    assert ops.fallbacks() == {}, ops.fallbacks()
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
        gl = step()
    restore()
    el = step().clone()
    eager = {k: v.clone() for k, v in m.state_dict().items()}
    restore()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gl, el)
    for k, v in m.state_dict().items():
        assert torch.equal(v, eager[k]), k
