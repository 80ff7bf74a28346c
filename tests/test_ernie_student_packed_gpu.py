"""Packed training of the Transformer student on the GPU: the varlen attention backward against float64 bounds (the
padded test's bound) with NaN guard rows, bitwise agreement of the varlen O / lse / dqkv with the padded kernels at
B = 1, isolation between sequences, and whole packed training steps of ErnieStudent (against float32 torch, bitwise
reproducible, CUDA-graph replay, no library fallback, the inference forward's logits, dropout)."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from edl_b200 import ops  # noqa: E402
from edl_b200.models.ernie import ErnieEncoder, pack_sequences  # noqa: E402
from edl_b200.ops.transformer import _draw  # noqa: E402
from f64_bounds import guarded  # noqa: E402
from test_dropout_gpu import (_attention_f64 as _attention_f64_z, _functional_encoder_dropout, _gen, _scale,  # noqa: E402
                              _student)
from test_ernie_packed_gpu import _cu, _key_mask, _length_set  # noqa: E402
from test_ernie_student_cpu import _functional_encoder  # noqa: E402
from test_ernie_student_gpu import _attention_f64, _batch, _check  # noqa: E402

DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 0.1
T = ops.transformer


def _inputs(lens, heads, masked, seed):
    gen = torch.Generator().manual_seed(seed)
    t = sum(lens)
    key_mask = _key_mask(lens, gen) if masked else None
    qkv = guarded((t, 3 * heads * 64), pad_rows=3, values=(torch.randn(t, 3 * heads * 64, generator=gen) * 1.5)
                  .to(torch.bfloat16).to(DEV))                         # NaN rows around every operand
    do = guarded((t, heads * 64), pad_rows=3, values=torch.randn(t, heads * 64, generator=gen).to(torch.bfloat16)
                 .to(DEV))
    return _cu(lens), key_mask, qkv, do


def _seq_ref(fn, qkv, do, cu, key_mask, h):
    """Per sequence: the float64 reference of attention_backward at B = 1, L = len_b."""
    refs, mags = [], []
    c = cu.tolist()
    for b, (s, e) in enumerate(zip(c[:-1], c[1:])):
        m = torch.ones(1, e - s, dtype=torch.uint8, device=DEV) if key_mask is None else key_mask[s:e].view(1, -1)
        r, g = fn(b, qkv[s:e], m, do[s:e], e - s)
        refs.append(r)
        mags.append(g)
    return torch.cat(refs), torch.cat(mags)


def _varlen_z(drop, b, h, n, p=P):
    """float64 Z of sequence b's probabilities [1, H, n, n]: element (b, h, i, j) at ((b H + h) 512 + i) 512 + j."""
    hh = torch.arange(h, device=DEV).view(-1, 1, 1)
    i = torch.arange(n, device=DEV)
    idx = ((b * h + hh) * 512 + i.view(1, -1, 1)) * 512 + i.view(1, 1, -1)
    return (ops.dropout_keep_reference(drop.seed, drop.offset, idx, p).double() * _scale(p)).unsqueeze(0)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("lengths", ["one", "max", "edges", "seeded", "short"])
def test_attention_varlen_backward_f64_bounds(lengths, masked):
    lens, h = _length_set(lengths), 2
    cu, key_mask, qkv, do = _inputs(lens, h, masked, len(lens) * 10 + masked)
    ml = max(lens)
    out, lse = T.attention_varlen_forward_saved(qkv.t, cu, ml, h, key_mask)
    assert torch.equal(out, ops.attention_varlen(qkv.t, cu, ml, h, key_mask))   # O bitwise the inference kernel's
    dqkv = T.attention_varlen_backward(qkv.t, cu, ml, h, key_mask, out, lse, do.t)
    ref, mag = _seq_ref(lambda b, q, m, d, n: _attention_f64(q, m, d, 1, n, h), qkv.t, do.t, cu, key_mask, h)
    _check(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, "varlen dqkv %s masked %s" % (lengths, masked))
    assert torch.equal(T.attention_varlen_backward(qkv.t, cu, ml, h, key_mask, out, lse, do.t), dqkv)
    qkv.assert_untouched("qkv")
    do.assert_untouched("dout")


def test_attention_varlen_backward_negative_control():
    """Swapped key rows inside one sequence of the reference's input must break the bound."""
    lens, h = [40, 96, 7], 2
    cu, key_mask, qkv, do = _inputs(lens, h, False, 5)
    out, lse = T.attention_varlen_forward_saved(qkv.t, cu, 96, h, None)
    dqkv = T.attention_varlen_backward(qkv.t, cu, 96, h, None, out, lse, do.t)
    bad = qkv.t.clone()
    bad[[43, 110]] = bad[[110, 43]]
    ref, mag = _seq_ref(lambda b, q, m, d, n: _attention_f64(q, m, d, 1, n, h), bad, do.t, cu, None, h)
    with pytest.raises(AssertionError):
        _check(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, "control")


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("lengths", ["edges", "short"])
def test_attention_varlen_matches_padded_at_b1(lengths, masked):
    """Per sequence, the packed O, lse and dqkv are bitwise the padded kernels' at B = 1, L = len_b."""
    lens, h = _length_set(lengths), 3
    cu, key_mask, qkv, do = _inputs(lens, h, masked, 77 + masked)
    out, lse = T.attention_varlen_forward_saved(qkv.t, cu, max(lens), h, key_mask)
    dqkv = T.attention_varlen_backward(qkv.t, cu, max(lens), h, key_mask, out, lse, do.t)
    c = cu.tolist()
    for s, e in zip(c[:-1], c[1:]):
        m = None if key_mask is None else key_mask[s:e].view(1, -1).contiguous()
        q = qkv.t[s:e].contiguous()
        o1, l1 = T.attention_forward_saved(q, m, 1, e - s, h)
        d1 = T.attention_backward(q, m, o1, l1, do.t[s:e].contiguous(), 1, e - s, h)
        assert torch.equal(out[s:e].view(torch.int16), o1.view(torch.int16)), (s, e)
        assert torch.equal(lse[:, s:e].view(torch.int32), l1.view(h, e - s).view(torch.int32)), (s, e)
        assert torch.equal(dqkv[s:e].view(torch.int16), d1.view(torch.int16)), (s, e)


@pytest.mark.parametrize("lengths", ["edges", "seeded"])
def test_attention_varlen_dropout(lengths):
    """With dropout: lse bitwise the p = 0 lse, O and dqkv within the float64 bound of the reference mask at
    ((b H + h) 512 + i) 512 + j, reproducible, and the padded kernel's index rule breaks the bound."""
    lens, h = _length_set(lengths), 2
    cu, key_mask, qkv, do = _inputs(lens, h, True, 31)
    ml = max(lens)
    _, lse0 = T.attention_varlen_forward_saved(qkv.t, cu, ml, h, key_mask)
    drop = _draw(DEV, P)
    out, lse = T.attention_varlen_forward_saved(qkv.t, cu, ml, h, key_mask, drop)
    assert torch.equal(lse, lse0)
    dqkv = T.attention_varlen_backward(qkv.t, cu, ml, h, key_mask, out, lse, do.t, drop)
    assert torch.equal(T.attention_varlen_backward(qkv.t, cu, ml, h, key_mask, out, lse, do.t, drop), dqkv)

    def ref_of(zf):
        os_, mos, rs, ms = [], [], [], []
        c = cu.tolist()
        for b, (s, e) in enumerate(zip(c[:-1], c[1:])):
            m = key_mask[s:e].view(1, -1)
            o, mo, r, g = _attention_f64_z(qkv.t[s:e], m, do.t[s:e], 1, e - s, h, zf(b, e - s))
            os_.append(o), mos.append(mo), rs.append(r), ms.append(g)
        return torch.cat(os_), torch.cat(mos), torch.cat(rs), torch.cat(ms)

    o, mo, ref, mag = ref_of(lambda b, n: _varlen_z(drop, b, h, n))
    _check(out, o, 2.0 ** -8 * o.abs() + 2.0 ** -6 * mo, "varlen dropout O %s" % lengths)
    _check(dqkv, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -6 * mag, "varlen dropout dqkv %s" % lengths)
    # negative control: the padded rule ((b H + h) L + i) L + j with L = len_b is not the packed mask
    def padded_rule(b, n):
        hh = torch.arange(h, device=DEV).view(-1, 1, 1)
        i = torch.arange(n, device=DEV)
        idx = ((b * h + hh) * n + i.view(1, -1, 1)) * n + i.view(1, 1, -1)
        return (ops.dropout_keep_reference(drop.seed, drop.offset, idx, P).double() * _scale(P)).unsqueeze(0)

    o2, mo2, _, _ = ref_of(padded_rule)
    with pytest.raises(AssertionError):
        _check(out, o2, 2.0 ** -8 * o2.abs() + 2.0 ** -6 * mo2, "control")


@pytest.mark.parametrize("masked", [False, True])
def test_attention_varlen_backward_isolation(masked):
    """A sequence's dqkv bits do not change when the other sequences' rows of qkv, O and dO hold NaN."""
    lens, h = [37, 200, 1, 129, 64, 300, 2], 2
    cu, key_mask, qkv, do = _inputs(lens, h, masked, 11 + masked)
    ml = max(lens)
    out, lse = T.attention_varlen_forward_saved(qkv.t, cu, ml, h, key_mask)
    base = T.attention_varlen_backward(qkv.t, cu, ml, h, key_mask, out, lse, do.t)
    c = cu.tolist()
    for b in range(len(lens)):
        other = torch.ones(qkv.t.shape[0], dtype=torch.bool, device=DEV)
        other[c[b]:c[b + 1]] = False
        x, o, d = qkv.t.clone(), out.clone(), do.t.clone()
        for t in (x, o, d):
            t[other] = float("nan")
        got = T.attention_varlen_backward(x, cu, ml, h, key_mask, o, lse, d)
        assert torch.equal(got[c[b]:c[b + 1]].view(torch.int16), base[c[b]:c[b + 1]].view(torch.int16)), b


def _packed(ids):
    b, l = ids.shape
    pk = pack_sequences(ids, torch.arange(l).expand(b, l), torch.zeros_like(ids), ids != 0)
    return tuple(t.to(DEV) if torch.is_tensor(t) else t for t in pk)


def test_packed_student_gradients_match_float32_torch():
    m = _student()
    ids, label = _batch(16, 128)
    pk = _packed(ids)
    assert pk[5] is not None                                          # _batch masks token 0 of sample 1
    ops.reset_fallbacks()
    F.cross_entropy(m.forward_packed(*pk), label).backward()
    assert ops.fallbacks() == {}
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    b, l = ids.shape
    ref = _functional_encoder(m, ids, torch.arange(l, device=DEV).expand(b, l), torch.zeros_like(ids), ids != 0)
    F.cross_entropy(ref, label).backward()
    worst = 0.0
    for n, p in m.named_parameters():
        r = float((got[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30))
        worst = max(worst, r)
        assert r < 0.03, "%s: relative L2 error %.4f" % (n, r)
    print("worst relative gradient error (packed) %.4f" % worst)


def test_packed_student_no_grad_matches_encoder_forward_packed():
    """Under no_grad at p = 0 the training path stores what the inference path stores: the logits are bitwise those of
    ErnieEncoder.forward_packed with the same state dict."""
    m = _student()
    enc = ErnieEncoder(vocab=1000, hidden=384, layers=4, heads=6, ffn=1536, max_pos=513, num_labels=2).to(DEV)
    enc.load_state_dict(m.state_dict())
    ids, _ = _batch(32, 128, seed=3)
    pk = _packed(ids)
    with torch.no_grad():
        got = m.forward_packed(*pk)
        want = enc.forward_packed(*pk)
    assert torch.equal(got, want), float((got - want).abs().max())


def _train(m, opt, pk, label):
    opt.zero_grad(set_to_none=False)
    loss = F.cross_entropy(m.forward_packed(*pk), label)
    loss.backward()
    opt.step()
    return loss


def test_packed_student_step_deterministic_and_graph_replay():
    ids, label = _batch()
    pk = _packed(ids)
    runs = []
    for _ in range(2):
        m = _student()
        opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)
        for _ in range(2):
            _train(m, opt, pk, label)
        runs.append({k: v.clone() for k, v in m.state_dict().items()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k
    m = _student()
    opt = torch.optim.AdamW(m.parameters(), 1e-4, capturable=True)
    ops.reset_fallbacks()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _train(m, opt, pk, label)
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
        gl = _train(m, opt, pk, label)
    restore()
    el = _train(m, opt, pk, label).clone()
    eager = {k: v.clone() for k, v in m.state_dict().items()}
    restore()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gl, el)
    for k, v in m.state_dict().items():
        assert torch.equal(v, eager[k]), k


def test_packed_student_dropout_gradients_match_float32_torch():
    """p = 0.1: the packed step against the float32 functional encoder with the reference masks of each site.  The
    hidden sites index packed rows and the probabilities use the 512 stride, so the padded reference takes the masks
    scattered to the padded positions."""
    m = _student(hidden_dropout=P, attention_dropout=P)
    ids, label = _batch(16, 128)
    pk = _packed(ids)
    seed, off = torch.cuda.initial_seed(), _gen().get_offset()
    ops.reset_fallbacks()
    F.cross_entropy(m.forward_packed(*pk), label).backward()
    assert ops.fallbacks() == {}
    assert _gen().get_offset() == off + 4 * (2 + 3 * len(m.layers))
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    # padded position of every packed row, and the packed-index masks scattered there
    b, l = ids.shape
    keep = ids != 0
    kept = keep.clone()
    kept[:, 0] = True
    bi, ii = kept.nonzero(as_tuple=True)                              # row-major: the packing order
    c, nh = m.hidden, m.heads

    def zf(o, shape):
        if shape == (b, l, c):                                        # a hidden site over the packed rows
            t = bi.numel()
            z = ops.dropout_keep_reference(seed, o, torch.arange(t * c, device=DEV), P).view(t, c).float()
            out = torch.zeros(b, l, c, device=DEV)
            out[bi, ii] = z * _scale(P)
            return out
        if shape == (b, nh, l, l):                                     # probabilities: positions within the sequence
            pos = torch.cumsum(kept, 1) - 1                           # packed position of each kept token
            hh = torch.arange(nh, device=DEV).view(1, -1, 1, 1)
            pi = pos.view(b, 1, l, 1).clamp_min(0)
            pj = pos.view(b, 1, 1, l).clamp_min(0)
            idx = ((torch.arange(b, device=DEV).view(-1, 1, 1, 1) * nh + hh) * 512 + pi) * 512 + pj
            return ops.dropout_keep_reference(seed, o, idx, P).float() * _scale(P)
        n = shape[0] * shape[1]                                        # pooled [B, C]
        return ops.dropout_keep_reference(seed, o, torch.arange(n, device=DEV), P).view(shape).float() * _scale(P)

    import test_dropout_gpu
    orig = test_dropout_gpu._z
    test_dropout_gpu._z = lambda s, o, shape, p=P: zf(o, tuple(shape)).double()
    try:
        ref = _functional_encoder_dropout(m, ids, keep, seed, off, P)
    finally:
        test_dropout_gpu._z = orig
    F.cross_entropy(ref, label).backward()
    worst = 0.0
    for n, p in m.named_parameters():
        r = float((got[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30))
        worst = max(worst, r)
        assert r < 0.03, "%s: relative L2 error %.4f" % (n, r)
    print("worst relative gradient error (packed, dropout) %.4f" % worst)


def test_distill_example_ernie_packed_on_gpu():
    p = subprocess.run([sys.executable, "examples/distill/nlp/distill.py", "--model", "ernie", "--packed", "--epochs",
                        "2", "--vocab", "400"], cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600,
                       text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", p.stdout)]
    assert len(losses) >= 4 and min(losses[-2:]) < losses[0], p.stdout
