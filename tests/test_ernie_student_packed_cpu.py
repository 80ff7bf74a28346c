"""Packed training of the Transformer student on the CPU: ErnieStudent.forward_packed against the padded student on the
same batch (logits and every parameter gradient, a masked token 0 and a length-1 sample included), with dropout against
a functional reference that applies dropout_keep_reference masks at the documented sites, and the --packed examples."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models.ernie import ErnieStudent, pack_sequences

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _student(**kw):
    torch.manual_seed(0)
    m = ErnieStudent(vocab=60, hidden=128, layers=2, heads=2, ffn=256, max_pos=40, num_labels=3, **kw)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    return m


def _batch():
    b, l = 5, 17
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(1, 60, (b, l), generator=g)
    ids[0, 12:] = 0
    ids[1, 0] = 0                                                    # token 0 masked: a query, not a key
    ids[1, 9:] = 0
    ids[2, 1:] = 0                                                   # a length-1 sample
    ids[4, 3:7] = 0                                                  # holes inside a sample
    pos = torch.arange(l).expand(b, l)
    seg = torch.randint(0, 2, (b, l), generator=g)
    return ids, pos, seg, ids != 0


def _grads(m, logits, w):
    m.zero_grad()
    (logits * w).sum().backward()
    return {n: p.grad.clone() for n, p in m.named_parameters()}


def test_packed_matches_padded_student():
    m = _student()
    ids, pos, seg, keep = _batch()
    packed = pack_sequences(ids, pos, seg, keep)
    assert packed[5] is not None                                     # the masked token 0 needs the key mask
    assert int(packed[3][3] - packed[3][2]) == 1
    w = torch.randn(ids.shape[0], 3)
    ref = m(ids, pos, seg, keep)
    g_ref = _grads(m, ref, w)
    got = m.forward_packed(*packed)
    g_got = _grads(m, got, w)
    assert torch.allclose(got, ref, rtol=1e-4, atol=1e-5)
    for n in g_ref:
        assert torch.allclose(g_got[n], g_ref[n], rtol=1e-3, atol=1e-6), n
        assert g_got[n].abs().sum() > 0, n
    with torch.no_grad():                                            # the encoder's packed inference forward
        enc = super(ErnieStudent, m).forward_packed(*packed)
    assert torch.allclose(got, enc, rtol=1e-5, atol=1e-6)


class _KeepMasks:
    """A stand-in for F.dropout whose k-th call applies the package's mask of (seed, 4 k) over the flat index of its
    input: the CPU sites then follow dropout_keep_reference, and the reference below rebuilds every mask itself."""

    def __init__(self, seed):
        self.seed, self.calls = seed, 0

    def z(self, k, shape, p):
        n = 1
        for d in shape:
            n *= d
        keep = ops.dropout_keep_reference(self.seed, 4 * k, torch.arange(n), p)
        return keep.float().view(shape) * torch.tensor(1.0 / (1.0 - p), dtype=torch.float32)

    def __call__(self, x, p=0.5, training=True, inplace=False):
        k, self.calls = self.calls, self.calls + 1
        return x * self.z(k, tuple(x.shape), p)


def _functional_packed(m, packed, zs, p):
    """The packed post-LN encoder from nn.functional ops, one sequence at a time for attention.  Site k's mask is
    zs.z(k, shape, p) at the documented indices: embedding output and both residual branches at packed row * C + col,
    the attention probabilities of sequence b at ((b H + h) M + i) M + j of a [B, H, M, M] mask (M = max_len), the
    pooled features at b * C + col."""
    ids, pos, seg, cu, max_len, key_mask = packed
    t, c, nh, nb = ids.numel(), m.hidden, m.heads, cu.numel() - 1
    d = c // nh
    cu = cu.tolist()
    site = iter(range(100))
    x = F.embedding(ids, m.word_emb) + F.embedding(pos, m.pos_emb) + F.embedding(seg, m.seg_emb)
    x = F.layer_norm(x, (c,), m.emb_ln_g, m.emb_ln_b, m.eps) * zs.z(next(site), (t, c), p)
    for lyr in m.layers:
        qkv = F.linear(x, lyr.qkv_w, lyr.qkv_b).view(t, 3, nh, d)
        za = zs.z(next(site), (nb, nh, max_len, max_len), p)
        outs = []
        for b in range(nb):
            s, e = cu[b], cu[b + 1]
            q, k, v = (qkv[s:e, i].transpose(0, 1) for i in range(3))          # [H, L, d]
            valid = torch.ones(e - s, dtype=torch.bool) if key_mask is None else key_mask[s:e] != 0
            sc = (q @ k.transpose(-1, -2) / d ** 0.5).masked_fill(~valid, float("-inf"))
            pr = torch.softmax(sc, -1).nan_to_num(0.0) * za[b, :, :e - s, :e - s]
            outs.append((pr @ v).transpose(0, 1).reshape(e - s, c))
        h = F.linear(torch.cat(outs), lyr.out_w, lyr.out_b) * zs.z(next(site), (t, c), p)
        x = F.layer_norm(h + x, (c,), lyr.ln1_g, lyr.ln1_b, m.eps)
        f = F.linear(F.gelu(F.linear(x, lyr.ffn1_w, lyr.ffn1_b)), lyr.ffn2_w, lyr.ffn2_b) * zs.z(next(site), (t, c), p)
        x = F.layer_norm(f + x, (c,), lyr.ln2_g, lyr.ln2_b, m.eps)
    pooled = torch.tanh(F.linear(x[cu[:-1]], m.pool_w, m.pool_b)) * zs.z(next(site), (nb, c), p)
    assert next(site) == 2 + 3 * m.num_layers                        # the documented number of sites
    return F.linear(pooled, m.cls_w, m.cls_b)


def test_packed_dropout_sites_match_functional_reference(monkeypatch):
    p = 0.2
    m = _student(hidden_dropout=p, attention_dropout=p).train()
    ids, pos, seg, keep = _batch()
    packed = pack_sequences(ids, pos, seg, keep)
    w = torch.randn(ids.shape[0], 3)
    fake = _KeepMasks(seed=1234)
    monkeypatch.setattr(torch.nn.functional, "dropout", fake)
    got = m.forward_packed(*packed)
    assert fake.calls == 2 + 3 * m.num_layers
    g_got = _grads(m, got, w)
    monkeypatch.undo()
    ref = _functional_packed(m, packed, _KeepMasks(seed=1234), p)
    g_ref = _grads(m, ref, w)
    assert torch.allclose(got, ref, rtol=1e-4, atol=1e-5)
    for n in g_ref:
        assert torch.allclose(g_got[n], g_ref[n], rtol=1e-3, atol=1e-6), n
    # the masks matter: a different seed gives different logits
    monkeypatch.setattr(torch.nn.functional, "dropout", _KeepMasks(seed=99))
    assert not torch.allclose(m.forward_packed(*packed), got)


def test_packed_eval_draws_nothing(monkeypatch):
    m = _student(hidden_dropout=0.3, attention_dropout=0.3).eval()
    ids, pos, seg, keep = _batch()
    fake = _KeepMasks(seed=1)
    monkeypatch.setattr(torch.nn.functional, "dropout", fake)
    with torch.no_grad():
        m.forward_packed(*pack_sequences(ids, pos, seg, keep))
    assert fake.calls == 0


def test_attention_varlen_trainable_reference_gradients():
    """The CPU op (float32 reference under autograd) against attention_trainable per sequence."""
    torch.manual_seed(2)
    lens, heads = [5, 1, 9], 2
    cu = torch.tensor([0, 5, 6, 15], dtype=torch.int32)
    qkv = torch.randn(15, 3 * heads * 64, requires_grad=True)
    km = torch.ones(15, dtype=torch.uint8)
    km[6] = 0
    out = ops.attention_varlen_trainable(qkv, cu, 9, heads, km)
    do = torch.randn_like(out)
    (gq,) = torch.autograd.grad(out, qkv, do)
    for s, e in ((0, 5), (5, 6), (6, 15)):
        x = qkv.detach()[s:e].clone().requires_grad_(True)
        o = ops.attention_trainable(x, km[s:e].view(1, -1), 1, e - s, heads)
        assert torch.allclose(o, out[s:e], atol=1e-6)
        (g,) = torch.autograd.grad(o, x, do[s:e])
        assert torch.allclose(g, gq[s:e], atol=1e-6)
    with pytest.raises(ValueError):
        ops.attention_varlen_trainable(qkv, cu, 9, heads, km, dropout_p=1.0)


def _run(args, timeout=900):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable] + args, cwd=ROOT, env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=timeout, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    return p.stdout


def test_train_example_ernie_packed_runs():
    out = _run(["examples/distill/nlp/train.py", "--model", "ernie", "--packed", "--epochs", "2", "--samples", "64",
                "--vocab", "400", "--seq_len", "16"])
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", out)]
    assert len(losses) == 2 and all(v == v for v in losses), out


def test_distill_example_ernie_packed_learns():
    out = _run(["examples/distill/nlp/distill.py", "--model", "ernie", "--packed", "--epochs", "2", "--vocab", "400"])
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", out)]
    assert len(losses) >= 4 and min(losses[-2:]) < losses[0], out


def test_packed_flag_needs_ernie():
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, "examples/distill/nlp/train.py", "--model", "bow", "--packed"], cwd=ROOT, env=e,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=300, text=True)
    assert p.returncode != 0 and "--packed needs --model ernie" in p.stdout
