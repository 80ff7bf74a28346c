"""Transformer student (models/ernie.py ErnieStudent) on the CPU: gradients against an independent float32 encoder built
from torch.nn.functional, the state-dict hand-off to ErnieEncoder, and the --model ernie examples."""
import os
import re
import subprocess
import sys

import torch
import torch.nn.functional as F

from edl_b200.models.ernie import ErnieEncoder, ErnieStudent, ernie_student

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _functional_encoder(m, ids, pos, seg, keep):
    """Post-LN BERT encoder from nn.functional ops, reading the student's parameters."""
    b, l = ids.shape
    c, nh = m.hidden, m.heads
    d = c // nh
    x = F.embedding(ids, m.word_emb) + F.embedding(pos, m.pos_emb) + F.embedding(seg, m.seg_emb)
    x = F.layer_norm(x, (c,), m.emb_ln_g, m.emb_ln_b, m.eps)
    bias = torch.zeros(b, 1, 1, l, device=ids.device).masked_fill(~keep.view(b, 1, 1, l), float("-inf"))
    for lyr in m.layers:
        q, k, v = F.linear(x, lyr.qkv_w, lyr.qkv_b).view(b, l, 3, nh, d).unbind(2)
        q, k, v = (t.transpose(1, 2) for t in (q, k, v))
        p = torch.softmax(q @ k.transpose(-1, -2) / d ** 0.5 + bias, -1)
        o = (p @ v).transpose(1, 2).reshape(b, l, c)
        x = F.layer_norm(F.linear(o, lyr.out_w, lyr.out_b) + x, (c,), lyr.ln1_g, lyr.ln1_b, m.eps)
        f = F.gelu(F.linear(x, lyr.ffn1_w, lyr.ffn1_b))
        x = F.layer_norm(F.linear(f, lyr.ffn2_w, lyr.ffn2_b) + x, (c,), lyr.ln2_g, lyr.ln2_b, m.eps)
    pooled = torch.tanh(F.linear(x[:, 0], m.pool_w, m.pool_b))
    return F.linear(pooled, m.cls_w, m.cls_b)


def _tiny_student():
    torch.manual_seed(0)
    m = ErnieStudent(vocab=60, hidden=128, layers=2, heads=2, ffn=256, max_pos=40, num_labels=3)
    with torch.no_grad():                       # non-trivial LayerNorm and bias parameters
        for n, p in m.named_parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    return m


def test_student_gradients_match_functional_encoder():
    m = _tiny_student()
    b, l = 3, 17
    ids = torch.randint(1, 60, (b, l))
    ids[0, 12:] = 0
    ids[2, 5:] = 0
    pos = torch.arange(l).expand(b, l)
    seg = torch.randint(0, 2, (b, l))
    keep = ids != 0
    w = torch.randn(b, 3)
    (m(ids, pos, seg, keep) * w).sum().backward()
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad()
    ref_logits = _functional_encoder(m, ids, pos, seg, keep)
    (ref_logits * w).sum().backward()
    assert torch.allclose(m(ids, pos, seg, keep), ref_logits, rtol=1e-4, atol=1e-5)
    for n, p in m.named_parameters():
        assert torch.allclose(got[n], p.grad, rtol=1e-3, atol=1e-5), n
        assert got[n].abs().sum() > 0 or n in ("pos_emb",), n
    # the ids-only form builds positions 0.., segment 0 and the mask ids != 0
    assert torch.equal(m(ids), m(ids, pos, torch.zeros_like(ids), keep))


def test_student_state_dict_serves_in_encoder():
    m = _tiny_student()
    enc = ErnieEncoder(vocab=60, hidden=128, layers=2, heads=2, ffn=256, max_pos=40, num_labels=3)
    enc.load_state_dict(m.state_dict())
    assert set(enc.state_dict()) == set(m.state_dict())
    ids = torch.randint(1, 60, (4, 9))
    ids[1, 4:] = 0
    pos, seg = torch.arange(9).expand(4, 9), torch.zeros_like(ids)
    with torch.no_grad():
        assert torch.allclose(enc(ids, pos, seg, ids != 0), m(ids), rtol=1e-6, atol=1e-6)


def test_ernie_student_config():
    m = ernie_student()
    assert (m.word_emb.shape, m.hidden, m.num_layers, m.heads, m.layers[0].ffn1_w.shape[0]) == \
        ((18000, 384), 384, 4, 6, 1536)
    assert all(p.requires_grad and p.dtype == torch.float32 for p in m.parameters())


def _run(args, timeout=900):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable] + args, cwd=ROOT, env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=timeout, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    return p.stdout


def test_train_example_ernie_runs():
    out = _run(["examples/distill/nlp/train.py", "--model", "ernie", "--epochs", "2", "--samples", "64", "--vocab",
                "400", "--seq_len", "16"])
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", out)]
    assert len(losses) == 2 and all(v == v for v in losses), out


def test_distill_example_ernie_learns():
    out = _run(["examples/distill/nlp/distill.py", "--model", "ernie", "--epochs", "2", "--vocab", "400"])
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", out)]
    assert len(losses) >= 4 and min(losses[-2:]) < losses[0], out
