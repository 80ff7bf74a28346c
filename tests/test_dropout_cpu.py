"""Dropout on the CPU: the host statement of the mask (ops.transformer.dropout_keep_reference) against the Random123
Philox4x32-10 known answers and its statistics, the probability checks, ErnieStudent with dropout (training differs
run to run, eval() is the encoder, no new state), and the --dropout examples."""
import math
import os
import re
import subprocess
import sys

import pytest
import torch

from edl_b200 import ops
from edl_b200.models.ernie import ErnieEncoder, ErnieStudent
from edl_b200.ops.transformer import philox4x32_10

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Random123 kat_vectors: key -> counter -> output
KAT = [((0, 0), (0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff, 0xffffffff), (0xffffffff,) * 4, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0xa4093822, 0x299f31d0), (0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("key,ctr,out", KAT)
def test_philox_known_answers(key, ctr, out):
    t = lambda v: torch.tensor([v], dtype=torch.int64)   # noqa: E731
    got = philox4x32_10(tuple(map(t, key)), tuple(map(t, ctr)))
    assert tuple(int(w) for w in got) == out


def test_keep_reference_reads_the_documented_word():
    """Element n uses key (seed lo, seed hi), counter (n / 4 lo, n / 4 hi, offset lo, offset hi) and word n % 4: the
    elements of the first known-answer group are kept iff their word >= floor(p 2^32); and a group with both counter
    halves and both key halves nonzero picks the words of that Philox evaluation."""
    for p in (0.3, 0.5, 0.9):
        t = int(p * 2 ** 32)
        keep = ops.dropout_keep_reference(0, 0, torch.arange(4, dtype=torch.int64), p)
        assert keep.tolist() == [w >= t for w in KAT[0][2]]
    seed, offset, group = 0x299f31d0a4093822, 0x0370734413198a2e, 0x05a308d3243f6a88
    words = philox4x32_10(tuple(torch.tensor([v], dtype=torch.int64) for v in (0xa4093822, 0x299f31d0)),
                          tuple(torch.tensor([v], dtype=torch.int64) for v in (0x243f6a88, 0x05a308d3, 0x13198a2e,
                                                                                0x03707344)))
    keep = ops.dropout_keep_reference(seed, offset, torch.arange(4, dtype=torch.int64) + 4 * group, 0.5)
    assert keep.tolist() == [int(w) >= 2 ** 31 for w in words]


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate_and_independence(p):
    n = 10_000_000
    idx = torch.arange(n, dtype=torch.int64)
    a = ops.dropout_keep_reference(12345, 8, idx, p)
    rate = float(a.double().mean())
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(rate - (1 - p)) < 6 * sigma, (rate, 1 - p)
    # the next site's offset (o + 4) gives an unrelated mask: agreement rate is that of independent draws
    b = ops.dropout_keep_reference(12345, 12, idx, p)
    agree = float((a == b).double().mean())
    q = (1 - p) ** 2 + p ** 2
    assert abs(agree - q) < 6 * math.sqrt(q * (1 - q) / n), (agree, q)


@pytest.mark.parametrize("p", [1.0, -0.1, 1.5, float("nan")])
def test_bad_probability_raises(p):
    x = torch.ones(8)
    with pytest.raises(ValueError):
        ops.dropout(x, p)
    with pytest.raises(ValueError):
        ops.dropout_keep_reference(0, 0, torch.arange(4), p)
    with pytest.raises(ValueError):
        ErnieStudent(vocab=60, hidden=128, layers=1, heads=2, ffn=256, max_pos=40, num_labels=2, hidden_dropout=p)


def test_dropout_op_cpu():
    x = torch.randn(1000)
    assert ops.dropout(x, 0.0) is x and ops.dropout(x, 0.5, training=False) is x
    y = ops.dropout(x, 0.25)
    kept = y != 0
    assert torch.allclose(y[kept], x[kept] / 0.75)


def _student(**kw):
    torch.manual_seed(0)
    m = ErnieStudent(vocab=60, hidden=128, layers=2, heads=2, ffn=256, max_pos=40, num_labels=3, **kw)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    return m


def test_student_dropout_cpu():
    m = _student(hidden_dropout=0.1, attention_dropout=0.1)
    ids = torch.randint(1, 60, (3, 17))
    ids[0, 12:] = 0
    a, b = m(ids), m(ids)
    assert not torch.equal(a, b)                                       # training: fresh masks per forward
    a.sum().backward()
    assert all(p.grad is not None for p in m.parameters())
    assert set(m.state_dict()) == set(_student().state_dict())        # no new parameters or buffers
    enc = ErnieEncoder(vocab=60, hidden=128, layers=2, heads=2, ffn=256, max_pos=40, num_labels=3)
    enc.load_state_dict(m.state_dict())
    m.eval()
    with torch.no_grad():
        assert torch.equal(m(ids), m(ids))
        assert torch.allclose(m(ids), enc(ids, torch.arange(17).expand(3, 17), torch.zeros_like(ids), ids != 0),
                              rtol=1e-6, atol=1e-6)


def _run(args, timeout=900):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable] + args, cwd=ROOT, env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=timeout, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    return [float(v) for v in re.findall(r"loss ([0-9.]+)", p.stdout)]


def test_examples_with_dropout():
    losses = _run(["examples/distill/nlp/train.py", "--model", "ernie", "--dropout", "0.1", "--epochs", "2",
                   "--samples", "64", "--vocab", "400", "--seq_len", "16"])
    assert len(losses) == 2 and all(v == v for v in losses)
    losses = _run(["examples/distill/nlp/distill.py", "--model", "ernie", "--dropout", "0.1", "--epochs", "2",
                   "--vocab", "400"])
    assert len(losses) >= 4 and all(v == v for v in losses)
