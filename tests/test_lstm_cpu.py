"""CPU checks of the bidirectional LSTM op (ops/rnn.py reference path), the BiLSTM student and its examples."""
import os
import re
import subprocess
import sys

import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

from edl_b200 import ops
from edl_b200.models.small import BiLSTM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lstm(e, h, seed, dtype=torch.float32):
    torch.manual_seed(seed)
    return torch.nn.LSTM(e, h, batch_first=True, bidirectional=True).to(dtype)


def _params(m):
    return [getattr(m, n) for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0", "weight_ih_l0_reverse",
                                    "weight_hh_l0_reverse", "bias_ih_l0_reverse", "bias_hh_l0_reverse")]


def _torch_packed(m, x, lengths):
    """float64 nn.LSTM over pack_padded_sequence(enforce_sorted=False): (y zero past each length, h_n)."""
    packed = pack_padded_sequence(x, lengths, batch_first=True, enforce_sorted=False)
    out, (hn, _) = m(packed)
    y, _ = pad_packed_sequence(out, batch_first=True, total_length=x.shape[1])
    return y, hn


@pytest.mark.parametrize("B,L,E,H,kind", [(5, 7, 6, 4, "random"), (4, 9, 8, 16, "one"), (3, 6, 5, 8, "full"),
                                          (6, 12, 16, 32, "random"), (7, 5, 3, 128, "random")])
def test_reference_matches_packed_nn_lstm(B, L, E, H, kind):
    g = torch.Generator().manual_seed(B * 100 + L)
    if kind == "one":
        lengths = torch.ones(B, dtype=torch.long)
    elif kind == "full":
        lengths = torch.full((B,), L, dtype=torch.long)
    else:
        lengths = torch.randint(1, L + 1, (B,), generator=g)
        lengths[0], lengths[-1] = 1, L              # unsorted, extremes included
    m64 = _lstm(E, H, 1, torch.float64)
    x = torch.randn(B, L, E, generator=g, dtype=torch.float64)
    x64 = x.clone().requires_grad_(True)
    y_ref, hn_ref = _torch_packed(m64, x64, lengths)
    w_y = torch.randn(y_ref.shape, generator=g, dtype=torch.float64)
    w_h = torch.randn(hn_ref.shape, generator=g, dtype=torch.float64)
    ((y_ref * w_y).sum() + (hn_ref * w_h).sum()).backward()

    m32 = _lstm(E, H, 1)
    x32 = x.float().requires_grad_(True)
    y, hn = ops.lstm(x32, lengths, _params(m32))
    ((y.double() * w_y).sum() + (hn.double() * w_h).sum()).backward()
    tol = dict(rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(y.double(), y_ref, **tol)
    torch.testing.assert_close(hn.double(), hn_ref, **tol)
    torch.testing.assert_close(x32.grad.double(), x64.grad, **tol)
    for p32, p64 in zip(_params(m32), _params(m64)):
        assert p32.grad.dtype == p32.dtype
        torch.testing.assert_close(p32.grad.double(), p64.grad, **tol)


def test_length_zero_gives_zeros():
    B, L, E, H = 4, 6, 5, 8
    m = _lstm(E, H, 2)
    lengths = torch.tensor([0, 3, 0, 6])
    x = torch.randn(B, L, E).requires_grad_(True)
    y, hn = ops.lstm(x, lengths, _params(m))
    (y.sum() + hn.sum()).backward()
    for b in (0, 2):
        assert torch.equal(y[b], torch.zeros_like(y[b]))
        assert torch.equal(hn[:, b], torch.zeros_like(hn[:, b]))
        assert torch.equal(x.grad[b], torch.zeros_like(x.grad[b]))
    # the others are what the batch without the empty samples gives
    keep = torch.tensor([1, 3])
    y2, hn2 = ops.lstm(x.detach()[keep], lengths[keep], _params(m))
    torch.testing.assert_close(y.detach()[keep], y2)
    torch.testing.assert_close(hn.detach()[:, keep], hn2)
    # a batch of only empty samples: zero parameter gradients
    m.zero_grad()
    y, hn = ops.lstm(torch.randn(2, L, E), torch.zeros(2, dtype=torch.long), _params(m))
    (y.sum() + hn.sum()).backward()
    for p in _params(m):
        assert p.grad is None or torch.count_nonzero(p.grad) == 0


def test_padded_rows_do_not_matter():
    B, L, E, H = 3, 8, 4, 8
    m = _lstm(E, H, 3)
    lengths = torch.tensor([3, 8, 5])
    x = torch.randn(B, L, E)
    x2 = x.clone()
    for b in range(B):
        x2[b, lengths[b]:] = float("nan")
    y, hn = ops.lstm(x, lengths, _params(m))
    y2, hn2 = ops.lstm(x2, lengths, _params(m))
    assert torch.equal(y, y2) and torch.equal(hn, hn2)
    for b in range(B):
        assert torch.equal(y[b, lengths[b]:], torch.zeros_like(y[b, lengths[b]:]))


def test_bilstm_state_dict_round_trip():
    a = BiLSTM(vocab_size=50, emb_dim=16, hidden=8)
    sd = a.state_dict()
    lstm_sd = {k[len("lstm."):]: v for k, v in sd.items() if k.startswith("lstm.")}
    ref = torch.nn.LSTM(16, 8, batch_first=True, bidirectional=True)
    ref.load_state_dict(lstm_sd)                                  # nn.LSTM names, unchanged
    b = BiLSTM(vocab_size=50, emb_dim=16, hidden=8)
    b.load_state_dict(sd)
    ids = torch.randint(1, 50, (4, 10))
    ids[0, 6:] = 0
    assert torch.equal(a(ids), b(ids))
    # the BiLSTM's final states are nn.LSTM's on the packed batch
    lengths = a.lengths(ids)
    assert lengths.tolist() == [6, 10, 10, 10]
    _, hn_ref = _torch_packed(ref, a.emb(ids), lengths)
    _, hn = ops.lstm(a.emb(ids), lengths, a.lstm_params())
    torch.testing.assert_close(hn, hn_ref, rtol=1e-5, atol=1e-6)


def _run(args, timeout=600):
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable] + args, cwd=ROOT, env=e, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       timeout=timeout, text=True)
    assert p.returncode == 0, p.stdout[-3000:]
    return p.stdout


def test_train_example_lstm_learns():
    out = _run(["examples/distill/nlp/train.py", "--model", "lstm", "--epochs", "3", "--samples", "128", "--vocab", "400",
                "--seq_len", "16"])
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", out)]
    assert len(losses) == 3 and losses[-1] < losses[0], out


def test_distill_example_lstm_learns():
    out = _run(["examples/distill/nlp/distill.py", "--model", "lstm", "--epochs", "2", "--vocab", "400"])
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", out)]
    assert len(losses) >= 4 and min(losses[-2:]) < losses[0], out
