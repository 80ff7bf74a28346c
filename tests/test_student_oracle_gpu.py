"""Whole ErnieStudent training steps held to the float64 layer-by-layer oracle (tests/student_oracle.py): padded and
packed batches, tile tails, dropout, gradients delivered into flat buckets with one FlatAdam step, and two negative
controls that the oracle must catch and name."""
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models.ernie import ErnieStudent, pack_sequences
from edl_b200.parallel.flat import FlatParams
from student_oracle import StudentRecorder

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
P = 0.1
STUDENT = dict(vocab=1000, hidden=384, layers=4, heads=6, ffn=1536, max_pos=513, num_labels=2)   # ernie_student
TAILS = dict(vocab=1000, hidden=320, layers=2, heads=5, ffn=1088, max_pos=513, num_labels=3)


def _gen():
    return torch.cuda.default_generators[0]


def _student(cfg, seed=0, p=0.0):
    torch.manual_seed(seed)
    m = ErnieStudent(**cfg, hidden_dropout=p, attention_dropout=p)
    with torch.no_grad():
        for t in m.parameters():
            if t.dim() == 1:
                t.add_(torch.randn_like(t) * 0.05)
    return m.to(DEV)


def _padded(b, l, labels, seed=0):
    """ids [B, L] with random lengths, sample 1 with its token 0 masked and sample 2 without a valid token."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    ids = torch.randint(1, 1000, (b, l), device=DEV, generator=g)
    lens = torch.randint(1, l + 1, (b, 1), device=DEV, generator=g)
    ids[torch.arange(l, device=DEV).unsqueeze(0) >= lens] = 0
    if b > 2:
        ids[1] = torch.randint(1, 1000, (l,), device=DEV, generator=g)
        ids[1, 0] = 0
        ids[2] = 0
    return ids, torch.randint(0, labels, (b,), device=DEV, generator=g)


def _packed(seed=0):
    """Lengths 1, 63, 64, 65, 128, 41 and 1 (T = 363): the first sample without a valid token (kept as its [CLS] row,
    fully key-masked), token 0 of the 65-long sample masked, and a length-1 sequence in the last packed row."""
    lens = [1, 63, 64, 65, 128, 41, 1]
    l = max(lens)
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, 1000, (len(lens), l), generator=g)
    mask = (torch.arange(l).unsqueeze(0) < torch.tensor(lens).unsqueeze(1)).to(torch.uint8)
    mask[3, 0] = 0
    mask[0] = 0
    pos = torch.arange(l).expand(len(lens), l)
    ids_p, pos_p, seg_p, cu, max_len, key_mask = pack_sequences(ids, pos, torch.zeros_like(ids), mask)
    assert ids_p.numel() == 363 and cu.diff().tolist() == lens and key_mask is not None
    labels = torch.randint(0, 2, (len(lens),), generator=g).to(DEV)
    return (ids_p.to(DEV), pos_p.to(DEV), seg_p.to(DEV), cu.to(DEV), max_len, key_mask.to(DEV)), labels


def _record(m, labels, run):
    ops.reset_fallbacks()
    off = _gen().get_offset()
    with StudentRecorder(m) as rec:
        F.cross_entropy(run(), labels).backward()
    assert ops.fallbacks() == {}
    per_step = 4 * (2 + 3 * len(m.layers)) if m.hidden_dropout > 0 else 0
    assert _gen().get_offset() == off + per_step
    if per_step:
        assert rec.draws[0][1] == off
    return rec


def test_student_padded_step():
    m = _student(STUDENT)
    ids, labels = _padded(16, 128, 2)
    _record(m, labels, lambda: m(ids)).check(labels)


def test_student_tails_step():
    m = _student(TAILS, seed=1)
    ids, labels = _padded(3, 77, 3, seed=1)
    _record(m, labels, lambda: m(ids)).check(labels)


def test_student_packed_step():
    m = _student(STUDENT, seed=2)
    feed, labels = _packed(2)
    _record(m, labels, lambda: m.forward_packed(*feed)).check(labels)


def test_student_padded_dropout_step():
    m = _student(STUDENT, seed=3, p=P)
    ids, labels = _padded(16, 128, 2, seed=3)
    _record(m, labels, lambda: m(ids)).check(labels)


def test_student_packed_dropout_step():
    m = _student(STUDENT, seed=4, p=P)
    feed, labels = _packed(4)
    _record(m, labels, lambda: m.forward_packed(*feed)).check(labels)


def test_student_flat_buckets_and_adam():
    """Every gradient delivered into its fp32 bucket window (weights through the weight-gradient hand-off), then one
    FlatAdam step against the float64 Adam rule."""
    from test_optim_gpu import assert_close, f32, ref_adam

    m = _student(STUDENT, seed=5)
    flat = FlatParams(m)
    assert set(flat.groups) == {torch.float32}
    opt = ops.FlatAdam(flat, lr=1e-3, weight_decay=0.01, decoupled=True)
    ids, labels = _padded(16, 128, 2, seed=5)
    opt.zero_grad()
    rec = _record(m, labels, lambda: m(ids))
    torch.cuda.synchronize()
    rec.check(labels)
    g = flat.groups[torch.float32]
    w0, grad = g.param.clone(), g.grad.clone()
    opt.step()
    torch.cuda.synchronize()
    st = opt.state[torch.float32]
    zero = torch.zeros_like(w0)
    w, m1, v1, tw, tm, tv = ref_adam(w0, zero, zero, grad, 1, f32(1e-3), f32(0.9), f32(0.999), f32(1e-8), f32(0.01),
                                     True)       # the kernel's fp32 hyperparameters
    assert_close(g.param, w, tw, "FlatAdam parameters")
    assert_close(st["m"], m1, tm, "FlatAdam m")
    assert_close(st["v"], v1, tv, "FlatAdam v")


def test_student_oracle_negative_controls():
    """One bf16 ulp on one recorded weight-gradient element, and one site's Z rebuilt at the neighbouring offset, must
    each fail and name the layer."""
    cfg = dict(STUDENT, layers=2)
    m = _student(cfg, seed=6, p=P)
    ids, labels = _padded(8, 128, 2, seed=6)
    rec = _record(m, labels, lambda: m(ids))
    rec.check(labels)
    w = rec.bwd[("layers.1.ffn", "ffn2 wgrad")]["out"]
    bits = w.view(torch.int16)
    bits.view(-1)[5] += 1
    with pytest.raises(AssertionError, match=r"layers\.1\.ffn ffn2 wgrad"):
        rec.check(labels)
    bits.view(-1)[5] -= 1
    rec.check(labels)
    a = rec.fwd[("layers.0.attention", "attention")]
    seed, off, p = a["drop"]
    a["drop"] = (seed, off + 4, p)
    with pytest.raises(AssertionError, match=r"layers\.0\.attention forward"):
        rec.check(labels)
