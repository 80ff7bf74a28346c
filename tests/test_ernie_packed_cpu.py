"""Packed variable-length batches for the ERNIE teacher on CPU: the packing rules, the packed reference forward against
the padded one on every mask kind, and a teacher server batching requests of different sequence lengths."""
import threading

import numpy as np
import pytest
import torch

from edl_b200 import ops
from edl_b200.models import ernie, teacher_zoo

KINDS = ("full", "right", "holes", "one", "empty", "cls_masked")


def _mask(kind, l, gen):
    m = torch.zeros(l)
    if kind == "full":
        m[:] = 1
    elif kind == "right":
        m[:int(torch.randint(1, l + 1, (1,), generator=gen))] = 1
    elif kind == "holes":
        m[:] = (torch.rand(l, generator=gen) > 0.5).float()
        m[0] = 1
    elif kind == "one":
        m[int(torch.randint(1, l, (1,), generator=gen))] = 1        # one real token that is not [CLS]
    elif kind == "cls_masked":
        m[1:] = (torch.rand(l - 1, generator=gen) > 0.3).float()
    return m


def _batch(kinds, l, seed, vocab=1000):
    gen = torch.Generator().manual_seed(seed)
    b = len(kinds)
    ids = torch.randint(0, vocab, (b, l), generator=gen)
    pos = torch.arange(l).expand(b, l).contiguous()
    seg = torch.randint(0, 2, (b, l), generator=gen)
    mask = torch.stack([_mask(k, l, gen) for k in kinds])
    return ids, pos, seg, mask


def test_pack_rules():
    l = 11
    ids, pos, seg, mask = _batch(KINDS, l, 0)
    pids, ppos, pseg, cu, max_len, key_mask = ernie.pack_sequences(ids, pos, seg, mask)
    keep = mask != 0
    keep[:, 0] = True
    lens = keep.sum(1)
    assert cu.dtype == torch.int32 and cu.tolist() == [0] + torch.cumsum(lens, 0).tolist()
    assert max_len == int(lens.max()) and len(pids) == int(lens.sum())
    for b in range(len(KINDS)):
        s, e = int(cu[b]), int(cu[b + 1])
        assert torch.equal(pids[s:e], ids[b][keep[b]]) and torch.equal(ppos[s:e], pos[b][keep[b]])
        assert torch.equal(pseg[s:e], seg[b][keep[b]])
        assert pids[s] == ids[b, 0]                                     # [CLS] first, always kept
    assert (lens[KINDS.index("empty")], lens[KINDS.index("one")], lens[KINDS.index("full")]) == (1, 2, l)
    # key_mask only when a kept token is masked: a sample whose [CLS] token is masked
    assert key_mask is not None and key_mask.dtype == torch.uint8
    assert torch.equal(key_mask, mask[keep].to(torch.uint8))
    no_cls_masked = [k for k in KINDS if k not in ("empty", "one", "cls_masked")]
    packed = ernie.pack_sequences(*_batch(no_cls_masked, l, 1))
    assert packed[5] is None
    # numpy [B, L, 1] feeds pack the same
    np_feeds = [t.numpy()[..., None] for t in (ids, pos, seg, mask)]
    again = ernie.pack_sequences(*np_feeds)
    assert all(torch.equal(a, b) for a, b in zip(again[:4], (pids, ppos, pseg, cu))) and again[4] == max_len
    # lengths: at most 512 kept tokens, and at most the position table
    long = torch.ones(2, 513)
    with pytest.raises(ValueError):
        ernie.pack_sequences(long.long(), long.long(), long.long(), long)
    ernie.pack_sequences(long.long(), long.long(), long.long(), torch.cat([long[:, :512], torch.zeros(2, 1)], 1))
    with pytest.raises(ValueError):
        ernie.pack_sequences(ids, pos, seg, torch.ones(len(KINDS), l), max_positions=l - 1)


def test_attention_varlen_reference_is_per_sequence_attention():
    gen = torch.Generator().manual_seed(3)
    lens = [1, 5, 37, 64, 2]
    h = 2
    cu = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32)
    t = int(cu[-1])
    qkv = torch.randn(t, 3 * h * 64, generator=gen)
    km = (torch.rand(t, generator=gen) > 0.3).to(torch.uint8)
    km[int(cu[3]):int(cu[4])] = 0                                     # an all-masked sequence
    for key_mask in (None, km):
        got = ops.attention_varlen(qkv, cu, max(lens), h, key_mask)
        assert got.shape == (t, h * 64)
        for b, n in enumerate(lens):
            s = int(cu[b])
            m = None if key_mask is None else key_mask[s:s + n].view(1, n)
            want = ops.attention(qkv[s:s + n], m, 1, n, h)
            assert torch.equal(got[s:s + n], want)
    assert torch.equal(got[int(cu[3]):int(cu[4])], torch.zeros(lens[3], h * 64))


@pytest.mark.parametrize("kind", KINDS)
def test_forward_packed_equals_padded(kind):
    torch.manual_seed(0)
    model = ernie.ernie_tiny()
    l = 24
    feeds = _batch([kind] * 4, l, KINDS.index(kind) + 10)
    packed = ernie.pack_sequences(*feeds)
    got = model.forward_packed(*packed)
    assert got.dtype == torch.float32 and got.shape == (4, 2)
    for b in range(4):
        want = model(*(t[b:b + 1] for t in feeds))
        assert torch.allclose(got[b:b + 1], want, atol=1e-5), (kind, b, got[b], want)


def _requests(lens, n_per, seed):
    """Requests as a client sends them: [n, L, 1] arrays, one L per request, masks of mixed kinds."""
    gen = torch.Generator().manual_seed(seed)
    reqs = []
    for i, l in enumerate(lens):
        kinds = [KINDS[(i * n_per + j) % len(KINDS)] for j in range(n_per)]
        ids, pos, seg, mask = _batch(kinds, l, int(torch.randint(0, 1 << 30, (1,), generator=gen)))
        reqs.append([ids.numpy()[..., None], pos.numpy()[..., None], seg.numpy()[..., None],
                     mask.numpy().astype(np.float32)[..., None]])
    return reqs


def test_server_batches_mixed_lengths():
    from edl_b200.distill.teacher_server import TeacherServer

    torch.manual_seed(0)
    model, feeds, fetches, shapes = teacher_zoo.build("ernie_tiny")
    srv = TeacherServer(model, feeds, fetches, shapes)
    reqs = _requests([16, 24], 3, 4)
    slots = [{"feeds": dict(zip(feeds, r)), "done": threading.Event(), "out": None, "err": None}
             for r in reqs]
    srv._run_batch(slots)
    for s, r in zip(slots, reqs):
        assert s["done"].is_set() and s["out"]["logits"].shape == (3, 2)
        for i in range(3):
            want = model(*(torch.from_numpy(a[i:i + 1]) for a in r))[0].numpy()
            assert np.allclose(s["out"]["logits"][i], want, atol=1e-5), (s["out"]["logits"][i], want)


def test_server_mixed_lengths_end_to_end():
    from edl_b200.distill.distill_reader import DistillReader
    from edl_b200.distill.teacher_server import TeacherServer

    torch.manual_seed(0)
    model, feeds, fetches, shapes = teacher_zoo.build("ernie_tiny")
    data = []
    for r in _requests([16, 24] * 4, 3, 5):
        for j in range(3):
            data.append(tuple(a[j] for a in r) + (np.array([len(data)], np.int64),))
    with TeacherServer(model, feeds, fetches, shapes, max_wait_ms=20.0) as srv:
        dr = DistillReader(ins=feeds + ["label"], predicts=["logits"])
        dr.set_teacher_batch_size(3)                 # one request per sample group of one length
        dr.set_fixed_teacher([srv.endpoint])
        r = dr.set_sample_list_generator(lambda: [data[i:i + 3] for i in range(0, len(data), 3)])
        n = 0
        for batch in r():
            for ids, pos, seg, mask, label, logits in batch:
                want = model(*(torch.from_numpy(t)[None] for t in (ids, pos, seg, mask)))[0].numpy()
                assert np.allclose(logits, want, atol=1e-5), (logits, want)
                n += 1
        dr.stop()
    assert n == len(data)
