"""Packed variable-length batches of the ERNIE teacher on the GPU kernels.

The varlen attention is checked element-wise against the float64 bound of ``test_ernie_gpu.attention_ref`` applied to
each sequence, with NaN rows around the operand and sentinel rows around the output.  Isolation: a sequence's output
bits do not change whatever the other sequences' rows hold.  The packed ernie_base forward is checked against the fp32
torch forward and the padded kernel forward, and a CUDA teacher server batches requests of different lengths."""
import threading

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from edl_b200 import ops  # noqa: E402
from edl_b200.models import ernie, teacher_zoo  # noqa: E402
from f64_bounds import check_bf16, guarded  # noqa: E402
from test_ernie_gpu import _inputs, _torch_forward32, attention_ref  # noqa: E402

DEV = torch.device("cuda", 0)


def _length_set(name):
    gen = torch.Generator().manual_seed(len(name))
    return {
        "one": [1],
        "max": [512],
        "edges": [1, 7, 63, 64, 65, 127, 128, 129, 200, 256, 511, 512],
        "seeded": torch.randint(1, 513, (16,), generator=gen).tolist(),
        "short": torch.randint(1, 9, (300,), generator=gen).tolist(),
    }[name]


def _cu(lens):
    return torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=DEV)


def _key_mask(lens, gen):
    """Holes in every sequence, a masked token 0 in every third, every fifth all masked."""
    parts = []
    for i, n in enumerate(lens):
        m = (torch.rand(n, generator=gen) > 0.4).to(torch.uint8)
        if i % 3 == 1:
            m[0] = 0
        if i % 5 == 2:
            m[:] = 0
        parts.append(m)
    return torch.cat(parts).to(DEV)


def _ref(qkv, cu, key_mask, h):
    refs, slacks = [], []
    c = cu.tolist()
    for s, e in zip(c[:-1], c[1:]):
        m = None if key_mask is None else key_mask[s:e].view(1, e - s)
        r, sl = attention_ref(qkv[s:e], m, 1, e - s, h)
        refs.append(r)
        slacks.append(sl)
    return torch.cat(refs), torch.cat(slacks)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("lengths", ["one", "max", "edges", "seeded", "short"])
def test_attention_varlen_vs_float64(lengths, heads, masked):
    lens = _length_set(lengths)
    gen = torch.Generator().manual_seed(len(lens) * 100 + heads * 2 + masked)
    cu = _cu(lens)
    t = sum(lens)
    key_mask = _key_mask(lens, gen) if masked else None
    vals = (torch.randn(t, 3 * heads * 64, generator=gen) * 2).to(torch.bfloat16)
    qkv = guarded((t, 3 * heads * 64), pad_rows=3, values=vals.to(DEV))              # NaN rows around the operand
    out = guarded((t, heads * 64), pad_rows=3, fill=7.0,
                  values=torch.full((t, heads * 64), float("nan"), device=DEV, dtype=torch.bfloat16))
    assert ops.attention_varlen_supported(qkv.t, cu, max(lens), heads)
    ops.attention_varlen(qkv.t, cu, max(lens), heads, key_mask, out=out.t)
    torch.cuda.synchronize()
    out.assert_untouched("attention_varlen output")
    assert not out.t.isnan().any(), "an output row kept its pre-fill"
    ref, slack = _ref(qkv.t, cu, key_mask, heads)
    check_bf16(out.t, ref, slack, tau=1.0, criteria=(1,), what="attention_varlen %s H %d masked %s" % (
        lengths, heads, masked))
    if key_mask is not None:
        seq = torch.repeat_interleave(torch.arange(len(lens), device=DEV), torch.tensor(lens, device=DEV))
        dead = torch.zeros(len(lens), dtype=torch.int64, device=DEV).index_add_(0, seq, key_mask.long()) == 0
        rows = dead[seq]
        assert bool(dead.any()) == (len(lens) > 2)
        assert torch.equal(out.t[rows], torch.zeros_like(out.t[rows]))


@pytest.mark.parametrize("masked", [False, True])
def test_attention_varlen_isolation(masked):
    lens = [37, 200, 1, 129, 64, 300, 2]
    heads = 2
    gen = torch.Generator().manual_seed(11 + masked)
    cu = _cu(lens)
    t = sum(lens)
    key_mask = _key_mask(lens, gen) if masked else None
    qkv = (torch.randn(t, 3 * heads * 64, generator=gen) * 2).to(torch.bfloat16).to(DEV)
    base = ops.attention_varlen(qkv, cu, max(lens), heads, key_mask)
    c = cu.tolist()
    sign = torch.where(torch.rand(t, 3 * heads * 64, generator=gen) > 0.5, 1.0, -1.0).to(DEV)
    fills = {"nan": torch.full_like(sign, float("nan")), "inf": sign * float("inf"), "large": sign * 3e38}
    for b in range(len(lens)):
        other = torch.ones(t, dtype=torch.bool, device=DEV)
        other[c[b]:c[b + 1]] = False
        for name, fill in fills.items():
            x = qkv.clone()
            x[other] = fill[other].to(torch.bfloat16)
            out = torch.full((t, heads * 64), 5.0, device=DEV, dtype=torch.bfloat16)
            ops.attention_varlen(x, cu, max(lens), heads, key_mask, out=out)
            got, want = out[c[b]:c[b + 1]], base[c[b]:c[b + 1]]
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), (b, name)


@pytest.mark.parametrize("dist", ["1-256", "L/4-L"])
def test_ernie_base_forward_packed(dist):
    torch.manual_seed(0)
    model = ernie.ernie_base().to(DEV).eval()
    with torch.no_grad():
        model.cls_w.mul_(20)                  # decisive logits for the top-1 comparison
    b, l = 16, (256 if dist == "1-256" else 128)
    ids, pos, seg, mask = _inputs(b, l, l)
    if dist == "1-256":
        gen = torch.Generator().manual_seed(7)
        lens = torch.randint(1, l + 1, (b,), generator=gen)
        mask = (torch.arange(l)[None] < lens[:, None]).float().to(DEV)
    packed = ernie.pack_sequences(ids.cpu(), pos.cpu(), seg.cpu(), mask.cpu())
    assert packed[5] is None
    packed = [p.to(DEV) if torch.is_tensor(p) else p for p in packed]
    ops.reset_fallbacks()
    got = model.forward_packed(*packed)
    padded = model(ids, pos, seg, mask)
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    want = _torch_forward32(model, ids, pos, seg, mask)
    for other in (want, padded):
        cos = F.cosine_similarity(got.flatten()[None].double(), other.flatten()[None].double()).item()
        agree = (got.argmax(1) == other.argmax(1)).float().mean().item()
        assert cos > 0.999 and agree >= 15 / 16, (cos, agree)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model.forward_packed(*packed)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = model.forward_packed(*packed)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, got)
    assert ops.fallbacks() == {}, ops.fallbacks()


def test_teacher_server_mixed_lengths_on_cuda():
    from edl_b200.distill.teacher_server import TeacherServer

    torch.manual_seed(0)
    model, feeds, fetches, shapes = teacher_zoo.build("ernie_tiny")
    gen = torch.Generator().manual_seed(3)
    reqs = []
    for l, n in ((16, 3), (40, 2)):
        mask = np.zeros((n, l, 1), np.float32)
        for i in range(n):
            mask[i, :1 + (7 * i + l) % l] = 1
        mask[-1, 0] = 0                                           # a masked [CLS] token
        reqs.append([torch.randint(0, 1000, (n, l, 1), generator=gen).numpy(),
                     np.broadcast_to(np.arange(l, dtype=np.int64)[None, :, None], (n, l, 1)).copy(),
                     np.zeros((n, l, 1), np.int64), mask])
    srv = TeacherServer(model, feeds, fetches, shapes, device="cuda:0", dtype=torch.bfloat16)
    slots = [{"feeds": dict(zip(feeds, r)), "done": threading.Event(), "out": None, "err": None} for r in reqs]
    ops.reset_fallbacks()
    srv._run_batch(slots)
    assert ops.fallbacks() == {}, ops.fallbacks()
    for s, r in zip(slots, reqs):
        got = s["out"]["logits"]
        assert s["done"].is_set() and got.shape == (len(r[0]), 2) and got.dtype == np.float32
        feed = [torch.from_numpy(a).to(DEV) for a in r]
        want = srv.model(*feed).cpu().numpy()
        assert np.allclose(got, want, atol=1e-2, rtol=2e-2), (got, want)
