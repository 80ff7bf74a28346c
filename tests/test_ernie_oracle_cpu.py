"""tests/ernie_oracle.py on the CPU: the FP8 emulation of the ERNIE teacher makes the same calls as the CUDA path, so
the oracle must accept it, padded and packed, at head dims 64 and 32; small corruptions (one ulp, a doubled k-block
scale, the pooler reading the wrong row, a stale weight) must fail and name their site.  And a forward after
``load_state_dict`` or an in-place parameter update serves the new weights."""
import copy
import functools

import pytest
import torch

import ernie_oracle as eo
import f64_bounds as fb
from edl_b200.models import ernie
from edl_b200.ops import fp8


def tiny_h32():
    """2 layers, hidden 128, 4 heads of 32, FFN 512."""
    return ernie.ErnieEncoder(1000, 128, 2, 4, 512, 513, 2, 2)


MODELS = {"ernie_tiny": ernie.ernie_tiny, "h128_heads4": tiny_h32}


def batch(b, l, seed, vocab, device="cpu", masked_cls=True, lens=None):
    """Right-padded samples of mixed lengths (or ``lens``): sample 0 full, sample 2 of length 1; with ``masked_cls``
    sample 1 has its token 0 masked (so the packed layout's ``key_mask`` is live) and, for b >= 4, sample 3 has no
    valid token at all."""
    gen = torch.Generator().manual_seed(seed)
    if lens is None:
        lens = torch.randint(1, l + 1, (b,), generator=gen)
        lens[0] = l
        if b > 2:
            lens[2] = 1
    else:
        lens = torch.tensor(lens)
    mask = (torch.arange(l)[None] < lens[:, None]).float()
    if masked_cls:
        mask[1, 0] = 0
        if b >= 4:
            mask[3] = 0
    ids = torch.randint(0, vocab, (b, l), generator=gen)
    seg = torch.randint(0, 2, (b, l), generator=gen)
    pos = torch.arange(l).expand(b, l).contiguous()
    return [t.to(device) for t in (ids, pos, seg, mask)]


def packed(model, feeds):
    pk = ernie.pack_sequences(*[t.cpu() for t in feeds], max_positions=model.pos_emb.shape[0])
    dev = model.word_emb.device
    return [t.to(dev) if torch.is_tensor(t) else t for t in pk]


def run(model, feeds, layout):
    """One recorded forward: (recorder, logits)."""
    args = packed(model, feeds) if layout == "packed" else feeds
    with eo.ErnieRecorder(model) as rec:
        logits = model.forward_packed(*args) if layout == "packed" else model(*args)
    return rec, logits


def fp8_model(name="ernie_tiny", seed=0):
    torch.manual_seed(seed)
    m = MODELS[name]()
    eo.random_vectors(m, seed + 100)
    m.enable_fp8()
    return m


@pytest.mark.parametrize("layout", ["padded", "packed"])
@pytest.mark.parametrize("name", sorted(MODELS))
def test_oracle_accepts_fp8_emulation(name, layout):
    m = fp8_model(name)
    feeds = batch(6, 40, 1, 1000)
    if layout == "packed":
        assert packed(m, feeds)[5] is not None                     # key_mask is live
    rec, logits = run(m, feeds, layout)
    assert logits.shape == (6, 2)
    worst = rec.check(logits)
    assert set(worst) >= {"FP8 GEMM (QKV, out, FFN2)", "FP8 FFN1 -> e4m3", "attention", "LayerNorm, embedding-LayerNorm",
                          "CPU head (fp32)"}, worst
    # padded and packed give the same logits on right-padded masks, so both runs judge the same forward
    other = run(m, feeds, "padded" if layout == "packed" else "packed")[1]
    assert torch.equal(logits, other)


def _site(rec, site):
    return dict(rec.sites())[site]


def test_one_ulp_fails_at_its_site():
    m = fp8_model()
    rec, logits = run(m, batch(6, 40, 2, 1000), "padded")
    rec.check(logits)
    s = _site(rec, "layers.1.ln1")
    y = s.out[0]
    ref, _ = eo.so.ln_ref(s.a["x"].double(), s.a["gamma"], s.a["beta"], m.eps)
    # the element whose rounding error is smallest relative to its ulp: one ulp there cannot hide in the bound
    rel = (y.double() - ref).abs() / fb.ulp(ref.abs(), 8).clamp_min(1e-300)
    i = int(rel.reshape(-1).argmin())
    y.view(torch.int16).view(-1)[i] += 1
    with pytest.raises(AssertionError, match=r"layers\.1\.ln1 \(fp8\)"):
        rec.check(logits)


def test_doubled_block_scale_fails_at_its_site(monkeypatch):
    """FFN2 of layer 1 (the sixth block-scaled GEMM) computes with k-block 2 of row 5's activation scale doubled; the
    recorder sees the scales the model passed."""
    orig = fp8.gemm_fp8_blockscaled
    n = [0]

    @functools.wraps(orig)                  # the recorder binds the arguments by the real signature
    def corrupt(a8, sa, *args, **kw):
        n[0] += 1
        if n[0] == 6:
            sa = sa.clone()
            sa[2, 5] *= 2
        return orig(a8, sa, *args, **kw)

    m = fp8_model()
    feeds = batch(6, 40, 3, 1000)
    monkeypatch.setattr(fp8, "gemm_fp8_blockscaled", corrupt)
    rec, logits = run(m, feeds, "padded")
    with pytest.raises(AssertionError, match=r"layers\.1\.ffn2 \(fp8\)"):
        rec.check(logits)


def shift_cls_rows(model):
    """Make the pooler read row 1 of each sample instead of its [CLS] row (undone by ``del model._forward_fp8``)."""
    orig = model._forward_fp8

    def fwd(ids, pos, seg, attend, cls_rows):
        return orig(ids, pos, seg, attend, lambda x: cls_rows(torch.roll(x, -1, 0)))

    model._forward_fp8 = fwd


@pytest.mark.parametrize("layout", ["padded", "packed"])
def test_pooler_reading_row_1_fails(layout):
    m = fp8_model()
    feeds = batch(6, 40, 4, 1000)
    shift_cls_rows(m)
    rec, logits = run(m, feeds, layout)
    with pytest.raises(AssertionError, match=r"pooler \(fp8\)"):
        rec.check(logits)


def _changed(m):
    """An in-place update of layer 1: its out-projection weight and bias and its second LayerNorm's gamma.  (The fp32
    vectors the forward reads are the parameters themselves; the weight matrices are converted copies.)"""
    with torch.no_grad():
        m.layers[1].out_w.mul_(1.25)
        m.layers[1].out_b.mul_(1.5)
        m.layers[1].ln2_g.mul_(0.75)


def test_stale_weights_are_named():
    """A cache left stale on purpose (its key set to the current parameters' without a rebuild) names the first layer
    whose parameters changed."""
    m = fp8_model()
    feeds = batch(6, 40, 5, 1000)
    m(*feeds)
    _changed(m)
    m._dev_key = m._weights_key()
    rec, logits = run(m, feeds, "padded")
    with pytest.raises(AssertionError, match=r"layers\.1\.out \(fp8\) .*weight"):
        rec.check(logits)


@pytest.mark.parametrize("update", ["load_state_dict", "in-place"])
def test_forward_serves_updated_weights(update):
    """After a forward has built the cached weights, ``load_state_dict`` or in-place ``mul_`` under ``no_grad`` are
    served by the next forward: bit for bit the forward of a freshly built model with those parameters."""
    a, b = fp8_model(seed=0), fp8_model(seed=1)
    m = copy.deepcopy(a)
    assert len(m._weights_key()) == 2 + len(list(m.parameters()))          # the key covers every parameter
    feeds = batch(6, 40, 6, 1000)
    first = m(*feeds)
    assert torch.equal(first, a(*feeds))
    if update == "load_state_dict":
        m.load_state_dict(b.state_dict())
        want = b
    else:
        _changed(m)
        want = fp8_model(seed=0)
        _changed(want)
    got = m(*feeds)
    assert not torch.equal(got, first)
    assert torch.equal(got, want(*feeds))
    rec, logits = run(m, feeds, "packed")
    rec.check(logits)
