"""The ERNIE teacher's inference forward on the GPU kernels, judged call by call by tests/ernie_oracle.py: ernie_base and
MiniLM-L12-H384 in bf16 and block-scaled FP8, padded, packed (with ``key_mask``) and request-batched, a CUDA-graph
replay, weights that follow ``load_state_dict`` and in-place updates, and negative controls that must fail at their
site.  Every model gets random biases and LayerNorm parameters first, so a wrong bias, gamma or beta cannot hide."""
import functools

import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import ernie_oracle as eo  # noqa: E402
import f64_bounds as fb  # noqa: E402
from edl_b200 import ops  # noqa: E402
from edl_b200.models import ernie  # noqa: E402
from edl_b200.ops import fp8  # noqa: E402
from test_ernie_oracle_cpu import _changed, batch, packed, shift_cls_rows  # noqa: E402

DEV = torch.device("cuda", 0)
BUILD = {"ernie_base": (ernie.ernie_base, 18000), "minilm_l12_h384": (ernie.minilm_l12_h384, 30522),
         "ernie_tiny": (ernie.ernie_tiny, 1000)}


def model_of(name, fp8_mode, seed=0):
    torch.manual_seed(seed)
    m = BUILD[name][0]().to(DEV).eval()
    eo.random_vectors(m, seed + 100)
    if fp8_mode:
        m.enable_fp8()
    return m


def judge(m, args, layout, what):
    """One recorded forward of ``m`` on ``args`` (padded feeds or ``pack_sequences`` output), judged by the oracle."""
    ops.reset_fallbacks()
    with eo.ErnieRecorder(m) as rec:
        logits = m.forward_packed(*args) if layout == "packed" else m(*args)
    torch.cuda.synchronize()
    worst = rec.check(logits, log=lambda s: print(what + ": " + s))
    return rec, logits, worst


@pytest.mark.parametrize("mode", ["bf16", "fp8"])
def test_ernie_base_padded_and_packed(mode):
    """B = 16, L = 128, right-padded lengths with a length-1 sample, padded and packed; then the same batch with
    sample 1's token 0 masked (the packed layout's key_mask) and sample 3 empty, packed."""
    m = model_of("ernie_base", mode == "fp8")
    feeds = batch(16, 128, 1, 18000, DEV, masked_cls=False)
    _, lp, _ = judge(m, feeds, "padded", "ernie_base %s padded" % mode)
    pk = packed(m, feeds)
    assert pk[5] is None
    _, lk, _ = judge(m, pk, "packed", "ernie_base %s packed" % mode)
    if mode == "fp8":
        assert torch.equal(lp, lk)               # right-padded: every step is row-wise or per sequence
    feeds = batch(16, 128, 2, 18000, DEV)
    pk = packed(m, feeds)
    assert pk[5] is not None
    judge(m, pk, "packed", "ernie_base %s packed, key_mask" % mode)


def test_ernie_base_fp8_long_sequences():
    m = model_of("ernie_base", True)
    feeds = batch(2, 512, 3, 18000, DEV, masked_cls=False, lens=[512, 301])
    judge(m, feeds, "padded", "ernie_base fp8 L 512 padded")
    judge(m, packed(m, feeds), "packed", "ernie_base fp8 L 512 packed")


@pytest.mark.parametrize("mode", ["bf16", "fp8"])
def test_minilm_packed_key_mask(mode):
    """Head dim 32, three k-blocks (hidden 384), FFN 1536."""
    m = model_of("minilm_l12_h384", mode == "fp8")
    assert m.head_dim == 32
    pk = packed(m, batch(16, 128, 4, 30522, DEV))
    assert pk[5] is not None
    judge(m, pk, "packed", "minilm %s packed, key_mask" % mode)


def test_ernie_tiny_fp8_odd_rows():
    m = model_of("ernie_tiny", True)
    pk = packed(m, batch(3, 45, 5, 1000, DEV, masked_cls=False, lens=[45, 31, 1]))
    assert pk[0].numel() == 77
    judge(m, pk, "packed", "ernie_tiny fp8 T 77")


def test_forward_requests_fp8():
    """Three requests of different L, packed on the host and judged call by call; the logits come back in request
    order: each request's rows are its own padded forward's bits."""
    m = model_of("ernie_base", True)
    reqs = [[t.cpu() for t in batch(n, l, 10 + l, 18000, masked_cls=False)] for n, l in ((3, 32), (2, 77), (4, 128))]
    ops.reset_fallbacks()
    with eo.ErnieRecorder(m) as rec:
        logits = m.forward_requests(reqs)
    torch.cuda.synchronize()
    rec.check(logits, log=lambda s: print("forward_requests: " + s))
    assert logits.shape == (9, 2)
    row = 0
    for r in reqs:
        n = r[0].shape[0]
        assert torch.equal(logits[row:row + n], m(*[t.to(DEV) for t in r])), row
        row += n


def test_graph_replay_fp8_packed():
    """The recorder's clones are captured with the forward, so they hold the replay's values: the ids in the static
    buffer are changed before the replay, and the oracle judges that replay."""
    m = model_of("ernie_base", True)
    pk = packed(m, batch(16, 128, 6, 18000, DEV))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m.forward_packed(*pk)                    # builds the weights and warms up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    ops.reset_fallbacks()
    g = torch.cuda.CUDAGraph()
    with eo.ErnieRecorder(m) as rec:
        with torch.cuda.graph(g):
            static = m.forward_packed(*pk)
    new_ids = torch.randint(0, 18000, pk[0].shape, generator=torch.Generator().manual_seed(7)).to(DEV)
    pk[0].copy_(new_ids)
    g.replay()
    torch.cuda.synchronize()
    emb = dict(rec.sites())["embeddings"]
    assert torch.equal(emb.a["ids"], new_ids)                # the judged values are the replay's
    rec.check(static, log=lambda s: print("graph replay: " + s))
    assert torch.equal(static, m.forward_packed(*pk))


@pytest.mark.parametrize("mode", ["bf16", "fp8"])
@pytest.mark.parametrize("update", ["load_state_dict", "in-place"])
def test_forward_serves_updated_weights(mode, update):
    """forward, then ``load_state_dict(other)`` or an in-place update under ``no_grad``, then forward again: bit for bit
    the forward of a model built with those parameters."""
    q = mode == "fp8"
    m = model_of("ernie_base", q, seed=0)
    feeds = batch(16, 128, 8, 18000, DEV, masked_cls=False)
    first = m(*feeds)
    if update == "load_state_dict":
        want = model_of("ernie_base", q, seed=1)
        m.load_state_dict(want.state_dict())
    else:
        _changed(m)
        want = model_of("ernie_base", q, seed=0)
        _changed(want)
    got = m(*feeds)
    assert not torch.equal(got, first)
    assert torch.equal(got, want(*feeds))
    judge(m, feeds, "padded", "ernie_base %s after %s" % (mode, update))


# ------------------------------------------------------------------------------------------------ negative controls
def test_negative_controls():
    """ernie_tiny in FP8 on the kernels: one ulp on a LayerNorm output, a doubled k-block activation scale given to a
    real FFN2 kernel call, the pooler reading row 1 instead of [CLS], and a stale weight each fail at their site."""
    feeds = batch(6, 40, 9, 1000, DEV)
    m = model_of("ernie_tiny", True)
    rec, logits, _ = judge(m, feeds, "padded", "control baseline")
    s = dict(rec.sites())["layers.1.ln1"]
    y = s.out[0]
    ref, _ = eo.so.ln_ref(s.a["x"].double(), s.a["gamma"], s.a["beta"], m.eps)
    rel = (y.double() - ref).abs() / fb.ulp(ref.abs(), 8).clamp_min(1e-300)
    y.view(torch.int16).view(-1)[int(rel.reshape(-1).argmin())] += 1
    with pytest.raises(AssertionError, match=r"layers\.1\.ln1 \(fp8\)"):
        rec.check(logits)

    orig = fp8.gemm_fp8_blockscaled
    n = [0]

    @functools.wraps(orig)
    def corrupt(a8, sa, *args, **kw):
        n[0] += 1
        if n[0] == 6:                                        # layers.1.ffn2: K = 512, four k-blocks
            sa = sa.clone()
            sa[2, 5] *= 2
        return orig(a8, sa, *args, **kw)

    fp8.gemm_fp8_blockscaled = corrupt
    try:
        ops.reset_fallbacks()
        with eo.ErnieRecorder(m) as rec:
            logits = m(*feeds)
    finally:
        fp8.gemm_fp8_blockscaled = orig
    with pytest.raises(AssertionError, match=r"layers\.1\.ffn2 \(fp8\)"):
        rec.check(logits)

    shift_cls_rows(m)
    try:
        ops.reset_fallbacks()
        with eo.ErnieRecorder(m) as rec:
            logits = m(*feeds)
    finally:
        del m._forward_fp8
    with pytest.raises(AssertionError, match=r"pooler \(fp8\) .*\[CLS\]"):
        rec.check(logits)

    _changed(m)
    m._dev_key = m._weights_key()                            # leave the cache stale on purpose
    ops.reset_fallbacks()
    with eo.ErnieRecorder(m) as rec:
        logits = m(*feeds)
    with pytest.raises(AssertionError, match=r"layers\.1\.out \(fp8\) .*weight"):
        rec.check(logits)
