"""Block-scaled FP8 mode of the ERNIE teacher on CPU: enable_fp8, the float32 emulation of the quantised pipeline, the
CPU paths of the fused ops (each the composition of the existing references), re-quantisation after a load, and the
server's choice of FP8 scaling per model."""
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models import ernie, teacher_zoo
from edl_b200.ops import fp8


def _feeds(b, l, seed, vocab=1000):
    gen = torch.Generator().manual_seed(seed)
    lens = torch.randint(l // 4, l + 1, (b,), generator=gen)
    mask = (torch.arange(l)[None] < lens[:, None]).float()
    ids = torch.randint(0, vocab, (b, l), generator=gen)
    seg = torch.randint(0, 2, (b, l), generator=gen)
    pos = torch.arange(l).expand(b, l).contiguous()
    return ids, pos, seg, mask


def test_enable_fp8_counts_and_rejects_tensor_scaling():
    assert ernie.ernie_base().enable_fp8() == 48
    assert ernie.ernie_tiny().enable_fp8(scaling="block") == 8
    assert ernie.ErnieEncoder(vocab=50, hidden=64, layers=3, heads=1, ffn=128).enable_fp8() == 12
    m = ernie.ernie_tiny()
    for bad in ("tensor", "row", None):
        with pytest.raises(ValueError, match="block"):
            m.enable_fp8(scaling=bad)
    assert not m._fp8


def test_fp8_weights_replace_the_bf16_matrices():
    m = ernie.ernie_tiny()
    m.enable_fp8()
    lyr = m._device_weights()["layers"][0]
    for i, name in ((0, "qkv_w"), (2, "out_w"), (6, "ffn1_w"), (8, "ffn2_w")):
        q, s = lyr[i]
        want_q, want_s = fp8.quantize_weight_blocks(getattr(m.layers[0], name))
        assert q.dtype == torch.uint8 and torch.equal(q, want_q) and torch.equal(s, want_s)
    assert m._device_weights()["emb"][0].dtype == torch.bfloat16              # embeddings and head stay bf16
    assert m._device_weights()["head"][0].dtype == torch.bfloat16


@pytest.mark.parametrize("packed", [False, True])
def test_emulated_fp8_forward_tracks_float32(packed):
    torch.manual_seed(0)
    ref = ernie.ernie_tiny()
    with torch.no_grad():
        ref.cls_w.mul_(20)                     # decisive logits for the top-1 comparison
    model = ernie.ernie_tiny()
    model.load_state_dict(ref.state_dict())
    assert model.enable_fp8() == 8
    feeds = _feeds(16, 48, 1)
    want = ref(*feeds)
    got = model.forward_packed(*ernie.pack_sequences(*feeds)) if packed else model(*feeds)
    assert got.dtype == torch.float32 and got.shape == want.shape
    cos = F.cosine_similarity(got.flatten()[None].double(), want.flatten()[None].double()).item()
    agree = (got.argmax(1) == want.argmax(1)).float().mean().item()
    assert cos > 0.998 and agree >= 15 / 16, (cos, agree)
    assert not torch.equal(got, want)          # it is the quantised pipeline, not the float32 one


def test_emulated_fp8_packed_equals_padded():
    torch.manual_seed(0)
    model = ernie.ernie_tiny()
    model.enable_fp8()
    feeds = _feeds(4, 24, 2)
    got = model.forward_packed(*ernie.pack_sequences(*feeds))
    for b in range(4):
        assert torch.allclose(got[b:b + 1], model(*(t[b:b + 1] for t in feeds)), atol=1e-5)


def test_load_after_enable_fp8_requantises():
    torch.manual_seed(0)
    model = ernie.ernie_tiny()
    model.enable_fp8()
    feeds = _feeds(4, 16, 3)
    before = model(*feeds)
    other = ernie.ernie_tiny()
    sd = {}
    for i, lyr in enumerate(other.layers):
        p = "encoder.layer.%d." % i
        q, k, v = lyr.qkv_w.chunk(3, 0)
        qb, kb, vb = lyr.qkv_b.chunk(3, 0)
        for n, w, b in (("query", q, qb), ("key", k, kb), ("value", v, vb)):
            sd[p + "attention.self.%s.weight" % n], sd[p + "attention.self.%s.bias" % n] = w, b
        sd[p + "attention.output.dense.weight"], sd[p + "attention.output.dense.bias"] = lyr.out_w, lyr.out_b
        sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"] = lyr.ln1_g, lyr.ln1_b
        sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"] = lyr.ffn1_w, lyr.ffn1_b
        sd[p + "output.dense.weight"], sd[p + "output.dense.bias"] = lyr.ffn2_w, lyr.ffn2_b
        sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"] = lyr.ln2_g, lyr.ln2_b
    e = "embeddings."
    sd[e + "word_embeddings.weight"], sd[e + "position_embeddings.weight"] = model.word_emb, model.pos_emb
    sd[e + "token_type_embeddings.weight"] = model.seg_emb
    sd[e + "LayerNorm.weight"], sd[e + "LayerNorm.bias"] = model.emb_ln_g, model.emb_ln_b
    sd["pooler.dense.weight"], sd["pooler.dense.bias"] = model.pool_w, model.pool_b
    model.load_bert_state_dict({k: v.clone() for k, v in sd.items()})
    assert model._fp8
    after = model(*feeds)
    assert not torch.allclose(before, after)
    q, s = model._device_weights()["layers"][1][6]
    assert torch.equal(q, fp8.quantize_weight_blocks(other.layers[1].ffn1_w)[0])


@pytest.mark.parametrize("c", [128, 320, 768])
def test_layer_norm_e4m3_cpu_is_the_composition(c):
    gen = torch.Generator().manual_seed(c)
    x = (torch.randn(7, c, generator=gen) * 3).to(torch.bfloat16)
    x[2] = 0                                                  # an all-zero row: s = 1
    g, b = torch.randn(c, generator=gen), torch.randn(c, generator=gen)
    b[:] = torch.where(torch.arange(c) % 2 == 0, b, torch.zeros(c))
    y, q, sa = ops.layer_norm_e4m3(x, g, b, 1e-12)
    want = ops.layer_norm(x, g, b, 1e-12)
    assert y.dtype == torch.bfloat16 and torch.equal(y, want)
    wq, ws = fp8.quantize_e4m3_blocks(want)
    assert torch.equal(q, wq) and torch.equal(sa, ws) and sa.shape == (-(-c // 128), 7)
    ids = torch.randint(0, 40, (5,), generator=gen)
    tabs = [(torch.randn(n, c, generator=gen)).to(torch.bfloat16) for n in (40, 9, 2)]
    pos, seg = torch.randint(0, 9, (5,), generator=gen), torch.randint(0, 2, (5,), generator=gen)
    y, q, sa = ops.embedding_layernorm_e4m3(ids, pos, seg, *tabs, g, b, 1e-12)
    want = ops.embedding_layernorm(ids, pos, seg, *tabs, g, b, 1e-12)
    assert torch.equal(y, want)
    wq, ws = fp8.quantize_e4m3_blocks(want)
    assert torch.equal(q, wq) and torch.equal(sa, ws)


def test_fused_gemm_cpu_paths_are_the_composition():
    gen = torch.Generator().manual_seed(5)
    m, n, k = 9, 320, 256
    a = torch.randn(m, k, generator=gen).to(torch.bfloat16)
    w = torch.randn(n, k, generator=gen) * 0.05
    bias = torch.randn(n, generator=gen)
    add = torch.randn(m, n, generator=gen).to(torch.bfloat16)
    qa, sa = fp8.quantize_e4m3_blocks(a)
    qw, sw = fp8.quantize_weight_blocks(w)
    plain = fp8.gemm_fp8_blockscaled(qa, sa, qw, sw, col_shift=bias)
    d = fp8._blockscaled_product(qa, sa, qw, sw)
    assert torch.equal(plain, (d + bias).to(torch.bfloat16))
    got = fp8.gemm_fp8_blockscaled(qa, sa, qw, sw, col_shift=bias, add=add)
    assert torch.equal(got, (d + bias + add.float()).to(torch.bfloat16))
    q, s = fp8.gemm_fp8_gelu_e4m3(qa, sa, qw, sw, bias=bias)
    wq, ws = fp8.quantize_e4m3_blocks(F.gelu(d + bias).to(torch.bfloat16))
    assert torch.equal(q, wq) and torch.equal(s, ws) and s.shape == (3, m)


def test_server_fp8_scaling_per_model():
    from edl_b200.distill.teacher_server import fp8_scaling, main

    seq = teacher_zoo.build("ernie_tiny")[0]
    net = getattr(seq, "net", seq)
    assert fp8_scaling(net) == "block" and fp8_scaling(net, "block") == "block"
    with pytest.raises(ValueError, match="block"):
        fp8_scaling(net, "tensor")

    class ImageNet(torch.nn.Module):             # an image teacher: enable_fp8 but no forward_requests
        def enable_fp8(self, calib):
            return 0

    img = ImageNet()
    assert fp8_scaling(img) == "tensor" and fp8_scaling(img, "block") == "block"
    assert fp8_scaling(img, "tensor") == "tensor"
    with pytest.raises(SystemExit) as e:
        main(["--model", "ernie_tiny", "--fp8", "--fp8_scaling", "tensor"])
    assert e.value.code == 2
