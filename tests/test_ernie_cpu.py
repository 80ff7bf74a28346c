"""The ERNIE sequence teacher on CPU: the BERT-layout loader and the float32 reference forward against ``transformers``,
the CPU reference ops (attention, LayerNorm, embedding + LayerNorm) against float64, and the serving contract with the
reference's four ERNIE feeds."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models import ernie, teacher_zoo


def _masks(b, l, gen):
    """Right-padded rows, rows with holes (the [CLS] position always kept) and one full row."""
    m = torch.zeros(b, l)
    for i in range(b):
        n = int(torch.randint(1, l + 1, (1,), generator=gen))
        m[i, :n] = 1
        if i % 2 == 1:
            m[i] = (torch.rand(l, generator=gen) > 0.4).float()
            m[i, 0] = 1
    m[0] = 1
    return m


def _bert(cfg_kw, num_labels, seed=0):
    transformers = pytest.importorskip("transformers")
    torch.manual_seed(seed)
    cfg = transformers.BertConfig(attn_implementation="eager", hidden_dropout_prob=0.0,
                                  attention_probs_dropout_prob=0.0, **cfg_kw)
    bert = transformers.BertModel(cfg).eval()
    cls = torch.nn.Linear(cfg.hidden_size, num_labels)
    sd = {"bert." + k: v for k, v in bert.state_dict().items()}
    sd.update({"classifier.weight": cls.weight.detach(), "classifier.bias": cls.bias.detach()})
    return bert, cls, sd


@pytest.mark.parametrize("prefix", [True, False])
def test_loader_and_reference_forward_match_transformers(prefix):
    kw = dict(vocab_size=300, hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
              max_position_embeddings=64, type_vocab_size=2, hidden_act="gelu", layer_norm_eps=1e-12)
    bert, cls, sd = _bert(kw, 3)
    if not prefix:
        sd = {k[len("bert."):] if k.startswith("bert.") else k: v for k, v in sd.items()}
    model = ernie.ErnieEncoder(300, 128, 2, 2, 256, 64, 2, 3)
    unused = model.load_bert_state_dict(sd)
    assert all("position_ids" in k or "token_type_ids" in k for k in unused), unused
    gen = torch.Generator().manual_seed(1)
    b, l = 5, 23
    ids = torch.randint(0, 300, (b, l), generator=gen)
    seg = torch.randint(0, 2, (b, l), generator=gen)
    pos = torch.arange(l).expand(b, l)
    mask = _masks(b, l, gen)
    got = model(ids, pos, seg, mask)
    with torch.no_grad():
        out = bert(input_ids=ids, token_type_ids=seg, position_ids=pos, attention_mask=mask.long())
        want = cls(out.pooler_output)
    assert got.dtype == torch.float32 and got.shape == (b, 3)
    assert torch.allclose(got, want, atol=2e-5, rtol=1e-5), (got - want).abs().max()


def test_loader_formats(tmp_path):
    _, _, sd = _bert(dict(vocab_size=50, hidden_size=32, num_hidden_layers=1, num_attention_heads=2,
                          intermediate_size=64, max_position_embeddings=16, type_vocab_size=2), 2)
    sd = {k: v.contiguous() for k, v in sd.items()}
    from safetensors.torch import save_file

    save_file(sd, str(tmp_path / "w.safetensors"))
    torch.save(sd, str(tmp_path / "w.pt"))
    a, b = ernie.ErnieEncoder(50, 32, 1, 2, 64, 16, 2, 2), ernie.ErnieEncoder(50, 32, 1, 2, 64, 16, 2, 2)
    a.load_weights(tmp_path / "w.safetensors")
    b.load_weights(tmp_path / "w.pt")
    for (n, p), (_, q) in zip(a.named_parameters(), b.named_parameters()):
        assert torch.equal(p, q), n
    assert torch.equal(a.cls_w, sd["classifier.weight"])
    with pytest.raises(ValueError):
        ernie.ErnieEncoder(50, 32, 1, 2, 128, 16, 2, 2).load_bert_state_dict(sd)       # FFN width differs
    with pytest.raises(KeyError):
        a.load_bert_state_dict({k: v for k, v in sd.items() if "pooler" not in k})


# ------------------------------------------------------------------------------------ reference ops vs float64
def _attention64(qkv, mask, b, l, h, d=64):
    x = qkv.double().view(b, l, 3, h, d)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))
    s = q @ k.transpose(-1, -2) / d ** 0.5
    keep = mask.view(b, 1, 1, l) != 0
    s = s.masked_fill(~keep, float("-inf"))
    p = torch.softmax(s, -1).nan_to_num(0.0)          # a row without a valid key: 0
    return (p @ v).transpose(1, 2).reshape(b * l, h * d)


def test_attention_reference_vs_float64():
    gen = torch.Generator().manual_seed(2)
    b, l, h = 4, 37, 3
    qkv = torch.randn(b * l, 3 * h * 64, generator=gen) * 2
    mask = _masks(b, l, gen)
    mask[2] = 0
    mask[2, 5] = 1                                     # one valid key
    mask[3] = 0                                        # no valid key
    got = ops.attention(qkv, mask, b, l, h)
    want = _attention64(qkv, mask, b, l, h)
    assert torch.allclose(got.double(), want, atol=1e-5, rtol=1e-5)
    rows = torch.arange(b * l) // l
    v = qkv.view(b, l, 3, h, 64)[2, 5, 2].reshape(-1)
    assert torch.allclose(got[rows == 2], v.expand(l, -1), atol=1e-6)
    assert torch.equal(got[rows == 3], torch.zeros(l, h * 64))


def test_layer_norm_references_vs_float64():
    gen = torch.Generator().manual_seed(3)
    for c in (768, 40):
        x = torch.randn(37, c, generator=gen) * 3 + 1
        g, bt = torch.randn(c, generator=gen), torch.randn(c, generator=gen)
        want = F.layer_norm(x.double(), (c,), g.double(), bt.double(), 1e-12)
        assert torch.allclose(ops.layer_norm(x, g, bt, 1e-12).double(), want, atol=1e-5)
        word, pos, seg = (torch.randn(n, c, generator=gen) for n in (50, 20, 2))
        ids, pids, sids = (torch.randint(0, n, (3, 11), generator=gen) for n in (50, 20, 2))
        x64 = word.double()[ids.reshape(-1)] + pos.double()[pids.reshape(-1)] + seg.double()[sids.reshape(-1)]
        want = F.layer_norm(x64, (c,), g.double(), bt.double(), 1e-12)
        got = ops.embedding_layernorm(ids, pids, sids, word, pos, seg, g, bt, 1e-12)
        assert torch.allclose(got.double(), want, atol=1e-5)
        with pytest.raises(IndexError):
            ops.embedding_layernorm(ids + 50, pids, sids, word, pos, seg, g, bt, 1e-12)


def test_gelu_gemm_reference():
    gen = torch.Generator().manual_seed(4)
    a, w, bias = torch.randn(9, 40, generator=gen), torch.randn(24, 40, generator=gen), torch.randn(24, generator=gen)
    got = ops.gemm_bf16(a.bfloat16(), w.bfloat16(), col_shift=bias, gelu=True)
    v = a.bfloat16().double() @ w.bfloat16().double().t() + bias.double()
    want = 0.5 * v * (1 + torch.erf(v / 2 ** 0.5))
    assert got.dtype == torch.bfloat16
    assert torch.allclose(got.double(), want, rtol=2 ** -7, atol=1e-6)
    with pytest.raises(ValueError):
        ops.gemm_bf16(a.bfloat16(), w.bfloat16(), gelu=True, relu=True)
    wp = torch.nn.Parameter(w.bfloat16())
    with pytest.raises(RuntimeError):
        ops.linear_bf16(a.bfloat16(), wp, gelu=True)


# ------------------------------------------------------------------------------------------- serving contract
def test_teacher_server_serves_ernie_logits():
    from edl_b200.distill.distill_reader import DistillReader
    from edl_b200.distill.teacher_server import TeacherServer

    torch.manual_seed(0)
    model, feeds, fetches, shapes = teacher_zoo.build("ernie_tiny")
    assert feeds == ["input_ids", "position_ids", "segment_ids", "input_mask"] and fetches == ["logits"]
    l = 16
    gen = torch.Generator().manual_seed(5)

    def samples():
        for i in range(12):
            ids = torch.randint(0, 1000, (l, 1), generator=gen).numpy()
            n = 1 + i % l
            mask = np.zeros((l, 1), np.float32)
            mask[:n] = 1
            yield (ids, np.arange(l, dtype=np.int64)[:, None], (np.arange(l) >= l // 2).astype(np.int64)[:, None],
                   mask, np.array([i % 2], np.int64))

    data = list(samples())
    with TeacherServer(model, feeds, fetches, shapes, max_wait_ms=1.0) as srv:
        dr = DistillReader(ins=feeds + ["label"], predicts=["logits"])
        dr.set_teacher_batch_size(4)
        dr.set_fixed_teacher([srv.endpoint])
        r = dr.set_sample_list_generator(lambda: [data[i:i + 3] for i in range(0, len(data), 3)])
        n = 0
        for batch in r():
            for ids, pos, seg, mask, label, logits in batch:
                want = model(*(torch.from_numpy(t)[None] for t in (ids, pos, seg, mask)))[0].numpy()
                assert logits.shape == (2,) and logits.dtype == np.float32
                assert np.allclose(logits, want, atol=1e-5), (logits, want)
                n += 1
        dr.stop()
    assert n == 12
