"""Head dim 32 on the CPU: the student's float32 path at 32-wide heads, the ``heads`` option of ``ernie_student``, the
``minilm_l12_h384`` teacher and the examples' ``--heads``."""
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

from edl_b200.models import teacher_zoo
from edl_b200.models.ernie import ErnieEncoder, ErnieStudent, ernie_student, minilm_l12_h384
from test_ernie_student_cpu import _functional_encoder, _run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_hd32_student_gradients_match_functional_encoder():
    torch.manual_seed(0)
    m = ErnieStudent(vocab=60, hidden=128, layers=2, heads=4, ffn=256, max_pos=40, num_labels=3)
    assert m.head_dim == 32
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 1:
                p.add_(torch.randn_like(p) * 0.1)
    b, l = 3, 17
    ids = torch.randint(1, 60, (b, l))
    ids[0, 9:] = 0
    ids[2, 0] = 0                                                     # token 0 masked
    label = torch.tensor([0, 2, 1])
    F.cross_entropy(m(ids), label).backward()
    got = {n: p.grad.clone() for n, p in m.named_parameters()}
    logits = m(ids).detach()
    m.zero_grad()
    pos = torch.arange(l).expand(b, l)
    ref = _functional_encoder(m, ids, pos, torch.zeros_like(ids), ids != 0)
    assert torch.allclose(logits, ref.detach(), atol=1e-5, rtol=1e-5)
    F.cross_entropy(ref, label).backward()
    for n, p in m.named_parameters():
        assert torch.allclose(got[n], p.grad, atol=1e-6, rtol=1e-4), n


def test_ernie_student_heads():
    m = ernie_student(heads=12)
    assert (m.hidden, m.heads, m.head_dim, m.num_layers) == (384, 12, 32, 4)
    assert m.layers[0].ffn1_w.shape == (1536, 384) and m.word_emb.shape == (18000, 384)
    default, six = ernie_student(), ErnieStudent(18000, 384, 4, 6, 1536, 513, 2, 2)
    assert (default.heads, default.head_dim) == (6, 64)
    want = {k: tuple(v.shape) for k, v in six.state_dict().items()}
    assert {k: tuple(v.shape) for k, v in default.state_dict().items()} == want
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == want    # heads do not change the parameters


def _bert_state_dict(m, gen):
    """A synthetic BERT-layout state dict for ``m``'s shapes (``bert.`` prefix, LayerNorm gamma / beta names)."""
    c, f = m.hidden, m.layers[0].ffn1_w.shape[0]
    r = lambda *s: torch.randn(*s, generator=gen) * 0.02             # noqa: E731
    sd = {"bert.embeddings.word_embeddings.weight": r(m.word_emb.shape[0], c),
          "bert.embeddings.position_embeddings.weight": r(m.pos_emb.shape[0], c),
          "bert.embeddings.token_type_embeddings.weight": r(m.seg_emb.shape[0], c),
          "bert.embeddings.LayerNorm.gamma": 1 + r(c), "bert.embeddings.LayerNorm.beta": r(c),
          "bert.pooler.dense.weight": r(c, c), "bert.pooler.dense.bias": r(c),
          "classifier.weight": r(m.num_labels, c), "classifier.bias": r(m.num_labels)}
    for i in range(m.num_layers):
        p = "bert.encoder.layer.%d." % i
        for n in ("query", "key", "value"):
            sd[p + "attention.self.%s.weight" % n], sd[p + "attention.self.%s.bias" % n] = r(c, c), r(c)
        sd.update({p + "attention.output.dense.weight": r(c, c), p + "attention.output.dense.bias": r(c),
                   p + "attention.output.LayerNorm.gamma": 1 + r(c), p + "attention.output.LayerNorm.beta": r(c),
                   p + "intermediate.dense.weight": r(f, c), p + "intermediate.dense.bias": r(f),
                   p + "output.dense.weight": r(c, f), p + "output.dense.bias": r(c),
                   p + "output.LayerNorm.gamma": 1 + r(c), p + "output.LayerNorm.beta": r(c)})
    return sd


def test_minilm_teacher_zoo_entry_loads_bert_state_dict():
    net, feeds, fetch, shapes = teacher_zoo.build("minilm_l12_h384")
    assert isinstance(net, ErnieEncoder)
    assert (net.word_emb.shape[0], net.hidden, net.num_layers, net.heads, net.head_dim) == (30522, 384, 12, 12, 32)
    assert (net.layers[0].ffn1_w.shape[0], net.pos_emb.shape[0], net.seg_emb.shape[0]) == (1536, 512, 2)
    assert net.num_labels == 2
    assert feeds == ["input_ids", "position_ids", "segment_ids", "input_mask"] and fetch == ["logits"]
    assert shapes == teacher_zoo.build("ernie_tiny")[3]
    sd = _bert_state_dict(net, torch.Generator().manual_seed(0))
    assert net.load_bert_state_dict(sd) == []
    assert torch.equal(net.layers[11].qkv_w[384:768], sd["bert.encoder.layer.11.attention.self.key.weight"])
    assert torch.equal(net.emb_ln_g, sd["bert.embeddings.LayerNorm.gamma"])
    b, l = 2, 9
    ids = torch.randint(0, 30522, (b, l, 1))
    pos = torch.arange(l).expand(b, l).reshape(b, l, 1)
    mask = torch.ones(b, l, 1)
    mask[1, 5:] = 0
    out = net(ids, pos, torch.zeros_like(ids), mask)
    assert out.shape == (b, 2) and torch.isfinite(out).all()
    assert minilm_l12_h384(num_labels=3).cls_w.shape == (3, 384)


def test_train_example_heads():
    out = _run(["examples/distill/nlp/train.py", "--model", "ernie", "--heads", "12", "--epochs", "1", "--samples",
                "32", "--vocab", "400", "--seq_len", "16"])
    assert "loss" in out, out


def test_distill_example_heads():
    out = _run(["examples/distill/nlp/distill.py", "--model", "ernie", "--heads", "12", "--epochs", "1", "--vocab",
                "400"])
    assert "loss" in out, out


def test_examples_parse_heads():
    e = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    for script in ("train.py", "distill.py"):
        p = subprocess.run([sys.executable, "examples/distill/nlp/" + script, "--help"], cwd=ROOT, env=e,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
        assert p.returncode == 0 and "--heads" in p.stdout, p.stdout
