"""The ERNIE sequence teacher on the GPU kernels, against float64.

Attention bound (criterion 1 of tests/f64_bounds.py, per element).  The kernel forms s~_j = fl(q . k_j) with fp32 MMA
steps, |s~_j - s_j| <= (64 / 16 + 1) 2^-23 sum_d |q_d k_jd|, scales by c = log2(e) / 8 and subtracts the running
maximum (two more fp32 roundings, 2^-23 of |c s_j| and of |c s_j - m|), so the exponent of key j is off by at most
delta_j (log2 units).  p~_j = bf16(ex2(.)) then has relative error
    eps_j <= 2^-8 (bf16 rounding of P before P V) + 2^-21 (ex2.approx) + 1.01 ln2 delta_j,
while the common factor 2^-m cancels between P V and the row sum, which the kernel takes over the same rounded p~.  The
weights w~_j = p~_j / sum p~ therefore satisfy |w~_j - w_j| <= 2 eps / (1 - eps) w_j with eps = max_j eps_j over the
row's valid keys, and
    |O~ - O| <= (2 eps / (1 - eps) + tau_acc) sum_j w_j |v_j|,   tau_acc = (8 n_tiles + 32) 2^-23
(fp32 accumulation of P V and of the row sum, the per-tile rescales and the final division), plus half a bf16 ulp of the
stored value (``check_bf16`` with ``tau = 1`` and this slack as ``mag``).  A row without a valid key must be exactly 0.

LayerNorm bound.  With fp32 sums of at most C terms, |mean~ - mean| <= C 2^-23 mean|x| = dmu; the variance is taken
about mean~ (a second-order change), so rstd~ has relative error eps_r <= (C + 2) 2^-24 + 2^-21 (rsqrtf) +
(dmu rstd)^2 / 2, and per element
    |y~ - y| <= |gamma| rstd (dmu + dx + |x - mean| eps_r) + 4 2^-23 (|x - mean| rstd |gamma| + |beta|)
where dx is the fp32 rounding of the embedding sum (2 2^-23 of the sum of the three |rows|; 0 for plain LayerNorm).

GELU epilogue: the GEMM's slack ``tau(k) * mag`` grows by at most max|gelu'| = 1.13 through the activation, and the
fp32 evaluation of 0.5 v (1 + erf(v / sqrt 2)) adds 6 2^-23 |v|; both criteria of ``check_bf16`` apply.

Worst ratios observed on one NVIDIA H100 80GB HBM3 (700 W power limit), criterion 1 / criterion 2:

    attention (all shapes and masks; criterion 1 only)              c1 0.554
    LayerNorm, embedding + LayerNorm                                c1 1.000   c2 1.00
    GELU epilogue                                                   c1 0.999   c2 1.00
    ernie_base layer by layer (every GEMM, attention, LayerNorm)    c1 0.997   c2 1.00"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from edl_b200 import ops
from edl_b200.models import ernie, teacher_zoo
from f64_bounds import EPS32, check_bf16, gemm_ref, guarded, tau as gemm_tau
from student_oracle import attention_ref, ln_ref

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

DEV = torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------------------ attention
def _mask(kind, b, l, gen):
    if kind == "none":
        return None
    m = torch.zeros(b, l, dtype=torch.uint8)
    for i in range(b):
        k = kind if kind != "mixed" else ("full", "right", "holes", "one", "empty")[i % 5]
        if k == "full":
            m[i] = 1
        elif k == "right":
            m[i, :int(torch.randint(1, l + 1, (1,), generator=gen))] = 1
        elif k == "holes":
            m[i] = (torch.rand(l, generator=gen) > 0.5).to(torch.uint8)
        elif k == "one":
            m[i, int(torch.randint(0, l, (1,), generator=gen))] = 1
    return m.to(DEV)


@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("seq_len", [1, 7, 64, 65, 128, 200, 256, 512])
@pytest.mark.parametrize("batch", [1, 3, 16])
def test_attention_vs_float64(batch, seq_len, heads):
    gen = torch.Generator().manual_seed(batch * 1000 + seq_len * 10 + heads)
    kinds = ["mixed"] if batch == 16 else ["none", "full", "right", "holes", "one", "empty"]
    for kind in kinds:
        mask = _mask(kind, batch, seq_len, gen)
        rows, cols = batch * seq_len, 3 * heads * 64
        vals = (torch.randn(rows, cols, generator=gen) * 2).to(torch.bfloat16)
        qkv = guarded((rows, cols), pad_rows=3, values=vals.to(DEV))               # NaN rows around the operand
        out = guarded((rows, heads * 64), pad_rows=3, fill=7.0, values=torch.full((rows, heads * 64), -3.0, device=DEV,
                                                                                  dtype=torch.bfloat16))
        assert ops.attention_supported(qkv.t, batch, seq_len, heads)
        ops.attention(qkv.t, mask, batch, seq_len, heads, out=out.t)
        torch.cuda.synchronize()
        out.assert_untouched("attention output %s" % kind)
        ref, slack = attention_ref(qkv.t, mask, batch, seq_len, heads)
        check_bf16(out.t, ref, slack, tau=1.0, criteria=(1,), what="attention B %d L %d H %d mask %s" % (
            batch, seq_len, heads, kind))
        if mask is not None:
            dead = (mask.sum(1) == 0).repeat_interleave(seq_len)
            assert torch.equal(out.t[dead], torch.zeros_like(out.t[dead]))


# ---------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("c", [768, 40])
@pytest.mark.parametrize("rows", [1, 13, 4099])
def test_layer_norms_vs_float64(c, rows):
    gen = torch.Generator().manual_seed(rows + c)
    x = (torch.randn(rows, c, generator=gen) * 3 + 0.5).to(torch.bfloat16).to(DEV)
    g, b = torch.randn(c, generator=gen).to(DEV), torch.randn(c, generator=gen).to(DEV)
    assert ops.layer_norm_supported(x)
    y = ops.layer_norm(x, g, b, 1e-12)
    ref, slack = ln_ref(x.double(), g, b, 1e-12)
    check_bf16(y, ref, slack, tau=1.0, what="layer_norm %d x %d" % (rows, c))

    word, pos, seg = (torch.randn(n, c, generator=gen).to(torch.bfloat16).to(DEV) for n in (1000, 513, 2))
    ids, pids, sids = (torch.randint(0, n, (rows,), generator=gen).to(DEV) for n in (1000, 513, 2))
    out = guarded((rows, c), pad_rows=2, fill=5.0)
    ops.embedding_layernorm(ids, pids, sids, word, pos, seg, g, b, 1e-12, out=out.t)
    torch.cuda.synchronize()
    out.assert_untouched("embedding_layernorm output")
    terms = [word.double()[ids], pos.double()[pids], seg.double()[sids]]
    x64 = sum(terms)
    ref, slack = ln_ref(x64, g, b, 1e-12, dx=2 * EPS32 * sum(t.abs() for t in terms))
    check_bf16(out.t, ref, slack, tau=1.0, what="embedding_layernorm %d x %d" % (rows, c))
    with pytest.raises(IndexError):
        ops.embedding_layernorm(ids, pids, sids + 2, word, pos, seg, g, b, 1e-12)


# ---------------------------------------------------------------------------------------------- GELU epilogue
def gelu_ref(a, w, bias):
    pre, mag = gemm_ref(a, w, shift=bias)
    ref = 0.5 * pre * (1 + torch.erf(pre / math.sqrt(2)))
    return ref, pre, mag


@pytest.mark.parametrize("m,n,k", [(4096, 3072, 768), (200, 72, 40), (129, 136, 100), (77, 40, 72), (1, 8, 64),
                                   (300, 512, 1000)])
def test_gelu_epilogue_vs_float64(m, n, k):
    gen = torch.Generator().manual_seed(m + n + k)
    a = torch.randn(m, k, generator=gen).to(torch.bfloat16).to(DEV)
    w = (torch.randn(n, k, generator=gen) / math.sqrt(k)).to(torch.bfloat16).to(DEV)
    bias = torch.randn(n, generator=gen).to(DEV)
    out = guarded((m, n), pad_rows=2, pad_cols=8, fill=3.0)
    ops.gemm_bf16(a, w, out=out.t, col_shift=bias, gelu=True)
    torch.cuda.synchronize()
    out.assert_untouched("gelu output")
    ref, pre, mag = gelu_ref(a, w, bias)
    slack = gemm_tau(k) * 1.13 * mag + 6 * EPS32 * pre.abs()
    check_bf16(out.t, ref, slack, tau=1.0, what="gemm gelu %d x %d x %d" % (m, n, k))


# ------------------------------------------------------------------------------------------------ whole encoder
def _inputs(b, l, seed):
    gen = torch.Generator().manual_seed(seed)
    lens = torch.randint(l // 4, l + 1, (b,), generator=gen)
    lens[0] = l
    mask = (torch.arange(l)[None] < lens[:, None]).float()
    ids = torch.randint(0, 18000, (b, l), generator=gen)
    seg = torch.randint(0, 2, (b, l), generator=gen)
    pos = torch.arange(l).expand(b, l).contiguous()
    return [t.to(DEV) for t in (ids, pos, seg, mask)]


def _torch_forward32(model, ids, pos, seg, mask):
    """fp32 torch forward with the bf16-rounded weights of the kernel path."""
    r = lambda t: t.detach().to(torch.bfloat16).float()                               # noqa: E731
    b, l = ids.shape
    c, h = model.hidden, model.heads
    x = r(model.word_emb)[ids] + r(model.pos_emb)[pos] + r(model.seg_emb)[seg]
    x = F.layer_norm(x, (c,), model.emb_ln_g.float(), model.emb_ln_b.float(), model.eps)
    keep = (mask != 0).view(b, 1, 1, l)
    for lyr in model.layers:
        q, k, v = F.linear(x, r(lyr.qkv_w), lyr.qkv_b.float()).view(b, l, 3, h, 64).permute(2, 0, 3, 1, 4)
        ctx = F.scaled_dot_product_attention(q, k, v, attn_mask=keep).transpose(1, 2).reshape(b, l, c)
        x = F.layer_norm(F.linear(ctx, r(lyr.out_w), lyr.out_b.float()) + x, (c,), lyr.ln1_g.float(), lyr.ln1_b.float(),
                         model.eps)
        f = F.gelu(F.linear(x, r(lyr.ffn1_w), lyr.ffn1_b.float()))
        x = F.layer_norm(F.linear(f, r(lyr.ffn2_w), lyr.ffn2_b.float()) + x, (c,), lyr.ln2_g.float(), lyr.ln2_b.float(),
                         model.eps)
    pooled = torch.tanh(F.linear(x[:, 0], r(model.pool_w), model.pool_b.float()))
    return F.linear(pooled, r(model.cls_w), model.cls_b.float())


@pytest.mark.parametrize("seq_len", [128, 256])
def test_ernie_base_layer_by_layer_and_end_to_end(seq_len):
    torch.manual_seed(0)
    model = ernie.ernie_base().to(DEV).eval()
    with torch.no_grad():
        model.cls_w.mul_(20)                  # decisive logits for the top-1 comparison
    b = 16
    ids, pos, seg, mask = _inputs(b, seq_len, seq_len)
    ops.reset_fallbacks()
    logits = model(ids, pos, seg, mask)
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()

    # layer by layer: every op of the kernel path, fed its own bf16 input, against float64
    w = model._device_weights()
    word, pemb, semb, g0, b0 = w["emb"]
    m8 = (mask != 0).to(torch.uint8).contiguous()
    x = ops.embedding_layernorm(ids, pos, seg, word, pemb, semb, g0, b0, model.eps)
    terms = [word.double()[ids.reshape(-1)], pemb.double()[pos.reshape(-1)], semb.double()[seg.reshape(-1)]]
    ref, slack = ln_ref(sum(terms), g0, b0, model.eps, dx=2 * EPS32 * sum(t.abs() for t in terms))
    check_bf16(x, ref, slack, tau=1.0, what="embeddings")
    c = model.hidden
    for i, (qkv_w, qkv_b, out_w, out_b, g1, be1, f1_w, f1_b, f2_w, f2_b, g2, be2) in enumerate(w["layers"]):
        qkv = ops.gemm_bf16(x, qkv_w, col_shift=qkv_b)
        check_bf16(qkv, *gemm_ref(x, qkv_w, shift=qkv_b), k=c, what="layer %d qkv" % i)
        ctx = ops.attention(qkv, m8, b, seq_len, model.heads)
        check_bf16(ctx, *attention_ref(qkv, m8, b, seq_len, model.heads), tau=1.0, criteria=(1,),
                   what="layer %d attention" % i)
        h1 = ops.gemm_bf16(ctx, out_w, col_shift=out_b, add=x)
        check_bf16(h1, *gemm_ref(ctx, out_w, add=x, shift=out_b), k=c, what="layer %d out proj" % i)
        x1 = ops.layer_norm(h1, g1, be1, model.eps)
        check_bf16(x1, *ln_ref(h1.double(), g1, be1, model.eps), tau=1.0, what="layer %d ln1" % i)
        f = ops.gemm_bf16(x1, f1_w, col_shift=f1_b, gelu=True)
        ref, pre, mag = gelu_ref(x1, f1_w, f1_b)
        check_bf16(f, ref, gemm_tau(c) * 1.13 * mag + 6 * EPS32 * pre.abs(), tau=1.0, what="layer %d ffn1" % i)
        h2 = ops.gemm_bf16(f, f2_w, col_shift=f2_b, add=x1)
        check_bf16(h2, *gemm_ref(f, f2_w, add=x1, shift=f2_b), k=f.shape[1], what="layer %d ffn2" % i)
        x = ops.layer_norm(h2, g2, be2, model.eps)
        check_bf16(x, *ln_ref(h2.double(), g2, be2, model.eps), tau=1.0, what="layer %d ln2" % i)
    pool_w, pool_b, cls_w, cls_b = w["head"]
    cls_rows = x.view(b, seq_len, c)[:, 0]
    pre = ops.linear_bf16(cls_rows, pool_w, pool_b)
    check_bf16(pre, *gemm_ref(cls_rows, pool_w, shift=pool_b), k=c, what="pooler")
    pooled = torch.tanh(pre)
    lg = ops.gemm_bf16(pooled, cls_w, col_shift=cls_b)
    check_bf16(lg, *gemm_ref(pooled, cls_w, shift=cls_b), k=c, what="classifier")
    # the model's forward is exactly this sequence of launches
    assert torch.equal(lg[:, :model.num_labels].float(), logits)

    # end to end against an fp32 torch forward with the same bf16 weights
    want = _torch_forward32(model, ids, pos, seg, mask)
    cos = F.cosine_similarity(logits.flatten()[None].double(), want.flatten()[None].double()).item()
    agree = (logits.argmax(1) == want.argmax(1)).float().mean().item()
    assert cos > 0.999 and agree >= 15 / 16, (cos, agree)

    # CUDA graph: the captured forward replays the eager bits
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        model(ids, pos, seg, mask)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = model(ids, pos, seg, mask)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, logits)
    assert ops.fallbacks() == {}, ops.fallbacks()


def test_teacher_server_on_cuda():
    from edl_b200.distill.predict_client import PredictClient  # noqa: F401  (the server's client stack is importable)
    from edl_b200.distill.distill_reader import DistillReader
    from edl_b200.distill.teacher_server import TeacherServer

    torch.manual_seed(0)
    model, feeds, fetches, shapes = teacher_zoo.build("ernie_tiny")
    l = 32
    gen = torch.Generator().manual_seed(9)
    data = []
    for i in range(10):
        mask = np.zeros((l, 1), np.float32)
        mask[:1 + 3 * i] = 1
        data.append((torch.randint(0, 1000, (l, 1), generator=gen).numpy(), np.arange(l, dtype=np.int64)[:, None],
                     np.zeros((l, 1), np.int64), mask, np.array([i], np.int64)))
    with TeacherServer(model, feeds, fetches, shapes, device="cuda:0", dtype=torch.bfloat16, max_wait_ms=1.0) as srv:
        dr = DistillReader(ins=feeds + ["label"], predicts=["logits"])
        dr.set_teacher_batch_size(4)
        dr.set_fixed_teacher([srv.endpoint])
        r = dr.set_sample_list_generator(lambda: [data[i:i + 5] for i in range(0, len(data), 5)])
        n = 0
        for batch in r():
            for ids, pos, seg, mask, label, logits in batch:
                feed = [torch.from_numpy(t)[None].to(DEV) for t in (ids, pos, seg, mask)]
                feed[3] = feed[3].to(torch.bfloat16)
                want = srv.model(*feed)[0].cpu().numpy()
                assert np.array_equal(logits, want), (logits, want)
                n += 1
        dr.stop()
    assert n == 10
