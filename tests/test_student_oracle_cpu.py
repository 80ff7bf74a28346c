"""The checker functions of tests/student_oracle.py on synthetic records built on the CPU: float32 computations rounded
to bf16 must pass, and small corruptions (one ulp, a swapped addend, a zeroed tail row of a packed dqkv, a shifted
dropout offset, a parameter gradient missing or counted twice) must fail and name their site."""
import math

import pytest
import torch

import f64_bounds as fb
import student_oracle as so
from edl_b200 import ops

BF = torch.bfloat16
SEED, OFF, P = 1234, 40, 0.1


def _bf(*shape, gen, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).to(BF)


def _smallest_rounding(ref64):
    """Flat index of the element whose bf16 rounding error is smallest relative to its ulp: one ulp there cannot hide
    in the bound."""
    err = (fb.bf16_round(ref64) - ref64).abs() / fb.ulp(ref64.abs(), 8).clamp_min(1e-300)
    return int(err.reshape(-1).argmin())


def test_gemm_checks():
    gen = torch.Generator().manual_seed(0)
    a, b, add = _bf(200, 136, gen=gen), _bf(72, 136, gen=gen, scale=0.1), _bf(200, 72, gen=gen)
    shift = torch.randn(72, generator=gen)
    out = (a.float() @ b.float().t() + add.float() + shift).to(BF)
    so.check_gemm(out, a, b, "layers.0.attention out forward", add=add, shift=shift)
    bad = out.clone()
    i = _smallest_rounding(fb.gemm_ref(a, b, add=add, shift=shift.double())[0])
    bad.view(torch.int16).view(-1)[i] += 1
    with pytest.raises(AssertionError, match=r"layers\.0\.attention out forward"):
        so.check_gemm(bad, a, b, "layers.0.attention out forward", add=add, shift=shift)
    other = _bf(200, 72, gen=gen)                                         # the dgrad took the wrong addend
    swapped = (a.float() @ b.float().t() + other.float() + shift).to(BF)
    with pytest.raises(AssertionError, match=r"layers\.1\.ffn dgrad dx"):
        so.check_gemm(swapped, a, b, "layers.1.ffn dgrad dx", add=add, shift=shift)
    # the dgrad form (B MN-major) and a weight gradient with its split
    dy = _bf(300, 72, gen=gen)
    so.check_gemm((dy.float() @ b.float()).to(BF), dy, b, "dgrad", b_mn_major=True)
    wg = (dy.float().t() @ a[:1].expand(300, -1).float()).to(BF)
    so.check_wgrad(wg, dy, a[:1].expand(300, -1).contiguous(), 2, "layers.0.ffn ffn1 wgrad")
    wrong = wg.clone()
    wrong[3] = 0
    with pytest.raises(AssertionError, match=r"layers\.0\.ffn ffn1 wgrad"):
        so.check_wgrad(wrong, dy, a[:1].expand(300, -1).contiguous(), 2, "layers.0.ffn ffn1 wgrad")


def _lse32(qkv, mask, b, l, h):
    """fp32 lse [B, H, L] (log2 units of s log2(e) / 8), +inf without a valid key."""
    x = qkv.float().view(b, l, 3, h, 64)
    q, k = (x[:, :, i].transpose(1, 2) for i in range(2))
    cs = (q @ k.transpose(-1, -2)) * (math.log2(math.e) / 8)
    cs = cs.masked_fill(~(mask != 0).view(b, 1, 1, l), float("-inf"))
    m = cs.amax(-1, keepdim=True)
    mf = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    tot = torch.exp2(cs - mf).sum(-1)
    return torch.where(tot > 0, mf.squeeze(-1) + torch.log2(tot), torch.full_like(tot, float("inf")))


def _padded_record(b=3, l=70, h=2, seed=1):
    gen = torch.Generator().manual_seed(seed)
    qkv = _bf(b * l, 3 * h * 64, gen=gen, scale=1.5)
    mask = (torch.rand(b, l, generator=gen) > 0.3).to(torch.uint8)
    mask[0] = 0
    mask[1, 0] = 0
    out = ops.transformer.attention_reference(qkv, mask, b, l, h)
    return dict(layout="padded", mask=mask, b=b, l=l, qkv=qkv, heads=h, drop=None, out=out,
                lse=_lse32(qkv, mask, b, l, h))


def test_attention_forward_and_lse_checks():
    r = _padded_record()
    ro, rl = so.check_attention_forward(r, "layers.0.attention forward")
    assert ro <= 1 and rl <= 1
    assert torch.isinf(r["lse"][0]).all()
    bad = dict(r, lse=r["lse"].clone())
    bad["lse"][2, 1, 5] += 0.05
    with pytest.raises(AssertionError, match=r"layers\.0\.attention forward lse"):
        so.check_attention_forward(bad, "layers.0.attention forward")
    bad = dict(r, lse=r["lse"].clone())
    bad["lse"][0, 0, 0] = 0.0                                             # a row without a valid key must be +inf
    with pytest.raises(AssertionError, match=r"layers\.0\.attention forward lse"):
        so.check_attention_forward(bad, "layers.0.attention forward")
    bad = dict(r, out=r["out"].clone())
    bad["out"][80] = bad["out"][81]
    with pytest.raises(AssertionError, match=r"layers\.0\.attention forward"):
        so.check_attention_forward(bad, "layers.0.attention forward")


def test_packed_attention_checks():
    lens, h = [1, 9, 64, 5], 2
    cu = [0] + torch.tensor(lens).cumsum(0).tolist()
    t = cu[-1]
    gen = torch.Generator().manual_seed(2)
    qkv = _bf(t, 3 * h * 64, gen=gen, scale=1.5)
    key_mask = torch.ones(t, dtype=torch.uint8)
    key_mask[cu[1]:cu[2]] = 0                                             # a fully key-masked sequence
    key_mask[cu[2]] = 0                                                   # a masked token 0
    cu_t = torch.tensor(cu, dtype=torch.int32)
    out = ops.transformer.attention_varlen_reference(qkv, cu_t, max(lens), h, key_mask)
    lse = torch.cat([_lse32(qkv[s:e], key_mask[s:e].view(1, -1), 1, e - s, h)[0] for s, e in zip(cu[:-1], cu[1:])], 1)
    r = dict(layout="packed", cu=cu, cu_t=cu_t, max_len=max(lens), key_mask=key_mask, qkv=qkv, heads=h, drop=None,
             out=out, lse=lse)
    so.check_attention_forward(r, "layers.0.attention forward (packed)")
    dout = _bf(t, h * 64, gen=gen)
    ref = torch.cat([so.attention_f64(qkv[s:e], key_mask[s:e].view(1, -1), dout[s:e], 1, e - s, h)[2]
                     for s, e in zip(cu[:-1], cu[1:])])
    dqkv = ref.to(BF)
    so.check_attention_backward(r, dqkv, dout, "layers.0.attention backward (packed)")
    tail = dqkv.clone()
    tail[-1] = 0                                                          # the last packed row lost
    with pytest.raises(AssertionError, match=r"layers\.0\.attention backward \(packed\)"):
        so.check_attention_backward(r, tail, dout, "layers.0.attention backward (packed)")


def test_layernorm_checks():
    gen = torch.Generator().manual_seed(3)
    x = _bf(50, 136, gen=gen, scale=2.0)
    gamma, beta = torch.randn(136, generator=gen), torch.randn(136, generator=gen)
    y = ops.transformer.layer_norm_reference(x, gamma, beta, 1e-12)
    so.check_layernorm(x, gamma, beta, 1e-12, y, "layers.0.ln1 forward")
    xr, g, b = x.float().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    dy = _bf(50, 136, gen=gen)
    ops.transformer.layer_norm_reference(xr, g, b, 1e-12).backward(dy.float())
    dx = xr.grad.to(BF)
    so.check_layernorm_backward(x, dy, gamma, 1e-12, dx, g.grad, b.grad, "layers.0.ln1 backward")
    bad = dx.clone()
    bad[7, 3] = bad[7, 3] * 1.05 + 0.01
    with pytest.raises(AssertionError, match=r"layers\.0\.ln1 backward dx"):
        so.check_layernorm_backward(x, dy, gamma, 1e-12, bad, g.grad, b.grad, "layers.0.ln1 backward")
    gb = b.grad.clone()
    gb[0] += 1e-3 * gb.abs().max()
    with pytest.raises(AssertionError, match=r"layers\.0\.ln1 backward dbeta"):
        so.check_layernorm_backward(x, dy, gamma, 1e-12, dx, g.grad, gb, "layers.0.ln1 backward")


def test_dropout_checks():
    gen = torch.Generator().manual_seed(4)
    x = _bf(33, 40, gen=gen)
    draw = (SEED, OFF, P)
    keep = ops.dropout_keep_reference(SEED, OFF, torch.arange(x.numel()), P).view(x.shape)
    scale = torch.tensor(1.0 / (1.0 - P), dtype=torch.float32).item()
    y = torch.where(keep, (x.float() * scale).to(BF), torch.zeros_like(x))
    so.check_dropout_apply(y, x, draw, "layers.0.ffn branch dropout backward")
    with pytest.raises(AssertionError, match=r"layers\.0\.ffn branch dropout backward"):
        so.check_dropout_apply(y, x, (SEED, OFF + 4, P), "layers.0.ffn branch dropout backward")
    # the residual-dropout epilogue: kept within the bound, dropped elements the addend bit for bit
    a, w, add = _bf(33, 64, gen=gen), _bf(40, 64, gen=gen, scale=0.1), _bf(33, 40, gen=gen)
    shift = torch.randn(40, generator=gen)
    z = so.rowwise_z(draw, 33, 40, "cpu")
    out = (add.float() + z.float() * (a.float() @ w.float().t() + shift)).to(BF)
    so.check_residual_dropout(out, a, w, shift, add, z, "layers.1.attention out forward (dropout)")
    with pytest.raises(AssertionError, match=r"layers\.1\.attention out forward"):
        so.check_residual_dropout(out, a, w, shift, add, so.rowwise_z((SEED, OFF - 4, P), 33, 40, "cpu"),
                                  "layers.1.attention out forward (dropout)")
    # the sites' draw order and offsets
    sites = ["embeddings", "layers.0.attention probabilities", "layers.0.attention branch", "layers.0.ffn branch",
             "pooled"]
    draws = [(SEED, OFF + 4 * k, P, s) for k, s in enumerate(sites)]
    so.check_draw_order(draws, sites)
    shifted = list(draws)
    shifted[3] = (SEED, OFF + 16, P, sites[3])
    with pytest.raises(AssertionError, match=r"layers\.0\.ffn branch drew"):
        so.check_draw_order(shifted, sites)
    with pytest.raises(AssertionError, match="sites drawn"):
        so.check_draw_order(draws[:1] + draws[2:3] + draws[1:2] + draws[3:], sites)


def test_coverage_and_bias_checks():
    names = ["word_emb", "layers.0.qkv_w", "cls_b"]
    so.check_coverage(names, {n: 1 for n in names})
    with pytest.raises(AssertionError, match=r"layers\.0\.qkv_w: gradient checked 0 times"):
        so.check_coverage(names, {"word_emb": 1, "cls_b": 1})
    with pytest.raises(AssertionError, match=r"cls_b: gradient checked 2 times"):
        so.check_coverage(names, {"word_emb": 1, "layers.0.qkv_w": 1, "cls_b": 2})
    gen = torch.Generator().manual_seed(5)
    dy = _bf(500, 24, gen=gen)
    db = dy.float().sum(0)
    so.check_bias(db, dy, "layers.0.attention qkv bias gradient")
    with pytest.raises(AssertionError, match=r"layers\.0\.attention qkv bias gradient"):
        so.check_bias(dy[1:].float().sum(0), dy, "layers.0.attention qkv bias gradient")   # row 0 dropped
