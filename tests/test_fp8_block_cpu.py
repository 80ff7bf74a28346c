"""Block-scaled e4m3 on CPU: the plain-torch paths of ``quantize_e4m3_blocks``, ``quantize_weight_blocks`` and
``gemm_fp8_blockscaled`` (the reference the GPU tests compare against), and the block mode's switch on the model."""
import pytest
import torch

from edl_b200.ops import fp8


def _e4m3(q):
    return q.view(torch.float8_e4m3fn).float()


def _half_ulp(v):
    """Half a unit in the last place of e4m3 at |v| (3 mantissa bits; subnormal spacing 2^-9 below 2^-6)."""
    e = torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -6)))
    return 2.0 ** (e - 4)


def _row_scaled(m, k, gen, lo=-4.0, hi=4.0):
    """randn rows whose magnitudes step from 2^lo to 2^hi (bf16)."""
    rs = 2.0 ** torch.linspace(lo, hi, m)
    return (torch.randn(m, k, generator=gen) * rs[:, None]).bfloat16()


@pytest.mark.parametrize("m,k", [(1, 64), (257, 144), (300, 1024), (128, 64)])
def test_quantiser_round_trip_within_half_ulp_of_block_scale(m, k):
    gen = torch.Generator().manual_seed(m + k)
    x = _row_scaled(m, k, gen)
    q, sa = fp8.quantize_e4m3_blocks(x)
    kb = -(-k // 128)
    assert q.dtype == torch.uint8 and q.shape == (m, k) and q.is_contiguous()
    assert sa.dtype == torch.float32 and sa.shape == (kb, m) and sa.is_contiguous()
    xf = x.float()
    for b in range(kb):
        blk = slice(b * 128, min(k, (b + 1) * 128))
        amax = xf[:, blk].abs().amax(1)
        assert torch.equal(sa[b], amax / torch.full_like(amax, 448.0))     # every block here is non-zero
        v = xf[:, blk] / sa[b][:, None]
        assert v.abs().max() <= 448.0 * (1 + 1e-6)
        err = (v - _e4m3(q[:, blk])).abs()
        assert (err <= _half_ulp(v) * (1 + 1e-6)).all()


def test_quantiser_zero_blocks_give_zeros_with_scale_one():
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(130, 272, generator=gen).bfloat16()
    x[:, 128:256] = 0                     # a whole middle block
    x[7] = 0                              # a whole row, tail block included
    q, sa = fp8.quantize_e4m3_blocks(x)
    assert (q[:, 128:256] == 0).all() and (q[7] == 0).all()
    assert (sa[1] == 1).all() and (sa[:, 7] == 1).all()
    assert (sa[0, :7] != 1).all() and (sa[2, 8:] != 1).all()


def test_quantiser_tail_block_scale_uses_real_elements_only():
    x = torch.zeros(3, 144).bfloat16()
    x[:, :128] = 100.0
    x[:, 128:] = torch.tensor([0.5, -2.0, 0.25]).bfloat16()[:, None]
    _, sa = fp8.quantize_e4m3_blocks(x)
    assert torch.equal(sa[1], torch.tensor([0.5, 2.0, 0.25]) / torch.full((3,), 448.0))


def test_quantiser_accepts_strided_rows():
    gen = torch.Generator().manual_seed(1)
    big = _row_scaled(40, 288, gen)
    x = big[:, :144]
    q, sa = fp8.quantize_e4m3_blocks(x)
    q2, sa2 = fp8.quantize_e4m3_blocks(x.contiguous())
    assert torch.equal(q, q2) and torch.equal(sa, sa2)


@pytest.mark.parametrize("n,k", [(64, 64), (200, 144), (256, 1024)])
def test_weight_blocks_round_trip(n, k):
    gen = torch.Generator().manual_seed(n)
    w = torch.randn(n, k, generator=gen) * 0.05
    w[:, :128] *= 40.0                     # a first k-block with a much larger range than the rest
    q, sb = fp8.quantize_weight_blocks(w)
    nb, kb = -(-n // 128), -(-k // 128)
    assert q.shape == (n, k) and sb.shape == (nb, kb)
    for i in range(nb):
        for b in range(kb):
            rows, cols = slice(i * 128, (i + 1) * 128), slice(b * 128, (b + 1) * 128)
            amax = w[rows, cols].abs().max()
            assert torch.equal(sb[i, b], amax / torch.tensor(448.0))
            v = w[rows, cols] / sb[i, b]
            assert ((v - _e4m3(q[rows, cols])).abs() <= _half_ulp(v) * (1 + 1e-6)).all()


def _dequantised_reference(a8, sa, b8, sb, col_scale, col_shift, relu):
    n = b8.shape[0]
    a = _e4m3(a8) * sa.t().repeat_interleave(128, 1)[:, :a8.shape[1]]
    b = _e4m3(b8) * sb.repeat_interleave(128, 0)[:n].repeat_interleave(128, 1)[:, :b8.shape[1]]
    d = a @ b.t()
    if col_scale is not None:
        d = d * col_scale
    if col_shift is not None:
        d = d + col_shift
    return torch.relu(d) if relu else d


@pytest.mark.parametrize("m,n,k", [(128, 128, 128), (70, 200, 144), (33, 64, 64), (257, 300, 512)])
@pytest.mark.parametrize("epilogue", [False, True])
def test_block_gemm_equals_dequantise_then_matmul(m, n, k, epilogue):
    gen = torch.Generator().manual_seed(m * n + k)
    x = _row_scaled(m, k, gen)
    w = torch.randn(n, k, generator=gen) * 0.05
    a8, sa = fp8.quantize_e4m3_blocks(x)
    b8, sb = fp8.quantize_weight_blocks(w)
    cs = torch.rand(n, generator=gen) + 0.5 if epilogue else None
    sh = torch.randn(n, generator=gen) if epilogue else None
    out = torch.empty(m, n)
    fp8.gemm_fp8_blockscaled(a8, sa, b8, sb, cs, sh, relu=epilogue, out=out)
    ref = _dequantised_reference(a8, sa, b8, sb, cs, sh, epilogue)
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5 * ref.abs().max().item())
    d = fp8.gemm_fp8_blockscaled(a8, sa, b8, sb, cs, sh, relu=epilogue)    # default bf16 output
    assert d.dtype == torch.bfloat16 and d.shape == (m, n)
    torch.testing.assert_close(d.float(), ref, rtol=1e-2, atol=1e-2 * ref.abs().max().item())


def _row_errors(x, deq):
    return ((x - deq).norm(dim=1) / x.norm(dim=1))


def test_block_scaling_keeps_rows_spanning_16_binades():
    gen = torch.Generator().manual_seed(3)
    x = _row_scaled(64, 512, gen, lo=-8.0, hi=8.0).float()
    q, sa = fp8.quantize_e4m3_blocks(x.bfloat16())
    deq = _e4m3(q) * sa.t().repeat_interleave(128, 1)
    block_err = _row_errors(x, deq)
    assert block_err.max() <= 0.07, block_err.max()
    # the per-tensor path on the same tensor: one scale fitted to the largest row
    scale = (x.abs().max() / fp8.E4M3_MAX).view(1)
    qt = fp8.quantize_e4m3(x.bfloat16(), scale)
    tensor_err = _row_errors(x, _e4m3(qt) * scale)
    assert tensor_err.max() > block_err.max(), (tensor_err.max(), block_err.max())


def test_enable_fp8_block_mode_needs_no_batch():
    from edl_b200.models.resnext import FoldedConv, ResNeXt_tiny

    m = ResNeXt_tiny().eval()
    convs = [c for c in m.modules() if isinstance(c, FoldedConv)]
    eligible = sum(1 for c in convs if c.fp8_eligible())
    assert eligible > 0
    assert m.enable_fp8(scaling="block") == eligible
    for c in convs:
        if c.fp8_eligible():
            w8, sb = fp8.quantize_weight_blocks(c.weight.view(c.cout, c.cin))
            assert torch.equal(c.w8_blocks, w8) and torch.equal(c.w_block_scales, sb)
            assert getattr(c, "w8", None) is None
        else:
            assert getattr(c, "w8_blocks", None) is None
    with pytest.raises(ValueError):
        m.enable_fp8(scaling="row")
    with pytest.raises(ValueError):
        m.enable_fp8()                      # tensor scaling still needs its calibration batch
