"""Block-scaled e4m3 quantiser and GEMM (csrc/gemm_fp8.cu) against their plain-torch CPU paths, and the
teacher's block-scaled fp8 mode: no calibration, no host synchronisation, CUDA-graph capturable."""
import pytest
import torch

from edl_b200.ops import fp8

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def _row_scaled(m, k, seed, lo=-6.0, hi=6.0):
    g = torch.Generator().manual_seed(seed)
    rs = 2.0 ** torch.linspace(lo, hi, m)
    return (torch.randn(m, k, generator=g) * rs[:, None]).bfloat16()


@pytest.mark.parametrize("m", [1, 257, 6272])
@pytest.mark.parametrize("k", [64, 144, 1024])
def test_quantiser_bit_identical_to_cpu(m, k):
    x = _row_scaled(m, k, m + k)
    if m > 2:
        x[m // 2] = 0                                    # an all-zero row: scale 1, zero bytes
    if k > 128:
        x[: m // 3, 128:256] = 0                         # all-zero blocks (for k = 144: the whole tail block)
    q_ref, sa_ref = fp8.quantize_e4m3_blocks(x)
    q, sa = fp8.quantize_e4m3_blocks(x.to(DEV))
    assert torch.equal(q.cpu(), q_ref)
    assert torch.equal(sa.cpu(), sa_ref)


def test_quantiser_strided_rows_bit_identical_to_cpu():
    big = _row_scaled(300, 1152, 7)
    x = big[:, 16:16 + 1040]                             # row pitch 1152, 32-byte offset, K = 1040 (tail of 16)
    q_ref, sa_ref = fp8.quantize_e4m3_blocks(x)
    xg = big.to(DEV)[:, 16:16 + 1040]
    assert xg.stride(0) == 1152
    q, sa = fp8.quantize_e4m3_blocks(xg)
    assert torch.equal(q.cpu(), q_ref) and torch.equal(sa.cpu(), sa_ref)


SHAPES = [(128, 128, 128), (300, 256, 512), (6272, 2048, 1024), (32, 1000, 2048), (257, 64, 144), (100352, 256, 64)]


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("epilogue", [False, True])
def test_block_gemm_matches_cpu_reference(m, n, k, epilogue):
    x = _row_scaled(m, k, m + n + k)
    g = torch.Generator().manual_seed(n)
    w = torch.randn(n, k, generator=g) * 0.05
    a8, sa = fp8.quantize_e4m3_blocks(x.to(DEV))
    b8, sb = fp8.quantize_weight_blocks(w.to(DEV))
    cs = (torch.rand(n, generator=g) + 0.5) if epilogue else None
    sh = torch.randn(n, generator=g) if epilogue else None
    dev = (lambda t: None if t is None else t.to(DEV))
    d = fp8.gemm_fp8_blockscaled(a8, sa, b8, sb, dev(cs), dev(sh), relu=epilogue)
    assert d.dtype == torch.bfloat16 and d.shape == (m, n)
    exact = torch.empty(m, n)
    fp8.gemm_fp8_blockscaled(a8.cpu(), sa.cpu(), b8.cpu(), sb.cpu(), cs, sh, relu=epilogue, out=exact)
    assert _rel(d.cpu(), exact) < 1e-2                   # kernel vs the same fp8 operands in fp32
    full = x.float() @ w.t()
    if epilogue:
        full = torch.relu(full * cs + sh)
    assert _rel(d.cpu(), full) < 8e-2                    # fp8 quantisation error budget of test_fp8_gpu


def test_block_gemm_rejects_bad_input():
    a8, sa = fp8.quantize_e4m3_blocks(torch.randn(64, 256, device=DEV).bfloat16())
    b8, sb = fp8.quantize_weight_blocks(torch.randn(128, 256, device=DEV))
    out = torch.empty(64, 128, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="sa must be"):
        fp8.gemm_fp8_blockscaled(a8, sa.t().contiguous(), b8, sb, out=out)
    with pytest.raises(RuntimeError, match="sb must be"):
        fp8.gemm_fp8_blockscaled(a8, sa, b8, sb[:, :1].contiguous(), out=out)
    with pytest.raises(RuntimeError, match="col_scale"):
        fp8.gemm_fp8_blockscaled(a8, sa, b8, sb, torch.ones(64, device=DEV), out=out)
    with pytest.raises(RuntimeError, match="K mismatch"):
        fp8.gemm_fp8_blockscaled(a8[:, :128], sa[:1].contiguous(), b8, sb, out=out)
    with pytest.raises(RuntimeError, match="16-byte"):
        a72 = torch.zeros(64, 72, device=DEV, dtype=torch.uint8)
        fp8.gemm_fp8_blockscaled(a72, sa[:1].contiguous(), b8[:, :72], sb[:, :1].contiguous(), out=out)
    with pytest.raises(RuntimeError, match="bf16"):
        fp8.quantize_e4m3_blocks(torch.randn(8, 128, device=DEV))
    with pytest.raises(RuntimeError, match="K % 8"):
        fp8.quantize_e4m3_blocks(torch.randn(8, 12, device=DEV).bfloat16())


def _teacher():
    from edl_b200.models.resnext import ResNeXt50_32x4d, to_inference_dtype

    torch.manual_seed(0)
    return to_inference_dtype(ResNeXt50_32x4d(class_dim=100), torch.bfloat16, DEV).eval()


def _agree(out, ref):
    cos = torch.nn.functional.cosine_similarity(out.float().flatten(), ref.float().flatten(), dim=0).item()
    top1 = (out.argmax(-1) == ref.argmax(-1)).float().mean().item()
    return cos, top1


def test_teacher_block_mode_tracks_bf16_logits_without_calibration():
    m = _teacher()
    x = torch.randn(4, 3, 128, 128, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    refs = [m(x).float(), m(x * 16).float()]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")              # switching to block mode must not synchronise
    try:
        n = m.enable_fp8(scaling="block")
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert n >= 30
    for xi, ref in zip([x, x * 16], refs):               # no calibration exists to redo for the larger input
        cos, top1 = _agree(m(xi).float(), ref)
        assert cos > 0.98, cos
        assert top1 >= 0.75, top1


def test_teacher_block_mode_graph_replay_bit_identical():
    m = _teacher()
    m.enable_fp8(scaling="block")
    x = torch.randn(4, 3, 128, 128, device=DEV).bfloat16().contiguous(memory_format=torch.channels_last)
    static_x = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            m(static_x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = m(static_x)
    eager = m(x).clone()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, eager)
    x2 = torch.randn_like(x) * 3
    static_x.copy_(x2)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(y, m(x2))
