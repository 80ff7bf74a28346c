"""The FP8 kernels of csrc/gemm_fp8.cu bit for bit.

Exact-operand GEMMs: e4m3 operands in {0, +-1, +-2}, at most 256 nonzeros per row of A, so every partial sum the tensor
core forms is an integer below 2^10 and is exact however many bits it keeps (at least 11).  Block scales are powers of
two in 2^[-3, 3], so the fp32 promotion of each k-block is exact; ``col_scale`` lies in [0.5, 2) and ``col_shift`` on a
2^-10 grid (below 16 here), so ``acc * col_scale + col_shift`` is exact in float64.  The kernel's output is then exactly
``bf16(f32(acc * col_scale + col_shift))`` (with an addend: ``bf16(f32(f32(...) + add))``), whatever the accumulator
width -- no model of the tensor core is involved.  Operands sit between NaN-byte (0x7F) guard rows, outputs in
sentinel-filled buffers with a padded pitch.  A negative control shows the comparison sees one wrong k-block scale and
one wrong channel shift.

Exhaustive quantisers: ``quantize_e4m3`` on all 65 536 bf16 bit patterns at four scales, ``quantize_e4m3_blocks`` on
every finite bf16 pattern (its behaviour on NaN and infinity is undefined and not tested), against the torch references.

Rejections: the per-tensor entries raise RuntimeError in the binding, before any launch, for host scalars, wrong
epilogue vectors, operands on other devices, K % 16 != 0 and misaligned operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

from edl_b200 import ops  # noqa: E402
from edl_b200.ops import fp8  # noqa: E402
from f64_bounds import guarded  # noqa: E402

DEV = torch.device("cuda", 0)
E4M3_NAN = 0x7F
NUM_SMS = 132


def _bits(t):
    """Bits of a float tensor with -0 and +0 identified (the sign of an exact zero sum is not specified)."""
    return (t.float() + 0.0).view(torch.int32)


def _e4m3_operand(rows, k, gen, max_nnz=None):
    """e4m3 bytes [rows, k] with values in {0, +-1, +-2}; with ``max_nnz``, at most that many nonzeros per row, the
    last 16 columns (the K-tail MMA, the tail block when K % 128 != 0) among them on purpose."""
    val = torch.randint(1, 3, (rows, k), generator=gen).float() * (torch.randint(0, 2, (rows, k), generator=gen) * 2 - 1)
    if max_nnz is None:
        keep = torch.rand(rows, k, generator=gen) < 0.6
    else:
        keep = torch.rand(rows, k, generator=gen) < min(1.0, 0.8 * max_nnz / k)
        keep[:, -16:] |= torch.rand(rows, 16, generator=gen) < 0.5
        keep &= keep.flip(1).cumsum(1).flip(1) <= max_nnz              # the last max_nnz nonzeros of each row
    return torch.where(keep, val, 0.0).to(torch.float8_e4m3fn).view(torch.uint8)


def _epilogue_vectors(n, gen, scale, shift):
    sc = (torch.rand(n, generator=gen) * 1.5 + 0.5) if scale else None                      # [0.5, 2)
    sh = (torch.randint(-2 ** 14 + 1, 2 ** 14, (n,), generator=gen).float() * 2.0 ** -10) if shift else None
    return sc, sh


def _exact_acc(a8, b8, sa=None, sb=None):
    """float64 [M, N]: the exact product of the e4m3 operands (per k-block scaled by sa[b, m] * sb[n // 128, b])."""
    a = a8.view(torch.float8_e4m3fn).float()
    b = b8.view(torch.float8_e4m3fn).float()
    if sa is None:
        return (a @ b.t()).double()                                  # integer sums below 2^10: exact in fp32
    n, k = b.shape[0], a.shape[1]
    sbn = sb.double().repeat_interleave(128, 0)[:n]
    acc = torch.zeros(a.shape[0], n, dtype=torch.float64, device=a.device)
    for i in range(-(-k // 128)):
        kk = slice(i * 128, min(k, (i + 1) * 128))
        acc += (a[:, kk] @ b[:, kk].t()).double() * sa[i].double()[:, None] * sbn[:, i][None, :]
    return acc


def _expected(acc, sc, sh, relu, add=None):
    v = acc
    if sc is not None:
        v = v * sc.double()
    if sh is not None:
        v = v + sh.double()
    v = v.float()                                                    # the epilogue's fma rounds once
    if add is not None:
        v = (v.double() + add.double()).float()
    if relu:
        v = v.clamp_min(0)
    return v.bfloat16()


def _setup(m, n, k, seed, block, scale, shift):
    gen = torch.Generator().manual_seed(seed)
    a8 = _e4m3_operand(m, k, gen, max_nnz=256)
    b8 = _e4m3_operand(n, k, gen)
    b8[n // 2] = 0                                  # a zero weight row: that column is col_shift alone
    sc, sh = _epilogue_vectors(n, gen, scale, shift)
    if sh is not None:
        sh[n // 2] = 5 * 2.0 ** -10
    kb = -(-k // 128)
    sa = sb = None
    if block:
        sa = (2.0 ** torch.randint(-3, 4, (kb, m), generator=gen)).float()
        sb = (2.0 ** torch.randint(-3, 4, (-(-n // 128), kb), generator=gen)).float()
    ag = guarded((m, k), pad_rows=2, pad_cols=16, fill=E4M3_NAN, dtype=torch.uint8, device=DEV, values=a8.to(DEV))
    bg = guarded((n, k), pad_rows=2, pad_cols=16, fill=E4M3_NAN, dtype=torch.uint8, device=DEV, values=b8.to(DEV))
    dev = (lambda t: None if t is None else t.to(DEV))
    return ag.t, bg.t, dev(sa), dev(sb), dev(sc), dev(sh), gen


def _negative_controls(out, acc_fn, a8, b8, sa, sb, sc, sh, relu, add=None):
    """The expectation built with one k-block scale doubled, or one channel's shift moved by 2^-10, differs from the
    kernel's output: the comparison would see either mistake."""
    n = b8.shape[0]
    if sa is not None:
        # the row whose last (tail) k-block moves some output furthest relative to its size, where the ReLU keeps it
        a = a8.view(torch.float8_e4m3fn).float()
        b = b8.view(torch.float8_e4m3fn).float()
        kb = sa.shape[0]
        kk = slice((kb - 1) * 128, a8.shape[1])
        delta = (a[:, kk] @ b[:, kk].t()).double() * sa[kb - 1].double()[:, None] * \
            sb.double().repeat_interleave(128, 0)[:n, kb - 1][None, :]
        v = acc_fn(sa, sb)
        if sc is not None:
            delta, v = delta * sc.double(), v * sc.double()
        if sh is not None:
            v = v + sh.double()
        score = delta.abs() / (v.abs() + delta.abs() + 2.0 ** -10)
        if relu:
            score = score * ((v > 0) | (v + delta > 0))
        m = int(score.amax(1).argmax())
        wrong = sa.clone()
        wrong[kb - 1, m] *= 2
        assert not torch.equal(_bits(out), _bits(_expected(acc_fn(wrong, sb), sc, sh, relu, add))), \
            "the check does not see a doubled k-block scale"
    if sh is not None:
        wrong = sh.clone()
        wrong[n // 2] += 2.0 ** -10
        assert not torch.equal(_bits(out), _bits(_expected(acc_fn(sa, sb), sc, wrong, relu, add))), \
            "the check does not see a channel's shift moved by 2^-10"


def _first_difference(out, want):
    bad = _bits(out) != _bits(want)
    i, j = bad.nonzero()[0].tolist()
    return "%d of %d elements differ, first at (%d, %d): got %r, want %r" % (
        int(bad.sum()), bad.numel(), i, j, float(out[i, j]), float(want[i, j]))


# M in {1, 127, 129, 128 * 132 + 1}, N in {8, 64, 72, 200, 1000, 2048} (64- and 128-column tiles, N tails),
# K in {16, 112, 128, 144, 1040, 4096} (K below one block, a tail block, one accumulation over all of K)
CASES = [
    # m, n, k, relu, col_scale, col_shift
    (1, 8, 16, False, False, False),
    (127, 64, 112, True, True, True),
    (129, 72, 128, False, True, False),
    (129, 200, 144, True, False, True),
    (127, 1000, 1040, False, True, True),
    (1, 2048, 4096, True, True, True),
    (128 * 132 + 1, 72, 4096, False, False, True),
    (128 * 132 + 1, 2048, 144, True, True, True),
    (129, 8, 1040, True, True, True),
]


@pytest.mark.parametrize("block", [False, True], ids=["tensor", "block"])
@pytest.mark.parametrize("m,n,k,relu,scale,shift", CASES)
def test_fp8_gemm_exact_operands_bitwise(m, n, k, relu, scale, shift, block):
    a8, b8, sa, sb, sc, sh, _ = _setup(m, n, k, m * 31 + n * 7 + k, block, scale, shift)
    out = guarded((m, n), pad_rows=3, pad_cols=8, fill=7.0, device=DEV)
    if block:
        fp8.gemm_fp8_blockscaled(a8, sa, b8, sb, sc, sh, relu, out=out.t)
    else:
        fp8.gemm_fp8(a8, b8, sc, sh, relu, out=out.t)
    torch.cuda.synchronize()
    out.assert_untouched("fp8 GEMM output")
    acc_fn = (lambda s_a, s_b: _exact_acc(a8, b8, s_a, s_b))
    want = _expected(acc_fn(sa, sb), sc, sh, relu)
    assert torch.equal(_bits(out.t), _bits(want)), "%s fp8 GEMM %d x %d x %d: %s" % (
        "block" if block else "tensor", m, n, k, _first_difference(out.t, want))
    if sh is not None:
        assert float(out.t[0, n // 2]) == 5 * 2.0 ** -10         # the zero weight row's column: col_shift alone
    _negative_controls(out.t, acc_fn, a8, b8, sa, sb, sc, sh, relu)


def _add_tile_n(m, n):
    """The residual epilogue's tile width, as gemm_fp8_blockscaled chooses it (csrc/gemm_fp8.cu)."""
    mt = -(-m // 128)
    w128 = 2 * (-(-(mt * -(-n // 128)) // NUM_SMS))
    w64 = -(-(mt * -(-n // 64)) // NUM_SMS)
    return 64 if (n <= 64 or w64 < w128) else 128


@pytest.mark.parametrize("m,n,k,relu,tile", [(127, 200, 144, True, 64), (1, 64, 4096, False, 64),
                                              (2330, 768, 1040, True, 128), (129 * 64 + 63, 256, 112, False, 128)])
def test_fp8_gemm_residual_epilogue_exact_operands_bitwise(m, n, k, relu, tile):
    assert _add_tile_n(m, n) == tile
    a8, b8, sa, sb, sc, sh, gen = _setup(m, n, k, m + n + k, True, True, True)
    addv = (torch.randn(m, n, generator=gen) * 4).bfloat16()
    addv[:, n // 2] = 0                             # the zero weight row's column stays col_shift alone
    add = guarded((m, n), pad_rows=1, pad_cols=8, device=DEV, values=addv.to(DEV))       # NaN around the addend
    out = guarded((m, n), pad_rows=3, pad_cols=8, fill=7.0, device=DEV)
    assert fp8.gemm_fp8_blockscaled_supported(a8, sa, b8, sb, add.t)
    ops.reset_fallbacks()
    fp8.gemm_fp8_blockscaled(a8, sa, b8, sb, sc, sh, relu, out=out.t, add=add.t)
    torch.cuda.synchronize()
    assert ops.fallbacks() == {}, ops.fallbacks()
    out.assert_untouched("fp8 residual epilogue output")
    acc_fn = (lambda s_a, s_b: _exact_acc(a8, b8, s_a, s_b))
    want = _expected(acc_fn(sa, sb), sc, sh, relu, add.t)
    assert torch.equal(_bits(out.t), _bits(want)), "fp8 residual epilogue %d x %d x %d (%d-column tiles): %s" % (
        m, n, k, tile, _first_difference(out.t, want))
    _negative_controls(out.t, acc_fn, a8, b8, sa, sb, sc, sh, relu, add.t)


# ------------------------------------------------------------------------------------------------------- quantisers
def _all_bf16():
    return torch.arange(-2 ** 15, 2 ** 15, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)


def _tensor_reference(x, scale):
    """``(x / scale).clamp(+-448)`` cast to e4m3 (the CPU path of ``quantize_e4m3``), on the CPU."""
    return (x.float() / scale).clamp(-fp8.E4M3_MAX, fp8.E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** -7, 0.37, 3.1e-3])
def test_quantize_e4m3_every_bf16_pattern(scale):
    x = _all_bf16()
    s = torch.tensor([scale], dtype=torch.float32)
    q = fp8.quantize_e4m3(x.to(DEV), s.to(DEV)).cpu()
    fin = torch.isfinite(x.float())
    want = _tensor_reference(x, s)
    bad = fin & (q != want)
    assert not bad.any(), "%d finite patterns differ, first x = %r: got 0x%02x, want 0x%02x" % (
        int(bad.sum()), float(x[bad][0]), int(q[bad][0]), int(want[bad][0]))
    nan = torch.isnan(x.float())
    assert ((q[nan] & 0x7F) == 0x7F).all(), "NaN must give a NaN byte"
    inf = torch.isinf(x.float())
    assert torch.equal(q[inf].view(torch.float8_e4m3fn).float(), x[inf].float().sign() * fp8.E4M3_MAX)

    # amax over the finite patterns, at lengths that exercise the 8-wide loop and the tail loop
    gen = torch.Generator().manual_seed(int(scale * 1e6))
    finite = x[fin][torch.randperm(int(fin.sum()), generator=gen)]
    top = finite[finite.float().abs().argmax()]
    for n in (1, 7, 8, 9, 65539):
        xs = (finite.repeat(2)[:n] if n > finite.numel() else finite[:n]).clone()
        xs[xs.float().abs() == top.float().abs()] = 0
        # the window's largest |x| once, in the tail loop's elements when n % 8 != 0 (else in the 8-wide loop)
        xs[n - 1 if n % 8 else n // 2] = top
        amax = torch.zeros(1, device=DEV)
        q = fp8.quantize_e4m3(xs.to(DEV), s.to(DEV), amax).cpu()
        assert torch.equal(q, _tensor_reference(xs, s)), n
        assert float(amax) == float(top.float().abs()), (n, float(amax))


def test_quantize_e4m3_misaligned_input_is_copied():
    x = (torch.randn(1001) * 3).bfloat16().to(DEV)
    buf = torch.zeros(1001 + 8, dtype=torch.bfloat16, device=DEV)
    view = buf[1:1002]
    view.copy_(x)
    assert view.is_contiguous() and view.data_ptr() % 16 != 0
    s = torch.tensor([0.01], device=DEV)
    assert torch.equal(fp8.quantize_e4m3(view, s), fp8.quantize_e4m3(x, s))


def _finite_bf16_rows(k, gen):
    x = _all_bf16()
    fin = x[torch.isfinite(x.float())]
    fin = fin[torch.randperm(fin.numel(), generator=gen)]
    rows = -(-fin.numel() // k)
    out = torch.zeros(rows * k, dtype=torch.bfloat16)
    out[:fin.numel()] = fin
    return out.view(rows, k)


@pytest.mark.parametrize("k", [8, 136, 1024])
def test_quantize_e4m3_blocks_every_finite_pattern(k):
    gen = torch.Generator().manual_seed(k)
    x = _finite_bf16_rows(k, gen)
    sub = _all_bf16()[1:128]                              # the positive bf16 subnormals 0x0001 .. 0x007f
    top = torch.tensor([0x7F7F], dtype=torch.int16).view(torch.bfloat16)             # the largest finite bf16
    extra = torch.zeros(4, k, dtype=torch.bfloat16)
    w = min(k, 128)
    extra[0, :w] = sub[torch.randint(0, 127, (w,), generator=gen)]                    # a block of subnormals only
    extra[1, :w] = -extra[0, :w]
    extra[2, :w] = sub[:1].expand(w)                      # only the smallest subnormal
    extra[3, :w] = torch.randn(w, generator=gen).bfloat16()
    extra[3, w // 2] = top
    extra[3, w // 3] = -top
    x = torch.cat([x, extra])
    q, sa = fp8.quantize_e4m3_blocks(x.to(DEV))
    q_ref, sa_ref = fp8.quantize_e4m3_blocks_reference(x)
    assert torch.equal(sa.cpu().view(torch.int32), sa_ref.view(torch.int32)), "block scales differ"
    bad = q.cpu() != q_ref
    assert not bad.any(), "%d bytes differ, first at %s" % (int(bad.sum()), bad.nonzero()[0].tolist())
    assert (sa_ref[0, -4:-2] > 0).all() and (sa_ref[0, -4:-2] < 2.0 ** -126).all()    # subnormal block scales


# ------------------------------------------------------------------------------------------------------- rejections
def test_per_tensor_entries_reject_bad_input():
    nat = ops.native()
    a8, _ = fp8.quantize_e4m3_blocks(torch.randn(64, 256, device=DEV).bfloat16())
    b8, _ = fp8.quantize_e4m3_blocks(torch.randn(128, 256, device=DEV).bfloat16())
    out = torch.empty(64, 128, device=DEV, dtype=torch.bfloat16)
    ones = torch.ones(128, device=DEV)
    # only the binding's own checks reject the first case, and a binding without them would read it in bounds: the test
    # stops there before any case that would not be read in bounds
    for cs, sh, match in ((ones.double(), None, "col_scale"), (ones.cpu(), None, "col_scale"),
                          (None, ones.cpu(), "col_shift"), (ones[:64], None, "col_scale"),
                          (None, ones.bfloat16(), "col_shift")):
        with pytest.raises(RuntimeError, match=match):
            nat.gemm_fp8(a8, b8, out, cs, sh, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        nat.gemm_fp8(a8, b8.cpu(), out, None, None, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        nat.gemm_fp8(a8, b8, out.cpu(), None, None, False)
    if torch.cuda.device_count() > 1:
        with pytest.raises(RuntimeError, match="different devices"):
            nat.gemm_fp8(a8, b8.to("cuda:1"), out, None, None, False)
    with pytest.raises(RuntimeError, match="16-byte"):
        nat.gemm_fp8(a8[:, :72], b8[:, :72], out, None, None, False)             # K % 16 != 0
    abuf = torch.zeros(64, 272, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        nat.gemm_fp8(abuf[:, 1:257], b8, out, None, None, False)                  # misaligned A
    bbuf = torch.zeros(128, 272, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        nat.gemm_fp8(a8, bbuf[:, 8:264], out, None, None, False)                  # misaligned B
    dbuf = torch.zeros(64 * 136 + 8, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        nat.gemm_fp8(a8, b8, dbuf[1:1 + 64 * 136].view(64, 136)[:, :128], None, None, False)        # misaligned D
    with pytest.raises(RuntimeError, match="16-byte aligned rows"):
        nat.gemm_fp8(a8, b8, dbuf[:64 * 130].view(64, 130)[:, :128], None, None, False)         # D pitch 130

    x = torch.randn(4096, device=DEV).bfloat16()
    q = torch.empty(4096, dtype=torch.uint8, device=DEV)
    s = torch.ones(1, device=DEV)
    # first a case only the amax check rejects: without it the kernel would write the first 4 bytes of this buffer
    with pytest.raises(RuntimeError, match="amax"):
        nat.quantize_e4m3(x, q, s, torch.zeros(1, device=DEV, dtype=torch.float64))
    with pytest.raises(RuntimeError, match="scale"):
        nat.quantize_e4m3(x, q, s.double(), None)
    with pytest.raises(RuntimeError, match="scale"):
        nat.quantize_e4m3(x, q, s.cpu(), None)                                     # host scale
    with pytest.raises(RuntimeError, match="amax"):
        nat.quantize_e4m3(x, q, s, torch.zeros(1))                                 # host amax
    xbuf = torch.zeros(4096 + 8, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="x must be 16-byte aligned"):
        nat.quantize_e4m3(xbuf[1:4097], q, s, None)                                # misaligned x
    qbuf = torch.zeros(4096 + 16, dtype=torch.uint8, device=DEV)
    with pytest.raises(RuntimeError, match="q must be 8-byte aligned"):
        nat.quantize_e4m3(x, qbuf[4:4100], s, None)                                # misaligned q
    with pytest.raises(RuntimeError, match="q must be"):
        nat.quantize_e4m3(x, q[:4095], s, None)
    with pytest.raises(RuntimeError, match="q must be"):
        nat.quantize_e4m3(x, q.cpu(), s, None)
