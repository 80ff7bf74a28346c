"""FP8 (e4m3) inference path for the teacher (csrc/gemm_fp8.cu).  Two scalings:

* per-tensor: activation scales from a calibration pass ("delayed scaling"), per-output-channel weight
  scales, dequantisation folded into the GEMM epilogue together with the folded BatchNorm scale / shift
  and the ReLU (``quantize_e4m3``, ``quantize_weight_rows``, ``gemm_fp8``);
* block-scaled: one fp32 scale per activation row and 128-element K block, computed from that block's own
  max|x| when the layer runs, and one per 128x128 weight block, applied per k-block inside the GEMM main
  loop -- no calibration pass and no host synchronisation (``quantize_e4m3_blocks``,
  ``quantize_weight_blocks``, ``gemm_fp8_blockscaled``).

For the sequence teacher's linear layers the block-scaled GEMM has two fused epilogues: a bf16 residual addend
(``gemm_fp8_blockscaled(..., add=x)``) and bias + erf-GELU quantised straight to the next GEMM's e4m3 operand and block
scales (``gemm_fp8_gelu_e4m3``).  Neither reads anything back to the host, so both can be captured in a CUDA graph.

The reference serves the teacher in fp32 through Paddle Serving (example/distill/resnet/scripts/
start_local_teacher.sh:24-30); SURVEY K12 asks for an fp8 wgmma path on Hopper."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

E4M3_MAX = 448.0
BLOCK = 128   # K block of the block-scaled mode (activations and weights), and N block of the weights


def quantize_weight_rows(w2: torch.Tensor):
    """w2 [N, K] float/bf16 -> (uint8 e4m3 bytes [N, K], fp32 scale [N])"""
    w = w2.float()
    scale = (w.abs().amax(1).clamp_min(1e-12) / E4M3_MAX)
    q = (w / scale[:, None]).to(torch.float8_e4m3fn).view(torch.uint8).contiguous()
    return q, scale


def quantize_e4m3(x: torch.Tensor, scale: torch.Tensor, amax: Optional[torch.Tensor] = None, out=None):
    """bf16 tensor -> e4m3 bytes with a per-tensor scale (device scalar); optionally tracks max|x|."""
    from . import native, count_launch

    x = x.contiguous()
    if x.is_cuda and x.data_ptr() % 16 != 0:
        x = x.clone()                       # the kernel reads 16-byte vectors: a fresh allocation is aligned
    q = out if out is not None else torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    if x.is_cuda:
        native().quantize_e4m3(x, q, scale, amax)
        count_launch()
    else:
        if amax is not None:
            amax.copy_(torch.maximum(amax, x.float().abs().max()))
        q.copy_((x.float() / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8))
    return q


def gemm_fp8(a8: torch.Tensor, b8: torch.Tensor, col_scale=None, col_shift=None, relu=False, out=None):
    """out bf16 [M, N] = relu?((a8 [M,K] @ b8 [N,K]^T) * col_scale + col_shift); a8 / b8 hold e4m3 bytes."""
    from . import native, count_launch

    m, n = a8.shape[0], b8.shape[0]
    if out is None:
        out = torch.empty((m, n), device=a8.device, dtype=torch.bfloat16)
    if a8.is_cuda:
        native().gemm_fp8(a8, b8, out, col_scale, col_shift, relu)
        count_launch()
        return out
    d = a8.view(torch.float8_e4m3fn).float() @ b8.view(torch.float8_e4m3fn).float().t()
    if col_scale is not None:
        d = d * col_scale
    if col_shift is not None:
        d = d + col_shift
    out.copy_(torch.relu(d) if relu else d)
    return out


# ---- block scaling -------------------------------------------------------------------------------------------
def _block_scale(amax: torch.Tensor) -> torch.Tensor:
    """s = amax / 448 in fp32 (an IEEE division, as in the kernel); 1 for an all-zero block.  The divisor is a
    tensor on purpose: torch turns division by a Python scalar into a multiplication by its reciprocal on CUDA."""
    return torch.where(amax > 0, amax / torch.full_like(amax, E4M3_MAX), torch.ones_like(amax))


def _to_e4m3_bytes(x: torch.Tensor) -> torch.Tensor:
    return x.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).view(torch.uint8)


def quantize_e4m3_blocks(x: torch.Tensor):
    """x bf16 [M, K] (last dim contiguous, any row pitch) -> (q uint8 e4m3 [M, K], sa fp32 [ceil(K/128), M]).

    For row m and K block b (the tail block is shorter): s = max|x| / 448 (1 when the block is all zero),
    sa[b, m] = s, q = sat(x / s).  K-block-major scales: one k-block's scales for 128 rows are contiguous."""
    from . import native, count_launch

    m, k = x.shape
    kb = -(-k // BLOCK)
    if x.is_cuda:
        q = torch.empty((m, k), dtype=torch.uint8, device=x.device)
        sa = torch.empty((kb, m), dtype=torch.float32, device=x.device)
        native().quantize_e4m3_blocks(x, q, sa)
        count_launch()
        return q, sa
    return quantize_e4m3_blocks_reference(x)


def quantize_e4m3_blocks_reference(x: torch.Tensor):
    """The math of ``quantize_e4m3_blocks`` in torch, on ``x``'s device (the CPU path and the fallbacks)."""
    m, k = x.shape
    kb = -(-k // BLOCK)
    xb = F.pad(x.float(), (0, kb * BLOCK - k)).view(m, kb, BLOCK)       # zero padding leaves max|x| unchanged
    s = _block_scale(xb.abs().amax(2))                                   # [M, KB]
    q = _to_e4m3_bytes(xb / s[:, :, None]).view(m, kb * BLOCK)[:, :k].contiguous()
    return q, s.t().contiguous()


def quantize_weight_blocks(w: torch.Tensor):
    """w [N, K] float/bf16 -> (uint8 e4m3 [N, K], sb fp32 [ceil(N/128), ceil(K/128)]), one scale per 128x128
    block with the same rule as ``quantize_e4m3_blocks``.  Runs once per layer, on the weight's device."""
    n, k = w.shape
    nb, kb = -(-n // BLOCK), -(-k // BLOCK)
    wb = F.pad(w.float(), (0, kb * BLOCK - k, 0, nb * BLOCK - n)).view(nb, BLOCK, kb, BLOCK)
    s = _block_scale(wb.abs().amax(dim=(1, 3)))                          # [NB, KB]
    q = _to_e4m3_bytes(wb / s[:, None, :, None]).view(nb * BLOCK, kb * BLOCK)[:n, :k].contiguous()
    return q, s.contiguous()


def _blockscaled_product(a8, sa, b8, sb):
    """fp32 [M, N] = sum_b (a8_b @ b8_b^T) * sa[b, m] * sb[n // 128, b], in torch on a8's device."""
    m, n, k = a8.shape[0], b8.shape[0], a8.shape[1]
    a = a8.view(torch.float8_e4m3fn).float()
    b = b8.view(torch.float8_e4m3fn).float()
    sb_n = sb.float().repeat_interleave(BLOCK, 0)[:n]                    # [N, KB]: the scale row of each output column
    d = torch.zeros((m, n), dtype=torch.float32, device=a8.device)
    for i in range(-(-k // BLOCK)):                                      # promote each k-block's partial product
        kk = slice(i * BLOCK, min(k, (i + 1) * BLOCK))
        d += (a[:, kk] @ b[:, kk].t()) * (sa[i].float()[:, None] * sb_n[:, i][None, :])
    return d


def _aligned(t, rows_mult=16):
    return t.is_cuda and t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % rows_mult == 0 and t.data_ptr() % 16 == 0


def gemm_fp8_blockscaled_supported(a8, sa, b8, sb, add=None) -> bool:
    """Whether ``gemm_fp8_blockscaled`` with ``add`` runs on the kernel: e4m3 operands with 16-byte aligned rows and
    K % 16 == 0, the scale layouts of ``quantize_e4m3_blocks`` / ``quantize_weight_blocks``, and a bf16 [M, N] addend
    with N % 8 == 0 and 16-byte aligned rows."""
    if not (a8.is_cuda and b8.is_cuda and a8.dim() == 2 and b8.dim() == 2 and a8.element_size() == 1
            and b8.element_size() == 1 and _aligned(a8) and _aligned(b8)):
        return False
    m, n, k = a8.shape[0], b8.shape[0], a8.shape[1]
    kb = -(-k // BLOCK)
    ok = (m > 0 and n > 0 and k > 0 and k % 16 == 0 and b8.shape[1] == k
          and sa.is_cuda and sa.dtype == torch.float32 and sa.is_contiguous() and tuple(sa.shape) == (kb, m)
          and sb.is_cuda and sb.dtype == torch.float32 and sb.is_contiguous() and tuple(sb.shape) == (-(-n // BLOCK), kb))
    if add is not None:
        ok = ok and (add.dtype == torch.bfloat16 and tuple(add.shape) == (m, n) and n % 8 == 0
                     and add.device == a8.device and _aligned(add, 8))
    return ok


def gemm_fp8_blockscaled(a8: torch.Tensor, sa: torch.Tensor, b8: torch.Tensor, sb: torch.Tensor, col_scale=None,
                         col_shift=None, relu=False, out=None, add=None):
    """out bf16 [M, N] = relu?((sum_b (a8_b @ b8_b^T) * sa[b, m] * sb[n // 128, b]) * col_scale + col_shift + add).

    a8 [M, K] / b8 [N, K] hold e4m3 bytes; b runs over the 128-element K blocks; sa [ceil(K/128), M] and
    sb [ceil(N/128), ceil(K/128)] come from ``quantize_e4m3_blocks`` / ``quantize_weight_blocks``.  ``add``: an optional
    bf16 [M, N] residual (any row pitch), added in the epilogue (the sequence teacher's out-projection and FFN2); on
    CUDA a shape ``gemm_fp8_blockscaled_supported`` rejects then runs the same math on the library through
    ``count_fallback``."""
    from . import native, count_launch, count_fallback

    m, n = a8.shape[0], b8.shape[0]
    if out is None:
        out = torch.empty((m, n), device=a8.device, dtype=torch.bfloat16)
    if a8.is_cuda and add is not None and not gemm_fp8_blockscaled_supported(a8, sa, b8, sb, add):
        count_fallback("gemm_fp8_blockscaled: no kernel for A %s, B %s, add %s: float32 math on the library"
                       % (tuple(a8.shape), tuple(b8.shape), tuple(add.shape)))
    elif a8.is_cuda:
        native().gemm_fp8_blockscaled(a8, sa, b8, sb, out, col_scale, col_shift, relu, add)
        count_launch()
        return out
    d = _blockscaled_product(a8, sa, b8, sb)
    if col_scale is not None:
        d = d * col_scale
    if col_shift is not None:
        d = d + col_shift
    if add is not None:
        d = d + add.float()
    out.copy_(torch.relu(d) if relu else d)
    return out


def gemm_fp8_gelu_e4m3_supported(a8, sa, b8, sb) -> bool:
    """Whether ``gemm_fp8_gelu_e4m3`` runs on the kernel: ``gemm_fp8_blockscaled_supported`` and N % 16 == 0."""
    return gemm_fp8_blockscaled_supported(a8, sa, b8, sb) and b8.shape[0] % 16 == 0


def gemm_fp8_gelu_e4m3(a8: torch.Tensor, sa: torch.Tensor, b8: torch.Tensor, sb: torch.Tensor, bias=None):
    """FFN1 of the sequence teacher, quantised for FFN2: g = bf16(gelu(sum_b (a8_b @ b8_b^T) * sa[b, m] *
    sb[n // 128, b] + bias)) (erf form), returned as ``quantize_e4m3_blocks(g)`` would: (q uint8 e4m3 [M, N],
    sa fp32 [ceil(N/128), M]).  The bf16 g is never stored.  ``bias``: fp32 [N] or None."""
    from . import native, count_launch, count_fallback

    m, n = a8.shape[0], b8.shape[0]
    if a8.is_cuda and gemm_fp8_gelu_e4m3_supported(a8, sa, b8, sb):
        q = torch.empty((m, n), dtype=torch.uint8, device=a8.device)
        sa_out = torch.empty((-(-n // BLOCK), m), dtype=torch.float32, device=a8.device)
        native().gemm_fp8_blockscaled_gelu_e4m3(a8, sa, b8, sb, q, sa_out,
                                                None if bias is None else bias.float().contiguous())
        count_launch()
        return q, sa_out
    if a8.is_cuda:
        count_fallback("gemm_fp8_gelu_e4m3: no kernel for A %s, B %s: float32 math on the library"
                       % (tuple(a8.shape), tuple(b8.shape)))
    d = _blockscaled_product(a8, sa, b8, sb)
    if bias is not None:
        d = d + bias.float()
    return quantize_e4m3_blocks_reference(F.gelu(d).to(torch.bfloat16))
