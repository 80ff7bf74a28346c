"""FP8 (e4m3) inference path for the teacher (csrc/gemm_fp8.cu).  Two scalings:

* per-tensor: activation scales from a calibration pass ("delayed scaling"), per-output-channel weight
  scales, dequantisation folded into the GEMM epilogue together with the folded BatchNorm scale / shift
  and the ReLU (``quantize_e4m3``, ``quantize_weight_rows``, ``gemm_fp8``);
* block-scaled: one fp32 scale per activation row and 128-element K block, computed from that block's own
  max|x| when the layer runs, and one per 128x128 weight block, applied per k-block inside the GEMM main
  loop -- no calibration pass and no host synchronisation (``quantize_e4m3_blocks``,
  ``quantize_weight_blocks``, ``gemm_fp8_blockscaled``).

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


def gemm_fp8_blockscaled(a8: torch.Tensor, sa: torch.Tensor, b8: torch.Tensor, sb: torch.Tensor, col_scale=None,
                         col_shift=None, relu=False, out=None):
    """out bf16 [M, N] = relu?((sum_b (a8_b @ b8_b^T) * sa[b, m] * sb[n // 128, b]) * col_scale + col_shift).

    a8 [M, K] / b8 [N, K] hold e4m3 bytes; b runs over the 128-element K blocks; sa [ceil(K/128), M] and
    sb [ceil(N/128), ceil(K/128)] come from ``quantize_e4m3_blocks`` / ``quantize_weight_blocks``."""
    from . import native, count_launch

    m, n, k = a8.shape[0], b8.shape[0], a8.shape[1]
    if out is None:
        out = torch.empty((m, n), device=a8.device, dtype=torch.bfloat16)
    if a8.is_cuda:
        native().gemm_fp8_blockscaled(a8, sa, b8, sb, out, col_scale, col_shift, relu)
        count_launch()
        return out
    a = a8.view(torch.float8_e4m3fn).float()
    b = b8.view(torch.float8_e4m3fn).float()
    sb_n = sb.float().repeat_interleave(BLOCK, 0)[:n]                    # [N, KB]: the scale row of each output column
    d = torch.zeros((m, n), dtype=torch.float32)
    for i in range(-(-k // BLOCK)):                                      # promote each k-block's partial product
        kk = slice(i * BLOCK, min(k, (i + 1) * BLOCK))
        d += (a[:, kk] @ b[:, kk].t()) * (sa[i].float()[:, None] * sb_n[:, i][None, :])
    if col_scale is not None:
        d = d * col_scale
    if col_shift is not None:
        d = d + col_shift
    out.copy_(torch.relu(d) if relu else d)
    return out
