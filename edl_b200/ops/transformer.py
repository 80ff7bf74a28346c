"""Front-ends of the Transformer encoder kernels (csrc/attention.cu, csrc/layernorm.cu) and the GELU GEMM epilogue:
the inference path of the ERNIE / BERT sequence teacher (models/ernie.py).

Dispatch rule of the package: CPU tensors run the small float32 reference implementations below; on CUDA a shape a
kernel cannot take (head dim other than 64, sequences longer than 512, a hidden size above 1024 or not a multiple of 8)
runs the same reference math on the library through ``count_fallback``.

``layer_norm_e4m3`` and ``embedding_layernorm_e4m3`` also return the block-scaled e4m3 copy of their bf16 output
(``ops.fp8.quantize_e4m3_blocks``), written by the same kernel, for the FP8 teacher's next GEMM."""
from __future__ import annotations

import torch


def _count(reason):
    from . import count_fallback

    count_fallback(reason)


# ---------------------------------------------------------------------------------------------------------- attention
def attention_reference(qkv, mask, batch, seq_len, heads, head_dim=64):
    """Float32 math of ``attention``: softmax(Q K^T / sqrt(head_dim) with masked keys at -inf) V; a query row without a
    valid key is 0.  Returns [B * L, H * head_dim] in qkv's dtype."""
    x = qkv.float().view(batch, seq_len, 3, heads, head_dim)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))           # [B, H, L, d]
    s = (q @ k.transpose(-1, -2)) / head_dim ** 0.5
    if mask is not None:
        keep = (mask.view(batch, 1, 1, seq_len) != 0)
        s = s.masked_fill(~keep, float("-inf"))
    mx = s.amax(-1, keepdim=True)
    p = torch.exp(s - torch.where(torch.isinf(mx), torch.zeros_like(mx), mx))
    den = p.sum(-1, keepdim=True)
    o = (p @ v) / torch.where(den > 0, den, torch.ones_like(den))
    return o.transpose(1, 2).reshape(batch * seq_len, heads * head_dim).to(qkv.dtype)


def attention_supported(qkv, batch, seq_len, heads, head_dim=64) -> bool:
    from . import native

    return (qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.is_contiguous()
            and qkv.data_ptr() % 16 == 0 and tuple(qkv.shape) == (batch * seq_len, 3 * heads * head_dim)
            and native().attention_supported(batch, seq_len, heads, head_dim))


def attention(qkv, mask, batch, seq_len, heads, head_dim=64, out=None):
    """Masked multi-head self-attention (inference).  ``qkv`` [B * L, 3 * H * head_dim] is the QKV projection's output
    (column blocks Q | K | V, heads inside each); ``mask`` [B, L] (nonzero = attend; any pattern) or None.  Returns
    O [B * L, H * head_dim], the output projection's input."""
    from . import native, count_launch

    if not qkv.is_cuda:
        return attention_reference(qkv, mask, batch, seq_len, heads, head_dim)
    if not attention_supported(qkv, batch, seq_len, heads, head_dim):
        _count("attention: no kernel for B %d, L %d, H %d, head dim %d (%s): float32 math on the library"
               % (batch, seq_len, heads, head_dim, qkv.dtype))
        return attention_reference(qkv, mask, batch, seq_len, heads, head_dim)
    if out is None:
        out = torch.empty((batch * seq_len, heads * head_dim), device=qkv.device, dtype=torch.bfloat16)
    m = None
    if mask is not None:
        m = mask if (mask.dtype == torch.uint8 and mask.is_contiguous()) else (mask != 0).to(torch.uint8).contiguous()
    native().attention_fwd(qkv, m, out, batch, seq_len, heads)
    count_launch()
    return out


# ----------------------------------------------------------------------------------------- variable-length attention
def attention_varlen_reference(qkv, cu_seqlens, max_len, heads, key_mask=None):
    """Float32 math of ``attention_varlen``: ``attention_reference`` on each packed sequence.  Rows outside every
    sequence are 0 (the kernel does not write them)."""
    d = qkv.shape[1] // (3 * heads)
    cu = [int(v) for v in cu_seqlens.tolist()]
    out = torch.zeros((qkv.shape[0], heads * d), device=qkv.device, dtype=qkv.dtype)
    for s, e in zip(cu[:-1], cu[1:]):
        if e > s:
            m = None if key_mask is None else key_mask[s:e].view(1, e - s)
            out[s:e] = attention_reference(qkv[s:e], m, 1, e - s, heads, d)
    return out


def attention_varlen_supported(qkv, cu_seqlens, max_len, heads) -> bool:
    from . import native

    return (qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.is_contiguous()
            and qkv.data_ptr() % 16 == 0 and qkv.shape[1] % (3 * heads) == 0
            and cu_seqlens.is_cuda and cu_seqlens.dim() == 1 and cu_seqlens.numel() >= 2
            and native().attention_varlen_supported(qkv.shape[0], cu_seqlens.numel() - 1, int(max_len), heads,
                                                    qkv.shape[1] // (3 * heads)))


def attention_varlen(qkv, cu_seqlens, max_len, heads, key_mask=None, out=None):
    """Masked multi-head self-attention over sequences packed back to back (inference).  ``qkv`` [T, 3 * H * 64] is the
    QKV projection's output on the packed tokens; sequence b is rows [cu_seqlens[b], cu_seqlens[b + 1]) (int32 [B + 1],
    offset 0, non-decreasing, lengths 1..512); ``max_len`` (host int) is at least the longest length; ``key_mask``
    [T] (nonzero = attend) or None.  Returns O [T, H * 64].  Per sequence this is ``attention`` with L = its length,
    and its output depends on its own rows only.

    ``cu_seqlens`` is not read back to the host, so the call can be captured in a CUDA graph; ``pack_sequences``
    (models/ernie.py) validates the offsets where they are made."""
    from . import native, count_launch

    if not qkv.is_cuda:
        return attention_varlen_reference(qkv, cu_seqlens, max_len, heads, key_mask)
    if not attention_varlen_supported(qkv, cu_seqlens, max_len, heads):
        _count("attention_varlen: no kernel for T %d, B %d, max_len %d, H %d, width %d (%s): float32 math on the "
               "library" % (qkv.shape[0], cu_seqlens.numel() - 1, max_len, heads, qkv.shape[-1], qkv.dtype))
        return attention_varlen_reference(qkv, cu_seqlens, max_len, heads, key_mask)
    b = cu_seqlens.numel() - 1
    if out is None:
        out = torch.empty((qkv.shape[0], qkv.shape[1] // 3), device=qkv.device, dtype=torch.bfloat16)
    cu = cu_seqlens if (cu_seqlens.dtype == torch.int32 and cu_seqlens.is_contiguous()) else \
        cu_seqlens.to(torch.int32).contiguous()
    km = None
    if key_mask is not None:
        km = key_mask if (key_mask.dtype == torch.uint8 and key_mask.is_contiguous()) else \
            (key_mask != 0).to(torch.uint8).contiguous()
    maps = torch.empty(b * 256, device=qkv.device, dtype=torch.uint8)        # two 128-byte tensor maps per sequence
    native().attention_varlen_fwd(qkv, cu, km, out, maps, int(max_len), heads)
    count_launch(2)
    return out


# ---------------------------------------------------------------------------------------------------------- LayerNorm
def layer_norm_reference(x, gamma, beta, eps):
    xf = x.float()
    mean = xf.mean(-1, keepdim=True)
    var = (xf - mean).square().mean(-1, keepdim=True)
    return ((xf - mean) * torch.rsqrt(var + eps) * gamma.float() + beta.float()).to(x.dtype)


def layer_norm_supported(x) -> bool:
    from . import native

    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.is_contiguous() and x.data_ptr() % 16 == 0
            and native().layernorm_supported(x.shape[1]))


def layer_norm(x, gamma, beta, eps=1e-12, out=None):
    """LayerNorm over the last dimension of ``x`` [rows, C] with fp32 ``gamma`` / ``beta`` and fp32 statistics."""
    from . import native, count_launch

    if not x.is_cuda:
        return layer_norm_reference(x, gamma, beta, eps)
    if not layer_norm_supported(x):
        _count("layer_norm: no kernel for %s %s: float32 math on the library" % (tuple(x.shape), x.dtype))
        return layer_norm_reference(x, gamma, beta, eps)
    if out is None:
        out = torch.empty_like(x)
    native().layernorm_fwd(x, gamma.float().contiguous(), beta.float().contiguous(), out, float(eps))
    count_launch()
    return out


# ------------------------------------------------------------------------------------------- embedding + LayerNorm
def _check_ids(ids, n, what):
    if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= n):
        raise IndexError("embedding_layernorm: %s out of range [0, %d): min %d, max %d"
                         % (what, n, int(ids.min()), int(ids.max())))


def embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps):
    for t, tab, what in ((ids, word, "input id"), (pos_ids, pos, "position id"), (seg_ids, seg, "segment id")):
        _check_ids(t, tab.shape[0], what)
    x = word.float()[ids.reshape(-1)] + pos.float()[pos_ids.reshape(-1)] + seg.float()[seg_ids.reshape(-1)]
    return layer_norm_reference(x, gamma, beta, eps).to(word.dtype)


def embedding_layernorm_supported(word, pos, seg) -> bool:
    from . import native

    c = word.shape[1]
    return (all(t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.is_contiguous() and t.shape[1] == c
                and t.data_ptr() % 16 == 0 for t in (word, pos, seg))
            and native().layernorm_supported(c))


def embedding_layernorm(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps=1e-12, out=None):
    """LayerNorm(word[ids] + pos[pos_ids] + seg[seg_ids]) -> [ids.numel(), C], summed and normalised in fp32.

    Out-of-range ids raise IndexError.  On CUDA the kernel never reads outside a table; it raises a device flag that is
    checked after the launch, except while a CUDA graph is being captured (a replay cannot raise: such a row is the
    LayerNorm of the embeddings whose ids are in range)."""
    from . import native, count_launch

    if not word.is_cuda:
        return embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps)
    if not embedding_layernorm_supported(word, pos, seg):
        _count("embedding_layernorm: no kernel for width %d %s: float32 math on the library" % (word.shape[1], word.dtype))
        return embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps)
    rows = ids.numel()
    if out is None:
        out = torch.empty((rows, word.shape[1]), device=word.device, dtype=torch.bfloat16)
    err = torch.zeros(1, dtype=torch.int32, device=word.device)
    ids, pos_ids, seg_ids = (t.reshape(-1).to(word.device, torch.int64).contiguous() for t in (ids, pos_ids, seg_ids))
    native().embedding_layernorm_fwd(ids, pos_ids, seg_ids, word, pos, seg, gamma.float().contiguous(),
                                     beta.float().contiguous(), out, float(eps), err)
    count_launch()
    if not torch.cuda.is_current_stream_capturing() and int(err.item()) != 0:
        for t, tab, what in ((ids, word, "input id"), (pos_ids, pos, "position id"), (seg_ids, seg, "segment id")):
            _check_ids(t, tab.shape[0], what)
    return out


# ------------------------------------------------------------------------------------- LayerNorm with e4m3 output
def _quant_out(y):
    from .fp8 import BLOCK

    rows, c = y.shape
    return (torch.empty((rows, c), dtype=torch.uint8, device=y.device),
            torch.empty((-(-c // BLOCK), rows), dtype=torch.float32, device=y.device))


def layer_norm_e4m3_supported(x) -> bool:
    return layer_norm_supported(x)


def layer_norm_e4m3(x, gamma, beta, eps=1e-12):
    """``layer_norm`` that also quantises its output for a block-scaled FP8 GEMM: returns (y bf16 [rows, C],
    q uint8 e4m3 [rows, C], sa fp32 [ceil(C/128), rows]) with (q, sa) bit for bit ``quantize_e4m3_blocks(y)``.
    On CPU (and for a shape the kernel cannot take) it is exactly that composition of the references."""
    from . import native, count_launch
    from .fp8 import quantize_e4m3_blocks_reference

    if x.is_cuda and layer_norm_e4m3_supported(x):
        y = torch.empty_like(x)
        q, sa = _quant_out(y)
        native().layernorm_e4m3_fwd(x, gamma.float().contiguous(), beta.float().contiguous(), y, q, sa, float(eps))
        count_launch()
        return y, q, sa
    if x.is_cuda:
        _count("layer_norm_e4m3: no kernel for %s %s: float32 math on the library" % (tuple(x.shape), x.dtype))
    y = layer_norm_reference(x, gamma, beta, eps)
    return (y,) + quantize_e4m3_blocks_reference(y)


def embedding_layernorm_e4m3_supported(word, pos, seg) -> bool:
    return embedding_layernorm_supported(word, pos, seg)


def embedding_layernorm_e4m3(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps=1e-12):
    """``embedding_layernorm`` that also returns the block-scaled e4m3 copy of its output: (y, q, sa) as in
    ``layer_norm_e4m3``.  Out-of-range ids are handled as in ``embedding_layernorm`` (checked after the launch except
    under CUDA-graph capture)."""
    from . import native, count_launch
    from .fp8 import quantize_e4m3_blocks_reference

    if word.is_cuda and embedding_layernorm_e4m3_supported(word, pos, seg):
        rows = ids.numel()
        y = torch.empty((rows, word.shape[1]), device=word.device, dtype=torch.bfloat16)
        q, sa = _quant_out(y)
        err = torch.zeros(1, dtype=torch.int32, device=word.device)
        ids, pos_ids, seg_ids = (t.reshape(-1).to(word.device, torch.int64).contiguous() for t in (ids, pos_ids, seg_ids))
        native().embedding_layernorm_e4m3_fwd(ids, pos_ids, seg_ids, word, pos, seg, gamma.float().contiguous(),
                                              beta.float().contiguous(), y, q, sa, float(eps), err)
        count_launch()
        if not torch.cuda.is_current_stream_capturing() and int(err.item()) != 0:
            for t, tab, what in ((ids, word, "input id"), (pos_ids, pos, "position id"), (seg_ids, seg, "segment id")):
                _check_ids(t, tab.shape[0], what)
        return y, q, sa
    if word.is_cuda:
        _count("embedding_layernorm_e4m3: no kernel for width %d %s: float32 math on the library"
               % (word.shape[1], word.dtype))
    y = embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps)
    return (y,) + quantize_e4m3_blocks_reference(y)
