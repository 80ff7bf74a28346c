"""Front-ends of the Transformer encoder kernels (csrc/attention.cu, csrc/layernorm.cu) and the GELU GEMM epilogue:
the inference path of the ERNIE / BERT sequence teacher (models/ernie.py).

Dispatch rule of the package: CPU tensors run the small float32 reference implementations below; on CUDA a shape a
kernel cannot take (head dim other than 32 or 64, sequences longer than 512, a hidden size above 1024 or not a
multiple of 8)
runs the same reference math on the library through ``count_fallback``.

``layer_norm_e4m3`` and ``embedding_layernorm_e4m3`` also return the block-scaled e4m3 copy of their bf16 output
(``ops.fp8.quantize_e4m3_blocks``), written by the same kernel, for the FP8 teacher's next GEMM.

Dropout (training): one mask definition for every kernel, the float32 fallback and the tests, see
``dropout_keep_reference``."""
from __future__ import annotations

import torch


def _count(reason):
    from . import count_fallback

    count_fallback(reason)


# ------------------------------------------------------------------------------------------------------------ dropout
# A dropout site draws one (seed, offset) pair from the default CUDA generator of its device, consuming 4 offset units
# (so torch.manual_seed governs the masks, and a CUDA graph draws fresh ones on every replay).  Element n of the site's
# flat index space is kept iff word n % 4 of Philox4x32-10 with key (seed_lo, seed_hi) and counter
# (floor(n / 4)_lo, floor(n / 4)_hi, offset_lo, offset_hi) is >= floor(p * 2^32); kept elements are scaled by
# fp32(1 / (1 - p)).  The kernels evaluate the same rule (csrc/philox.cuh).  On CPU the sites use F.dropout.
_M32 = 0xFFFFFFFF
_ATTN_MAX_LEN = 512            # kAttnMaxLen: the row stride of the packed attention-probability index
_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def _check_p(p):
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise ValueError("dropout probability must satisfy 0 <= p < 1, got %r" % p)
    return p


def _mulhilo(m, c):
    """(hi, lo) 32-bit words of the 64-bit product m * c (c int64 in [0, 2^32)) without leaving int64."""
    a, b = c * (m & 0xFFFF), c * (m >> 16)            # < 2^48 each
    return (b + (a >> 16)) >> 16, (a + ((b & 0xFFFF) << 16)) & _M32


def philox4x32_10(key, ctr):
    """Philox4x32-10 of int64 tensors holding 32-bit words: key (k0, k1), counter (c0, c1, c2, c3) -> four words."""
    k0, k1 = key
    c0, c1, c2, c3 = ctr
    for r in range(10):
        if r:
            k0, k1 = (k0 + _PHILOX_W[0]) & _M32, (k1 + _PHILOX_W[1]) & _M32
        hi0, lo0 = _mulhilo(_PHILOX_M[0], c0)
        hi1, lo1 = _mulhilo(_PHILOX_M[1], c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return c0, c1, c2, c3


def _keep(seed, offset, index, threshold):
    index = index.to(torch.int64)
    g = index >> 2
    w = lambda v: torch.full_like(index, v & _M32)   # noqa: E731
    words = philox4x32_10((w(seed), w(seed >> 32)), (g & _M32, g >> 32, w(offset), w(offset >> 32)))
    word = torch.stack(words, -1).gather(-1, (index & 3).unsqueeze(-1)).squeeze(-1)
    return word >= threshold


def dropout_keep_reference(seed, offset, index, p):
    """The keep mask (bool, index's shape and device) of a dropout site with generator state (seed, offset) at the flat
    element indices ``index`` (int64 tensor), in torch int64 arithmetic on any device.  The single host-side statement
    of the rule the kernels use; the scale of a kept element is ``fp32(1 / (1 - p))``.

    The flat index of each site: attention probability (b, h, i, j) at ((b H + h) L + i) L + j in the padded layout
    [B, L], and at ((b H + h) 512 + i) 512 + j for packed sequences (the fixed stride 512, the longest sequence the
    kernels take, keeps the sequences' index ranges disjoint whatever their lengths); a row-wise site (residual
    branches, embedding-LayerNorm output) at row * C + col, padded or packed rows alike; the pooled features at
    b * C + col."""
    p = _check_p(p)
    return _keep(int(seed), int(offset), index, int(p * 4294967296.0))


def _draw(device, p):
    """Draw one dropout site (p > 0) from the default CUDA generator of ``device``."""
    from . import native

    return native().dropout_draw(device.index if device.index is not None else torch.cuda.current_device(), p)


def _fallback_z(drop, shape, device, strides=None):
    """Z = keep * scale (float32, ``shape``) of a drawn site, element (k_0, k_1, ...) at the flat index
    sum_d k_d strides_d (by default the strides of a contiguous ``shape``): the kernels' mask for the float32 fallback.
    Needs the host values of the draw, so it cannot run under CUDA-graph capture."""
    if drop.captured:
        raise RuntimeError("dropout: the float32 fallback cannot be captured in a CUDA graph")
    index = torch.zeros((), dtype=torch.int64, device=device)
    for n, s in zip(shape, strides or torch.empty(shape, device="meta").stride()):
        index = index.unsqueeze(-1) + torch.arange(n, device=device) * s
    return _keep(drop.seed, drop.offset, index, drop.threshold).float() * drop.scale


def _site_z(t, p, shape, strides=None):
    """Z of a dropout site on the float32 reference path: None at p = 0, F.dropout's mask on CPU, the kernels' mask
    (one generator draw, flat indices as in ``_fallback_z``) on CUDA."""
    if p == 0.0:
        return None
    if not t.is_cuda:
        return torch.nn.functional.dropout(torch.ones(shape, dtype=torch.float32), p, True)
    return _fallback_z(_draw(t.device, p), shape, t.device, strides)


def _dropout_apply(x, drop):
    from . import native, count_launch

    y = torch.empty_like(x)
    native().dropout_fwd(x, y, drop)
    count_launch()
    return y


class _DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, drop):
        ctx.drop = drop
        return _dropout_apply(x, drop)

    @staticmethod
    def backward(ctx, dy):
        return _dropout_apply(dy.contiguous(), ctx.drop), None


def dropout(x, p, training=True):
    """Inverted dropout: zero each element with probability ``p`` and scale the others by 1 / (1 - p).  Identity when
    not ``training`` or at p = 0 (no generator draw).  On CUDA, bf16 runs dropout.cu with the package's mask over the
    flat index of ``x`` (one draw of 4 offset units); other dtypes take the same mask in float32 math through
    ``count_fallback``.  On CPU it is ``F.dropout``."""
    p = _check_p(p)
    if not training or p == 0.0:
        return x
    if not x.is_cuda:
        return torch.nn.functional.dropout(x, p, True)
    if x.dtype == torch.bfloat16:
        return _DropoutFn.apply(x.contiguous(), _draw(x.device, p))
    _count("dropout: no kernel for %s: float32 math on the library" % x.dtype)
    return (x.float() * _site_z(x, p, tuple(x.shape))).to(x.dtype)


# ---------------------------------------------------------------------------------------------------------- attention
def attention_reference(qkv, mask, batch, seq_len, heads, head_dim=64, drop_z=None):
    """Float32 math of ``attention``: softmax(Q K^T / sqrt(head_dim) with masked keys at -inf) V; a query row without a
    valid key is 0.  ``drop_z`` [B, H, L, L]: dropout (keep * scale) on the probabilities.  Returns [B * L, H * head_dim]
    in qkv's dtype."""
    x = qkv.float().view(batch, seq_len, 3, heads, head_dim)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))           # [B, H, L, d]
    s = (q @ k.transpose(-1, -2)) / head_dim ** 0.5
    if mask is not None:
        keep = (mask.view(batch, 1, 1, seq_len) != 0)
        s = s.masked_fill(~keep, float("-inf"))
    mx = s.amax(-1, keepdim=True)
    p = torch.exp(s - torch.where(torch.isinf(mx), torch.zeros_like(mx), mx))
    den = p.sum(-1, keepdim=True)
    if drop_z is not None:
        p = p * drop_z
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
    native().attention_fwd(qkv, _mask_u8(mask), out, batch, seq_len, heads, None, None)
    count_launch()
    return out


def _mask_u8(mask):
    if mask is None:
        return None
    return mask if (mask.dtype == torch.uint8 and mask.is_contiguous()) else (mask != 0).to(torch.uint8).contiguous()


def _cu_i32(cu_seqlens):
    return cu_seqlens if (cu_seqlens.dtype == torch.int32 and cu_seqlens.is_contiguous()) else \
        cu_seqlens.to(torch.int32).contiguous()


# ----------------------------------------------------------------------------------------- variable-length attention
def attention_varlen_reference(qkv, cu_seqlens, max_len, heads, key_mask=None, drop_z=None):
    """Float32 math of ``attention_varlen``: ``attention_reference`` on each packed sequence.  Rows outside every
    sequence are 0 (the kernel does not write them).  ``drop_z``: per sequence b a [1, H, len_b, len_b] dropout
    (keep * scale) on its probabilities, or None."""
    d = qkv.shape[1] // (3 * heads)
    cu = [int(v) for v in cu_seqlens.tolist()]
    out = torch.zeros((qkv.shape[0], heads * d), device=qkv.device, dtype=qkv.dtype)
    for b, (s, e) in enumerate(zip(cu[:-1], cu[1:])):
        if e > s:
            m = None if key_mask is None else key_mask[s:e].view(1, e - s)
            z = None if drop_z is None else drop_z[b]
            out[s:e] = attention_reference(qkv[s:e], m, 1, e - s, heads, d, z)
    return out


def attention_varlen_supported(qkv, cu_seqlens, max_len, heads) -> bool:
    from . import native

    return (qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.dim() == 2 and qkv.is_contiguous()
            and qkv.data_ptr() % 16 == 0 and qkv.shape[1] % (3 * heads) == 0
            and cu_seqlens.is_cuda and cu_seqlens.dim() == 1 and cu_seqlens.numel() >= 2
            and native().attention_varlen_supported(qkv.shape[0], cu_seqlens.numel() - 1, int(max_len), heads,
                                                    qkv.shape[1] // (3 * heads)))


def attention_varlen(qkv, cu_seqlens, max_len, heads, key_mask=None, out=None):
    """Masked multi-head self-attention over sequences packed back to back (inference).  ``qkv`` [T, 3 * H * D] is the
    QKV projection's output on the packed tokens (head dim D = qkv.shape[1] / 3H; the kernels take 32 and 64);
    sequence b is rows [cu_seqlens[b], cu_seqlens[b + 1]) (int32 [B + 1], offset 0, non-decreasing, lengths 1..512);
    ``max_len`` (host int) is at least the longest length; ``key_mask`` [T] (nonzero = attend) or None.  Returns
    O [T, H * D].  Per sequence this is ``attention`` with L = its length,
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
    maps = torch.empty(b * 256, device=qkv.device, dtype=torch.uint8)        # two 128-byte tensor maps per sequence
    native().attention_varlen_fwd(qkv, _cu_i32(cu_seqlens), _mask_u8(key_mask), out, maps, int(max_len), heads, None,
                                  None)
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
def _check_ids(ids, pos_ids, seg_ids, word, pos, seg):
    for t, tab, what in ((ids, word, "input id"), (pos_ids, pos, "position id"), (seg_ids, seg, "segment id")):
        n = tab.shape[0]
        if t.numel() and (int(t.min()) < 0 or int(t.max()) >= n):
            raise IndexError("embedding_layernorm: %s out of range [0, %d): min %d, max %d"
                             % (what, n, int(t.min()), int(t.max())))


def embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps):
    _check_ids(ids, pos_ids, seg_ids, word, pos, seg)
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
    if not word.is_cuda:
        return embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps)
    if not embedding_layernorm_supported(word, pos, seg):
        _count("embedding_layernorm: no kernel for width %d %s: float32 math on the library" % (word.shape[1], word.dtype))
        return embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps)
    return _embedding_layernorm_kernel(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps, out, None)


def _embedding_launch(launch, ids, pos_ids, seg_ids, word, pos, seg):
    """``launch(ids, pos_ids, seg_ids, err)``, an embedding-LayerNorm kernel, on the ids flattened to int64 on word's
    device.  The kernel never reads outside a table; it raises the device flag ``err``, checked after the launch except
    while a CUDA graph is being captured."""
    from . import count_launch

    err = torch.zeros(1, dtype=torch.int32, device=word.device)
    ids, pos_ids, seg_ids = (t.reshape(-1).to(word.device, torch.int64).contiguous() for t in (ids, pos_ids, seg_ids))
    launch(ids, pos_ids, seg_ids, err)
    count_launch()
    if not torch.cuda.is_current_stream_capturing() and int(err.item()) != 0:
        _check_ids(ids, pos_ids, seg_ids, word, pos, seg)


def _embedding_layernorm_kernel(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps, out, drop):
    from . import native

    if out is None:
        out = torch.empty((ids.numel(), word.shape[1]), device=word.device, dtype=torch.bfloat16)
    _embedding_launch(lambda i, p, s, err: native().embedding_layernorm_fwd(
        i, p, s, word, pos, seg, gamma.float().contiguous(), beta.float().contiguous(), out, float(eps), err, drop),
        ids, pos_ids, seg_ids, word, pos, seg)
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
    from . import native
    from .fp8 import quantize_e4m3_blocks_reference

    if word.is_cuda and embedding_layernorm_e4m3_supported(word, pos, seg):
        y = torch.empty((ids.numel(), word.shape[1]), device=word.device, dtype=torch.bfloat16)
        q, sa = _quant_out(y)
        _embedding_launch(lambda i, p, s, err: native().embedding_layernorm_e4m3_fwd(
            i, p, s, word, pos, seg, gamma.float().contiguous(), beta.float().contiguous(), y, q, sa, float(eps), err),
            ids, pos_ids, seg_ids, word, pos, seg)
        return y, q, sa
    if word.is_cuda:
        _count("embedding_layernorm_e4m3: no kernel for width %d %s: float32 math on the library"
               % (word.shape[1], word.dtype))
    y = embedding_layernorm_reference(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps)
    return (y,) + quantize_e4m3_blocks_reference(y)


# ------------------------------------------------------------------------------------------------------------ training
# The training path of the Transformer student (models/ernie.py ErnieStudent).  Each entry point below takes the float
# master parameters and casts the matrices to bf16 at every forward.  On CUDA the forward and backward run on the
# package's kernels (attention.cu / attention_bwd.cu, layernorm.cu, the persistent GEMM with its GELU epilogues); on CPU,
# and for shapes the kernels do not take (counted through ``count_fallback`` on CUDA), the float32 references run under
# torch autograd.  Dropout (the ``*_dropout`` / ``dropout_p`` arguments, default 0): the attention probabilities in the
# attention kernels, the two residual branches in the output-projection / FFN2 GEMM epilogues (D = x + Z o branch) and
# the embedding-LayerNorm output in its kernel; each backward regenerates its mask.  At p = 0 nothing is drawn and the
# p = 0 kernels run.  Nothing reads back to the host, so a whole training step can be captured in a CUDA graph.
def _needs_grad(*ts):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


def _bf16(t):
    return t if t.dtype == torch.bfloat16 else t.to(torch.bfloat16)


def _bias_grad(db, bias, sink):
    """A bias gradient the way ``_LinearFn`` delivers it: into the flat gradient bucket when the parameter has a sink
    (returns None to autograd), else returned in the parameter's dtype."""
    s, ready = sink
    if s is not None:
        s.add_(db)
        if ready is not None:
            ready()
        return None
    return db.to(bias.dtype)


def _wgrad_to(dy, x, w, sink):
    from .gemm import _wgrad

    g = _wgrad(dy, x, w.shape, *sink)
    return None if g is None else g.to(w.dtype)


def _weight_bias_grads(needs, sinks, *layers):
    """The gradients (weight, bias, weight, bias, ...) of linear layers y = x W^T + b given as (dy, x, W, b), each
    delivered by ``_wgrad_to`` / ``_bias_grad`` through its sink in ``sinks`` when its flag in ``needs`` is set."""
    g = []
    for i, (dy, x, w, b) in enumerate(layers):
        g.append(_wgrad_to(dy, x, w, sinks[2 * i]) if needs[2 * i] else None)
        g.append(_bias_grad(dy.float().sum(0), b, sinks[2 * i + 1]) if needs[2 * i + 1] else None)
    return g


def attention_train_supported(x, batch, seq_len, heads, head_dim=64) -> bool:
    return (x.is_cuda and x.dim() == 2 and x.shape[1] % 8 == 0
            and _Padded(None, batch, seq_len).supported(x.shape[0], heads, head_dim))


def attention_forward_saved(qkv, mask, batch, seq_len, heads, drop=None):
    """The kernel forward with the statistics the backward needs: (out bf16 [B * L, H * D], lse fp32 [B, H, L]), D the
    head dim of qkv [B * L, 3 * H * D] (32 or 64).
    ``drop``: a drawn dropout site (``_draw``) for the probabilities, element (b, h, i, j) at ((b H + h) L + i) L + j;
    lse is that of the undropped softmax."""
    from . import native, count_launch

    out = torch.empty((batch * seq_len, qkv.shape[1] // 3), device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty((batch, heads, seq_len), device=qkv.device, dtype=torch.float32)
    native().attention_fwd(qkv, mask, out, batch, seq_len, heads, lse, drop)
    count_launch()
    return out, lse


def attention_backward(qkv, mask, out, lse, dout, batch, seq_len, heads, drop=None):
    """dqkv bf16 [B * L, 3 * H * D] (dQ | dK | dV in qkv's layout) of ``attention``, from the forward's ``out`` and
    ``lse`` (``attention_forward_saved``, with the same ``drop``) and the output gradient ``dout``."""
    from . import native, count_launch

    dqkv = torch.empty_like(qkv)
    delta = torch.empty((batch, heads, seq_len), device=qkv.device, dtype=torch.float32)
    native().attention_bwd(qkv, mask, out, lse, _bf16(dout).contiguous(), dqkv, delta, batch, seq_len, heads, drop)
    count_launch(3)
    return dqkv


def attention_varlen_forward_saved(qkv, cu_seqlens, max_len, heads, key_mask=None, drop=None):
    """The packed kernel forward with the statistics the backward needs: (out bf16 [T, H * D], lse fp32 [H, T], lse
    of head h and packed row r at [h, r]).  ``drop``: a drawn dropout site for the probabilities, element (b, h, i, j) at
    ((b H + h) 512 + i) 512 + j; lse is that of the undropped softmax.  ``cu_seqlens`` int32 and ``key_mask`` uint8 (or
    None), contiguous, on qkv's device."""
    from . import native, count_launch

    t = qkv.shape[0]
    out = torch.empty((t, qkv.shape[1] // 3), device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty((heads, t), device=qkv.device, dtype=torch.float32)
    maps = torch.empty((cu_seqlens.numel() - 1) * 256, device=qkv.device, dtype=torch.uint8)
    native().attention_varlen_fwd(qkv, cu_seqlens, key_mask, out, maps, int(max_len), heads, lse, drop)
    count_launch(2)
    return out, lse


def attention_varlen_backward(qkv, cu_seqlens, max_len, heads, key_mask, out, lse, dout, drop=None):
    """dqkv bf16 [T, 3 * H * D] of ``attention_varlen`` from the forward's ``out`` and ``lse``
    (``attention_varlen_forward_saved``, with the same ``drop``) and the output gradient ``dout``.  Every row must
    belong to a sequence (cu_seqlens[-1] == T, as ``pack_sequences`` makes it): rows outside all sequences are not
    written."""
    from . import native, count_launch

    dqkv = torch.empty_like(qkv)
    delta = torch.empty((heads, qkv.shape[0]), device=qkv.device, dtype=torch.float32)
    native().attention_varlen_bwd(qkv, cu_seqlens, key_mask, out, lse, _bf16(dout).contiguous(), dqkv, delta,
                                  int(max_len), heads, drop)
    count_launch(3)
    return dqkv


# A layout is everything the training attention knows about how sequences sit in the rows: the kernels' shape check,
# the kernel forward / backward pair, the float32 reference, the fallback mask of the probability-dropout site and the
# shape in a fallback message.  The other dropout sites are row-wise and do not depend on it.
class _Padded:
    """The padded layout [B, L]: rows b * L + i, ``mask`` [B, L] (nonzero = attend) or None."""

    def __init__(self, mask, batch, seq_len):
        self.mask, self.batch, self.seq_len = _mask_u8(mask), batch, seq_len

    def supported(self, rows, heads, head_dim):
        from . import native

        return rows == self.batch * self.seq_len and native().attention_supported(self.batch, self.seq_len, heads,
                                                                                  head_dim)

    def forward(self, qkv, heads, drop):
        return attention_forward_saved(qkv, self.mask, self.batch, self.seq_len, heads, drop)

    def backward(self, qkv, out, lse, dout, heads, drop):
        return attention_backward(qkv, self.mask, out, lse, dout, self.batch, self.seq_len, heads, drop)

    def reference(self, qkv, heads, head_dim, drop_z):
        return attention_reference(qkv, self.mask, self.batch, self.seq_len, heads, head_dim, drop_z)

    def dropout_z(self, t, p, heads):
        """Probability (b, h, i, j) at ((b H + h) L + i) L + j."""
        return _site_z(t, p, (self.batch, heads, self.seq_len, self.seq_len))

    def describe(self, rows, heads, width):
        return "B %d, L %d, H %d, width %d" % (self.batch, self.seq_len, heads, width)


class _Packed:
    """Sequences packed back to back: ``cu_seqlens`` [B + 1], host ``max_len``, ``key_mask`` [T] (nonzero = attend) or
    None."""

    def __init__(self, cu_seqlens, max_len, key_mask):
        self.cu_seqlens, self.max_len, self.key_mask = _cu_i32(cu_seqlens), int(max_len), _mask_u8(key_mask)

    def supported(self, rows, heads, head_dim):
        from . import native

        cu = self.cu_seqlens
        return (cu.is_cuda and cu.dim() == 1 and cu.numel() >= 2
                and native().attention_varlen_supported(rows, cu.numel() - 1, self.max_len, heads, head_dim))

    def forward(self, qkv, heads, drop):
        return attention_varlen_forward_saved(qkv, self.cu_seqlens, self.max_len, heads, self.key_mask, drop)

    def backward(self, qkv, out, lse, dout, heads, drop):
        return attention_varlen_backward(qkv, self.cu_seqlens, self.max_len, heads, self.key_mask, out, lse, dout, drop)

    def reference(self, qkv, heads, head_dim, drop_z):
        return attention_varlen_reference(qkv, self.cu_seqlens, self.max_len, heads, self.key_mask, drop_z)

    def dropout_z(self, t, p, heads):
        """Per sequence b a [1, H, len_b, len_b] block, probability (b, h, i, j) at ((b H + h) 512 + i) 512 + j; on
        CPU the blocks of one F.dropout mask of [B, H, max_len, max_len]."""
        m, k = self.max_len, _ATTN_MAX_LEN
        z = _site_z(t, p, (self.cu_seqlens.numel() - 1, heads, m, m), (heads * k * k, k * k, k, 1))
        if z is None:
            return None
        cu = self.cu_seqlens.tolist()
        return [z[b:b + 1, :, :e - s, :e - s] for b, (s, e) in enumerate(zip(cu[:-1], cu[1:]))]

    def describe(self, rows, heads, width):
        return "T %d, B %d, max_len %d, H %d, width %d" % (rows, self.cu_seqlens.numel() - 1, self.max_len, heads,
                                                           width)


class _AttentionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, layout, heads, drop):
        out, lse = layout.forward(qkv, heads, drop)
        ctx.save_for_backward(qkv, out, lse)
        ctx.layout, ctx.heads, ctx.drop = layout, heads, drop
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, out, lse = ctx.saved_tensors
        return ctx.layout.backward(qkv, out, lse, dout, ctx.heads, ctx.drop), None, None, None


def _attention_trainable(name, qkv, layout, heads, head_dim, dropout_p):
    """``attention_trainable`` / ``attention_varlen_trainable`` over ``layout``; ``name`` heads the fallback message."""
    p = _check_p(dropout_p)
    if qkv.is_cuda and qkv.dim() == 2 and qkv.shape[1] == 3 * heads * head_dim:
        q = _bf16(qkv).contiguous()
        if q.data_ptr() % 16 == 0 and layout.supported(q.shape[0], heads, head_dim):
            return _AttentionFn.apply(q, layout, heads, _draw(q.device, p) if p > 0.0 else None)
    if qkv.is_cuda:
        _count("%s: no training kernel for %s: float32 math on the library"
               % (name, layout.describe(qkv.shape[0], heads, qkv.shape[-1])))
    return layout.reference(qkv.float(), heads, head_dim, layout.dropout_z(qkv, p, heads))


def attention_varlen_trainable(qkv, cu_seqlens, max_len, heads, key_mask=None, dropout_p=0.0):
    """``attention_varlen`` with a gradient, the packed sibling of ``attention_trainable``: the kernel path saves lse
    [H, T] and runs the packed backward of attention_bwd.cu.  ``qkv`` [T, 3 * H * D] with every row inside a sequence
    (cu_seqlens[-1] == T).  ``dropout_p``: dropout on the attention probabilities (one site, index
    ((b H + h) 512 + i) 512 + j).  On CPU, and for a shape the kernels do not take, ``attention_varlen_reference`` runs
    under autograd (counted through ``count_fallback`` on CUDA)."""
    return _attention_trainable("attention_varlen", qkv, _Packed(cu_seqlens, max_len, key_mask), heads,
                                qkv.shape[-1] // (3 * heads), dropout_p)


def attention_trainable(qkv, mask, batch, seq_len, heads, head_dim=64, dropout_p=0.0):
    """``attention`` with a gradient: the kernel path saves lse and runs attention_bwd.cu in the backward.
    ``dropout_p``: dropout on the attention probabilities (one site, index ((b H + h) L + i) L + j)."""
    return _attention_trainable("attention", qkv, _Padded(mask, batch, seq_len), heads, head_dim, dropout_p)


class _AttentionBlockFn(torch.autograd.Function):
    """h = attention(x W_qkv^T + b_qkv) W_o^T + b_o + x, the attention half of a post-LN encoder layer before its
    LayerNorm.  Backward: dctx = dh W_o, dqkv by attention_bwd.cu, and dx = dqkv W_qkv + dh as ONE dgrad GEMM with the
    residual gradient as its fused addend; dW_qkv and dW_o through ``_wgrad``.  ``layout`` (``_Padded`` or ``_Packed``)
    picks the attention forward / backward pair; everything else is row-wise and the same for both.

    ``drops`` = (attention-probability site, output-branch site), each None at p = 0.  With the branch dropout the output
    projection's epilogue stores x + Z o (o W_o^T + b_o); the backward forms dh_b = Z o dh (dropout.cu) for dctx, dW_o
    and db_o, while the residual still receives dh."""

    @staticmethod
    def forward(ctx, x, qkv_w, qkv_b, out_w, out_b, layout, heads, sinks, drops):
        from .gemm import gemm_bf16, gemm_bf16_residual_dropout

        x = _bf16(x).contiguous()
        wq, wo = _bf16(qkv_w).contiguous(), _bf16(out_w).contiguous()
        qkv = gemm_bf16(x, wq, col_shift=qkv_b.float())
        o, lse = layout.forward(qkv, heads, drops[0])
        if drops[1] is None:
            h = gemm_bf16(o, wo, col_shift=out_b.float(), add=x)
        else:
            h = gemm_bf16_residual_dropout(o, wo, out_b, x, drops[1])
        ctx.save_for_backward(x, wq, wo, qkv, o, lse, qkv_w, qkv_b, out_w, out_b)
        ctx.layout, ctx.heads, ctx.sinks, ctx.drops = layout, heads, sinks, drops
        return h

    @staticmethod
    def backward(ctx, dh):
        from .gemm import gemm_bf16

        x, wq, wo, qkv, o, lse, qkv_w, qkv_b, out_w, out_b = ctx.saved_tensors
        dh = _bf16(dh).contiguous()
        dhb = dh if ctx.drops[1] is None else _dropout_apply(dh, ctx.drops[1])
        dctx = gemm_bf16(dhb, wo, b_mn_major=True)
        dqkv = ctx.layout.backward(qkv, o, lse, dctx, ctx.heads, ctx.drops[0])
        dx = gemm_bf16(dqkv, wq, b_mn_major=True, add=dh) if ctx.needs_input_grad[0] else None
        g = _weight_bias_grads(ctx.needs_input_grad[1:5], ctx.sinks, (dqkv, x, qkv_w, qkv_b), (dhb, o, out_w, out_b))
        return (dx, *g, None, None, None, None)


def _attention_block(name, x, qkv_w, qkv_b, out_w, out_b, layout, heads, attn_dropout, hidden_dropout):
    """``attention_block`` / ``attention_block_varlen`` over ``layout``; ``name`` heads the fallback message."""
    from .gemm import _grad_sink

    pa, ph = _check_p(attn_dropout), _check_p(hidden_dropout)
    c = x.shape[-1]
    if x.is_cuda and x.dim() == 2 and c % 8 == 0 and c % heads == 0 and layout.supported(x.shape[0], heads, c // heads):
        sinks = tuple(_grad_sink(p) for p in (qkv_w, qkv_b, out_w, out_b))
        drops = tuple(_draw(x.device, p) if p > 0.0 else None for p in (pa, ph))
        return _AttentionBlockFn.apply(x, qkv_w, qkv_b, out_w, out_b, layout, heads, sinks, drops)
    if x.is_cuda:
        _count("%s: no kernel for %s: float32 math on the library" % (name, layout.describe(x.shape[0], heads, c)))
    za = layout.dropout_z(x, pa, heads)
    zh = _site_z(x, ph, (x.shape[0], c))
    f = torch.float32
    xf = x.float()
    qkv = torch.nn.functional.linear(xf, qkv_w.to(f), qkv_b.to(f))
    h = torch.nn.functional.linear(layout.reference(qkv, heads, qkv.shape[1] // (3 * heads), za), out_w.to(f),
                                   out_b.to(f))
    return (h if zh is None else zh * h) + xf


def attention_block(x, qkv_w, qkv_b, out_w, out_b, mask, batch, seq_len, heads, attn_dropout=0.0, hidden_dropout=0.0):
    """Attention sub-layer with its residual: attention(x W_qkv^T + b_qkv) W_o^T + b_o + x, x [B * L, C] (bf16 on
    CUDA), the weights in any float dtype (cast to bf16 here), ``mask`` [B, L] (nonzero = attend) or None.  Returns
    bf16 on the kernel path (the input of the following LayerNorm); differentiable in x and the four parameters.
    ``attn_dropout`` drops attention probabilities, then ``hidden_dropout`` the output branch before the residual add
    (two sites, in that order; branch index row * C + col).  The kernels take head dim C / heads = 32 or 64."""
    return _attention_block("attention_block", x, qkv_w, qkv_b, out_w, out_b, _Padded(mask, batch, seq_len), heads,
                            attn_dropout, hidden_dropout)


def attention_block_varlen(x, qkv_w, qkv_b, out_w, out_b, cu_seqlens, max_len, heads, key_mask=None,
                           attn_dropout=0.0, hidden_dropout=0.0):
    """``attention_block`` on sequences packed back to back: x [T, C] holds the real tokens only, sequence b in rows
    [cu_seqlens[b], cu_seqlens[b + 1]) (every row inside a sequence, as ``pack_sequences`` makes them), ``max_len``
    (host int) at least the longest length, ``key_mask`` [T] (nonzero = attend) or None.  The same GEMMs, fused residual
    gradient and weight-gradient hand-off as the padded form; attention runs the packed kernels.  Dropout sites as in
    ``attention_block``: the probabilities at ((b H + h) 512 + i) 512 + j, then the output branch at row * C + col.
    Nothing reads back to the host on the kernel path."""
    return _attention_block("attention_block_varlen", x, qkv_w, qkv_b, out_w, out_b,
                            _Packed(cu_seqlens, max_len, key_mask), heads, attn_dropout, hidden_dropout)


class _GeluFfnFn(torch.autograd.Function):
    """h = gelu(x W1^T + b1) W2^T + b2 + x, the feed-forward half of a post-LN encoder layer before its LayerNorm.
    FFN1 runs the GELU training epilogue (stores gelu(u) for FFN2 and u for the backward); FFN2's dgrad applies gelu'(u)
    in its epilogue, so dU comes out of one GEMM; dx = dU W1 + dh is one dgrad GEMM with the residual gradient fused.
    ``drop``: the output-branch dropout site or None; FFN2's epilogue then stores x + Z o (y W2^T + b2) and the backward
    takes dh_b = Z o dh for dU, dW2 and db2 (the residual receives dh)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, sinks, drop):
        from .gemm import gemm_bf16, gemm_bf16_gelu_train, gemm_bf16_residual_dropout

        x = _bf16(x).contiguous()
        w1h, w2h = _bf16(w1).contiguous(), _bf16(w2).contiguous()
        y, u = gemm_bf16_gelu_train(x, w1h, b1.float())
        if drop is None:
            h = gemm_bf16(y, w2h, col_shift=b2.float(), add=x)
        else:
            h = gemm_bf16_residual_dropout(y, w2h, b2, x, drop)
        ctx.save_for_backward(x, w1h, w2h, y, u, w1, b1, w2, b2)
        ctx.sinks, ctx.drop = sinks, drop
        return h

    @staticmethod
    def backward(ctx, dh):
        from .gemm import gemm_bf16, gemm_bf16_gelu_grad

        x, w1h, w2h, y, u, w1, b1, w2, b2 = ctx.saved_tensors
        dh = _bf16(dh).contiguous()
        dhb = dh if ctx.drop is None else _dropout_apply(dh, ctx.drop)
        du = gemm_bf16_gelu_grad(dhb, w2h, u)
        dx = gemm_bf16(du, w1h, b_mn_major=True, add=dh) if ctx.needs_input_grad[0] else None
        g = _weight_bias_grads(ctx.needs_input_grad[1:5], ctx.sinks, (du, x, w1, b1), (dhb, y, w2, b2))
        return (dx, *g, None, None)


def gelu_ffn_reference(x, w1, b1, w2, b2, drop_z=None):
    """Float32 math of ``gelu_ffn``; ``drop_z`` [rows, C]: dropout (keep * scale) on the output branch."""
    f = torch.float32
    xf = x.float()
    u = torch.nn.functional.linear(xf, w1.to(f), b1.to(f))
    h = torch.nn.functional.linear(torch.nn.functional.gelu(u), w2.to(f), b2.to(f))
    return (h if drop_z is None else drop_z * h) + xf


def gelu_ffn(x, w1, b1, w2, b2, dropout_p=0.0):
    """Feed-forward sub-layer with its residual: gelu(x W1^T + b1) W2^T + b2 + x (erf GELU), x [rows, C] (bf16 on
    CUDA), weights in any float dtype.  This is the trainable GELU linear: its backward needs FFN2's dgrad, which is
    where gelu'(u) is applied.  Returns bf16 on the kernel path; differentiable in x and the four parameters.
    ``dropout_p``: dropout on the output branch before the residual add (one site, index row * C + col)."""
    from .gemm import _grad_sink, _tma_compatible
    from . import native

    p = _check_p(dropout_p)
    ffn, c = w1.shape
    if (x.is_cuda and x.dim() == 2 and c % 8 == 0 and ffn % 8 == 0 and native().persistent_gemm_enabled()
            and _tma_compatible(_bf16(x).contiguous(), _bf16(w1), None, ffn)):
        sinks = tuple(_grad_sink(t) for t in (w1, b1, w2, b2))
        return _GeluFfnFn.apply(x, w1, b1, w2, b2, sinks, _draw(x.device, p) if p > 0.0 else None)
    if x.is_cuda:
        _count("gelu_ffn: no kernel for x %s, FFN %d (persistent GEMM on, widths % 8 == 0): float32 math on the library"
               % (tuple(x.shape), ffn))
    return gelu_ffn_reference(x, w1, b1, w2, b2, _site_z(x, p, (x.shape[0], c)))


def _ln_part(rows, c, device):
    from . import native

    return torch.empty(native().layernorm_bwd_ctas(rows) * 2 * c, device=device, dtype=torch.float32)


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        x = _bf16(x).contiguous()
        y = layer_norm(x, gamma, beta, eps)
        ctx.save_for_backward(x, gamma, beta)
        ctx.eps = eps
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        x, gamma, beta = ctx.saved_tensors
        dy = _bf16(dy).contiguous()
        dx = torch.empty_like(x)
        c = x.shape[1]
        dg = torch.empty(c, device=x.device, dtype=torch.float32)
        db = torch.empty_like(dg)
        native().layernorm_bwd(x, dy, gamma.float().contiguous(), dx, _ln_part(x.shape[0], c, x.device), dg, db,
                               float(ctx.eps))
        count_launch(2)
        return dx, dg.to(gamma.dtype), db.to(beta.dtype), None


def layer_norm_trainable(x, gamma, beta, eps=1e-12):
    """``layer_norm`` with a gradient: the forward kernel, and layernorm_bwd (dx from the saved input, dgamma / dbeta by
    per-CTA partials and a fixed-order reduction)."""
    if x.is_cuda and layer_norm_supported(_bf16(x).contiguous()):
        return _LayerNormFn.apply(x, gamma, beta, eps)
    if x.is_cuda:
        _count("layer_norm: no training kernel for %s %s: float32 math on the library" % (tuple(x.shape), x.dtype))
    return layer_norm_reference(x.float(), gamma, beta, eps)


_ONE_HOT_ROWS = 1024


def _table_grad(dE, idx, rows):
    if rows <= _ONE_HOT_ROWS:
        return torch.nn.functional.one_hot(idx, rows).to(dE.dtype).t() @ dE
    return torch.ops.aten.embedding_dense_backward(dE, idx, rows, -1, False)


class _EmbeddingLayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps, drop):
        tabs = tuple(_bf16(t).contiguous() for t in (word, pos, seg))
        ids, pos_ids, seg_ids = (t.reshape(-1).to(word.device, torch.int64).contiguous() for t in (ids, pos_ids, seg_ids))
        if drop is None:
            y = embedding_layernorm(ids, pos_ids, seg_ids, *tabs, gamma, beta, eps)
        else:
            y = _embedding_layernorm_kernel(ids, pos_ids, seg_ids, *tabs, gamma, beta, eps, None, drop)
        ctx.save_for_backward(ids, pos_ids, seg_ids, *tabs, gamma, beta)
        ctx.eps, ctx.drop = eps, drop
        ctx.dtypes = (word.dtype, pos.dtype, seg.dtype)
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        ids, pos_ids, seg_ids, word, pos, seg, gamma, beta = ctx.saved_tensors
        rows, c = ids.numel(), word.shape[1]
        dE = torch.empty((rows, c), device=word.device, dtype=torch.float32)
        dg = torch.empty(c, device=word.device, dtype=torch.float32)
        db = torch.empty_like(dg)
        native().embedding_layernorm_bwd(ids, pos_ids, seg_ids, word, pos, seg, _bf16(dy).contiguous(),
                                         gamma.float().contiguous(), dE, _ln_part(rows, c, word.device), dg, db,
                                         float(ctx.eps), ctx.drop)
        count_launch(2)
        # the three table gradients, dE summed per table row.  The word table: the library's embedding backward, the
        # call nn.Embedding makes for the BiLSTM student.  The position and segment tables (at most _ONE_HOT_ROWS rows)
        # see every id many times per batch, where that call was measured to vary from run to run; for them the sum is a
        # one-hot GEMM, which is bitwise reproducible.
        grads = [None if not ctx.needs_input_grad[3 + i] else _table_grad(dE, idx, tab.shape[0]).to(dt)
                 for i, (idx, tab, dt) in enumerate(zip((ids, pos_ids, seg_ids), (word, pos, seg), ctx.dtypes))]
        return None, None, None, *grads, dg.to(gamma.dtype), db.to(beta.dtype), None, None


def embedding_layernorm_trainable(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps=1e-12, dropout_p=0.0):
    """``embedding_layernorm`` with a gradient in the three tables and gamma / beta (tables in any float dtype, cast
    to bf16 for the kernels).  Out-of-range ids raise as in ``embedding_layernorm``.  ``dropout_p``: dropout on the
    output (one site, index row * C + col), applied by the same kernel."""
    c = word.shape[1]
    from . import native

    p = _check_p(dropout_p)
    if word.is_cuda and all(t.is_cuda and t.dim() == 2 and t.shape[1] == c for t in (pos, seg)) \
            and native().layernorm_supported(c):
        return _EmbeddingLayerNormFn.apply(ids, pos_ids, seg_ids, word, pos, seg, gamma, beta, eps,
                                           _draw(word.device, p) if p > 0.0 else None)
    if word.is_cuda:
        _count("embedding_layernorm: no training kernel for width %d: float32 math on the library" % c)
    f = torch.float32
    y = embedding_layernorm_reference(ids, pos_ids, seg_ids, word.to(f), pos.to(f), seg.to(f), gamma, beta, eps)
    z = _site_z(word, p, (ids.numel(), c))
    return y if z is None else y * z
