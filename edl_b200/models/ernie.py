"""ERNIE 1.0 / BERT-style encoder for sequence classification, the NLP teacher of the ERNIE -> BOW distillation
(the reference serves ERNIE 1.0 base with Paddle Serving; example/distill/nlp).

Post-LN Transformer layers: QKV projection, masked multi-head attention, output projection + residual, LayerNorm,
FFN1 with bias + erf-GELU, FFN2 + residual, LayerNorm; the [CLS] row goes through a tanh pooler and the classifier.
Inference only.

On CUDA every layer runs on the package's own kernels: the wgmma GEMM (bias in the epilogue, the residual as its fused
addend, GELU as a compile-time epilogue variant), the attention kernel reading Q / K / V in place from the QKV output,
the LayerNorm and the embedding-sum + LayerNorm kernels.  The weight matrices are cast to bf16 once, at the first CUDA
forward after a load or a move; biases and LayerNorm parameters stay fp32.  On CPU the same forward runs in float32
PyTorch math (the reference the GPU path is tested against).

``forward_packed`` runs the same layers on a batch packed to its real tokens (``pack_sequences``) with the
variable-length attention kernel; ``forward_requests`` packs requests of different lengths for the teacher server.
``ErnieStudent.forward_packed`` is its training form.

``enable_fp8()`` switches the four linear layers of every encoder layer to the block-scaled e4m3 GEMM (ops/fp8.py):
the LayerNorms write the next GEMM's quantised operand themselves, FFN1's epilogue quantises its GELU output for FFN2,
and the residual adds run in the out-projection's and FFN2's epilogues.  The attention output is quantised by
``quantize_e4m3_blocks``.  Embeddings, attention, pooler and classifier stay bf16.  On CPU an enabled model emulates
that pipeline through the float32 paths of the same ops, rounding to bf16 wherever the GPU stores bf16."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..ops import fp8

CLS_PAD = 8      # classifier rows after padding: a 2-class output row (4 bytes) is not a TMA-describable pitch


MAX_SEQ_LEN = 512  # the attention kernels' longest sequence


def pack_sequences(input_ids, position_ids, segment_ids, input_mask, max_positions=None):
    """Pack a padded batch ([B, L] or [B, L, 1] numpy arrays or CPU tensors) into its real tokens, for
    ``ErnieEncoder.forward_packed``.

    Keeps every token whose mask is nonzero and always token 0 of each sample (the [CLS] row the pooler reads), in
    order.  Returns int64 CPU tensors ``ids, pos, seg`` [T], int32 ``cu_seqlens`` [B + 1], the host int ``max_len`` and
    ``key_mask``: uint8 [T] when some sample's token 0 is masked (it is kept as a query but is not a key), else None.
    The packed forward is then the padded forward for any mask, an empty one included.  Raises ValueError for a sample
    of more than 512 kept tokens, or more than ``max_positions`` (the position table) when given."""
    def arr(t):
        return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)

    mask = arr(input_mask)
    b = mask.shape[0]
    mask = mask.reshape(b, -1) != 0
    if b == 0 or mask.shape[1] == 0:
        raise ValueError("pack_sequences: empty batch %s" % (mask.shape,))
    keep = mask.copy()
    keep[:, 0] = True
    lens = keep.sum(1)
    limit = MAX_SEQ_LEN if max_positions is None else min(MAX_SEQ_LEN, int(max_positions))
    if int(lens.max()) > limit:
        raise ValueError("pack_sequences: a sample has %d tokens; at most %d are supported" % (int(lens.max()), limit))
    cu = np.zeros(b + 1, np.int32)
    np.cumsum(lens, out=cu[1:])
    ids, pos, seg = (torch.from_numpy(np.ascontiguousarray(arr(t).reshape(mask.shape)[keep], dtype=np.int64))
                     for t in (input_ids, position_ids, segment_ids))
    key_mask = None if mask[:, 0].all() else torch.from_numpy(mask[keep].astype(np.uint8))
    return ids, pos, seg, torch.from_numpy(cu), int(lens.max()), key_mask


class ErnieEncoder(nn.Module):
    def __init__(self, vocab=18000, hidden=768, layers=12, heads=12, ffn=3072, max_pos=513, type_vocab=2,
                 num_labels=2, eps=1e-12):
        super().__init__()
        if hidden % heads != 0:
            raise ValueError("hidden %d is not a multiple of heads %d" % (hidden, heads))
        self.hidden, self.heads, self.head_dim, self.num_labels, self.eps = hidden, heads, hidden // heads, num_labels, eps
        self.num_layers = layers
        std = 0.02

        def mat(*shape):
            return nn.Parameter(torch.randn(*shape) * std)

        def vec(n, value=0.0):
            return nn.Parameter(torch.full((n,), float(value)))

        self.word_emb, self.pos_emb, self.seg_emb = mat(vocab, hidden), mat(max_pos, hidden), mat(type_vocab, hidden)
        self.emb_ln_g, self.emb_ln_b = vec(hidden, 1.0), vec(hidden)
        self.layers = nn.ModuleList()
        for _ in range(layers):
            lyr = nn.Module()
            lyr.qkv_w, lyr.qkv_b = mat(3 * hidden, hidden), vec(3 * hidden)
            lyr.out_w, lyr.out_b = mat(hidden, hidden), vec(hidden)
            lyr.ln1_g, lyr.ln1_b = vec(hidden, 1.0), vec(hidden)
            lyr.ffn1_w, lyr.ffn1_b = mat(ffn, hidden), vec(ffn)
            lyr.ffn2_w, lyr.ffn2_b = mat(hidden, ffn), vec(hidden)
            lyr.ln2_g, lyr.ln2_b = vec(hidden, 1.0), vec(hidden)
            self.layers.append(lyr)
        self.pool_w, self.pool_b = mat(hidden, hidden), vec(hidden)
        self.cls_w, self.cls_b = mat(num_labels, hidden), vec(num_labels)
        self.requires_grad_(False)
        self._dev = None          # CUDA copies of the weights (bf16 matrices, fp32 vectors), built at first use
        self._fp8 = False         # enable_fp8: the encoder's linear layers run block-scaled e4m3

    def enable_fp8(self, scaling="block"):
        """Run QKV, out-projection, FFN1 and FFN2 of every layer as block-scaled e4m3 GEMMs: one scale per activation
        row and 128-element K block, computed on the fly, and one per 128 x 128 weight block (no calibration, no host
        synchronisation).  Returns the number of converted linear layers (4 per encoder layer).  Only ``"block"``
        scaling is offered: a per-tensor activation scale needs a calibration pass."""
        if scaling != "block":
            raise ValueError("ErnieEncoder.enable_fp8: scaling %r is not supported; use 'block'" % (scaling,))
        self._fp8 = True
        self._dev = None
        return 4 * self.num_layers

    def _apply(self, fn, *args, **kwargs):
        self._dev = None
        return super()._apply(fn, *args, **kwargs)

    # ------------------------------------------------------------------------------------------------- weights
    def _device_weights(self):
        if self._dev is None:
            def m(t):
                return t.detach().to(torch.bfloat16).contiguous()

            def v(t):
                return t.detach().float().contiguous()

            if self._fp8:                         # (e4m3 bytes, block scales); no bf16 copy of these matrices
                def m_lin(t):
                    return fp8.quantize_weight_blocks(t.detach())
            else:
                m_lin = m

            n, c = self.num_labels, self.hidden
            cls_w = torch.zeros(max(CLS_PAD, -(-n // CLS_PAD) * CLS_PAD), c, device=self.cls_w.device)
            cls_w[:n] = self.cls_w.detach().float()
            cls_b = torch.zeros(cls_w.shape[0], device=self.cls_w.device)
            cls_b[:n] = self.cls_b.detach().float()
            self._dev = {
                "emb": (m(self.word_emb), m(self.pos_emb), m(self.seg_emb), v(self.emb_ln_g), v(self.emb_ln_b)),
                "layers": [tuple(f(getattr(lyr, k)) for f, k in (
                    (m_lin, "qkv_w"), (v, "qkv_b"), (m_lin, "out_w"), (v, "out_b"), (v, "ln1_g"), (v, "ln1_b"),
                    (m_lin, "ffn1_w"), (v, "ffn1_b"), (m_lin, "ffn2_w"), (v, "ffn2_b"), (v, "ln2_g"), (v, "ln2_b")))
                    for lyr in self.layers],
                "head": (m(self.pool_w), v(self.pool_b), m(cls_w), v(cls_b)),
            }
        return self._dev

    def load_bert_state_dict(self, sd, strict=True):
        """Load a BERT-layout state dict (``[bert.]embeddings.*``, ``[bert.]encoder.layer.N.*``, ``[bert.]pooler.*``
        and optionally ``classifier.*``; LayerNorm ``weight``/``bias`` or ``gamma``/``beta``).  Returns the names that
        were not used.  ``strict``: every encoder tensor must be present with the model's shape."""
        src = {}
        for k, t in sd.items():
            k = k[len("bert."):] if k.startswith("bert.") else k
            src[k.replace("LayerNorm.gamma", "LayerNorm.weight").replace("LayerNorm.beta", "LayerNorm.bias")] = t
        used = set()

        def take(name):
            if name not in src:
                raise KeyError("BERT state dict has no %r" % name)
            used.add(name)
            return src[name]

        def put(param, value):
            value = torch.as_tensor(value)
            if tuple(value.shape) != tuple(param.shape):
                raise ValueError("shape mismatch: %s for a parameter of %s" % (tuple(value.shape), tuple(param.shape)))
            param.data.copy_(value.to(param.dtype))

        e = "embeddings."
        put(self.word_emb, take(e + "word_embeddings.weight"))
        put(self.pos_emb, take(e + "position_embeddings.weight"))
        put(self.seg_emb, take(e + "token_type_embeddings.weight"))
        put(self.emb_ln_g, take(e + "LayerNorm.weight"))
        put(self.emb_ln_b, take(e + "LayerNorm.bias"))
        for i, lyr in enumerate(self.layers):
            p = "encoder.layer.%d." % i
            a = p + "attention.self."
            put(lyr.qkv_w, torch.cat([torch.as_tensor(take(a + n + ".weight")) for n in ("query", "key", "value")], 0))
            put(lyr.qkv_b, torch.cat([torch.as_tensor(take(a + n + ".bias")) for n in ("query", "key", "value")], 0))
            put(lyr.out_w, take(p + "attention.output.dense.weight"))
            put(lyr.out_b, take(p + "attention.output.dense.bias"))
            put(lyr.ln1_g, take(p + "attention.output.LayerNorm.weight"))
            put(lyr.ln1_b, take(p + "attention.output.LayerNorm.bias"))
            put(lyr.ffn1_w, take(p + "intermediate.dense.weight"))
            put(lyr.ffn1_b, take(p + "intermediate.dense.bias"))
            put(lyr.ffn2_w, take(p + "output.dense.weight"))
            put(lyr.ffn2_b, take(p + "output.dense.bias"))
            put(lyr.ln2_g, take(p + "output.LayerNorm.weight"))
            put(lyr.ln2_b, take(p + "output.LayerNorm.bias"))
        put(self.pool_w, take("pooler.dense.weight"))
        put(self.pool_b, take("pooler.dense.bias"))
        if "classifier.weight" in src:
            put(self.cls_w, take("classifier.weight"))
            put(self.cls_b, take("classifier.bias"))
        if strict and "encoder.layer.%d.attention.self.query.weight" % self.num_layers in src:
            raise ValueError("the state dict has more than %d encoder layers" % self.num_layers)
        self._dev = None
        return sorted(set(src) - used)

    def load_weights(self, path, strict=True):
        """``load_bert_state_dict`` from a ``.safetensors`` file or a torch-saved state dict."""
        if str(path).endswith(".safetensors"):
            from safetensors.torch import load_file

            sd = load_file(str(path))
        else:
            sd = torch.load(str(path), map_location="cpu", weights_only=True)
            sd = sd.get("state_dict", sd) if isinstance(sd, dict) else sd
        return self.load_bert_state_dict(sd, strict=strict)

    # ------------------------------------------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, input_ids, position_ids, segment_ids, input_mask):
        """ids int64 [B, L]; ``input_mask`` [B, L], nonzero = a real token.  Returns fp32 logits [B, num_labels]."""
        b, l = input_ids.shape[0], input_ids.shape[1]
        ids, pos, seg = (t.reshape(b, l).long() for t in (input_ids, position_ids, segment_ids))
        keep = input_mask.reshape(b, l) != 0
        if self.word_emb.is_cuda:
            mask, fwd = keep.to(torch.uint8).contiguous(), self._forward_cuda
        else:
            mask, fwd = keep, self._forward_reference
        return fwd(ids, pos, seg, lambda qkv: ops.attention(qkv, mask, b, l, self.heads, self.head_dim),
                   lambda x: x.view(b, l, self.hidden)[:, 0])                   # [B, C], row pitch L * C

    @torch.no_grad()
    def forward_packed(self, ids, pos, seg, cu_seqlens, max_len, key_mask=None):
        """The forward over packed sequences (``pack_sequences``): ids / pos / seg int64 [T], ``cu_seqlens`` int32
        [B + 1], ``max_len`` the longest length, ``key_mask`` uint8 [T] or None.  Every row-wise layer runs on the T real
        tokens only.  Returns fp32 logits [B, num_labels].  On CUDA the inputs are expected on the model's device; the
        path makes no host synchronisation under CUDA-graph capture, so it can be captured for fixed shapes."""
        dev = self.word_emb.device
        ids, pos, seg, cu_seqlens = (t.to(dev) for t in (ids, pos, seg, cu_seqlens))
        key_mask = None if key_mask is None else key_mask.to(dev)
        first = cu_seqlens[:-1].long()
        fwd = self._forward_cuda if self.word_emb.is_cuda else self._forward_reference
        return fwd(ids, pos, seg, lambda qkv: ops.attention_varlen(qkv, cu_seqlens, max_len, self.heads, key_mask),
                   lambda x: x.index_select(0, first))

    def forward_requests(self, requests):
        """Serve a batch of requests whose sequence lengths may differ: each request is the forward's four feeds
        ([n, L] or [n, L, 1], L per request).  Packs all samples on the host, copies the real tokens to the device and
        runs ``forward_packed``.  Returns fp32 logits [sum n, num_labels] in request order."""
        packs = [pack_sequences(*r, max_positions=self.pos_emb.shape[0]) for r in requests]
        ids, pos, seg = (torch.cat([p[i] for p in packs]) for i in range(3))
        lens = torch.cat([p[3].diff() for p in packs])
        cu = torch.zeros(len(lens) + 1, dtype=torch.int32)
        torch.cumsum(lens, 0, out=cu[1:])
        key_mask = None
        if any(p[5] is not None for p in packs):
            key_mask = torch.cat([p[5] if p[5] is not None else torch.ones(len(p[0]), dtype=torch.uint8) for p in packs])
        return self.forward_packed(ids, pos, seg, cu, max(p[4] for p in packs), key_mask)

    def _forward_cuda(self, ids, pos, seg, attend, cls_rows):
        if self._fp8:
            return self._forward_fp8(ids, pos, seg, attend, cls_rows)
        w = self._device_weights()
        word, pemb, semb, g, beta = w["emb"]
        x = ops.embedding_layernorm(ids, pos, seg, word, pemb, semb, g, beta, self.eps)
        for qkv_w, qkv_b, out_w, out_b, ln1_g, ln1_b, f1_w, f1_b, f2_w, f2_b, ln2_g, ln2_b in w["layers"]:
            qkv = ops.gemm_bf16(x, qkv_w, col_shift=qkv_b)
            ctx = attend(qkv)
            x = ops.layer_norm(ops.gemm_bf16(ctx, out_w, col_shift=out_b, add=x), ln1_g, ln1_b, self.eps)
            f = ops.gemm_bf16(x, f1_w, col_shift=f1_b, gelu=True)
            x = ops.layer_norm(ops.gemm_bf16(f, f2_w, col_shift=f2_b, add=x), ln2_g, ln2_b, self.eps)
        pool_w, pool_b, cls_w, cls_b = w["head"]
        pooled = torch.tanh(ops.linear_bf16(cls_rows(x), pool_w, pool_b))
        return ops.gemm_bf16(pooled, cls_w, col_shift=cls_b)[:, :self.num_labels].float()

    def _forward_fp8(self, ids, pos, seg, attend, cls_rows):
        """The FP8 layer flow; on CPU every op takes its float32 reference path on bf16 activations, which makes this
        the emulation the CUDA path is tested against."""
        w = self._device_weights()
        word, pemb, semb, g, beta = w["emb"]
        x, q, sa = ops.embedding_layernorm_e4m3(ids, pos, seg, word, pemb, semb, g, beta, self.eps)
        last = len(w["layers"]) - 1
        for i, (qkv_w, qkv_b, out_w, out_b, ln1_g, ln1_b, f1_w, f1_b, f2_w, f2_b, ln2_g, ln2_b) in enumerate(w["layers"]):
            qkv = fp8.gemm_fp8_blockscaled(q, sa, *qkv_w, col_shift=qkv_b)
            q, sa = fp8.quantize_e4m3_blocks(attend(qkv))
            x, q, sa = ops.layer_norm_e4m3(fp8.gemm_fp8_blockscaled(q, sa, *out_w, col_shift=out_b, add=x),
                                           ln1_g, ln1_b, self.eps)
            q, sa = fp8.gemm_fp8_gelu_e4m3(q, sa, *f1_w, bias=f1_b)
            h = fp8.gemm_fp8_blockscaled(q, sa, *f2_w, col_shift=f2_b, add=x)
            if i < last:
                x, q, sa = ops.layer_norm_e4m3(h, ln2_g, ln2_b, self.eps)
            else:                                  # the pooler reads bf16 x only
                x = ops.layer_norm(h, ln2_g, ln2_b, self.eps)
        pool_w, pool_b, cls_w, cls_b = w["head"]
        if x.is_cuda:
            pooled = torch.tanh(ops.linear_bf16(cls_rows(x), pool_w, pool_b))
            return ops.gemm_bf16(pooled, cls_w, col_shift=cls_b)[:, :self.num_labels].float()
        bf = torch.bfloat16
        pooled = torch.tanh(F.linear(cls_rows(x).float(), pool_w.float(), pool_b).to(bf))
        return F.linear(pooled.float(), cls_w.float(), cls_b).to(bf)[:, :self.num_labels].float()

    def _forward_reference(self, ids, pos, seg, attend, cls_rows):
        if self._fp8:
            return self._forward_fp8(ids, pos, seg, attend, cls_rows)
        f32 = torch.float32
        x = ops.embedding_layernorm(ids, pos, seg, self.word_emb.to(f32), self.pos_emb.to(f32), self.seg_emb.to(f32),
                                    self.emb_ln_g, self.emb_ln_b, self.eps)
        for lyr in self.layers:
            qkv = F.linear(x, lyr.qkv_w.to(f32), lyr.qkv_b.to(f32))
            ctx = attend(qkv)
            x = ops.layer_norm(F.linear(ctx, lyr.out_w.to(f32), lyr.out_b.to(f32)) + x, lyr.ln1_g, lyr.ln1_b, self.eps)
            f = F.gelu(F.linear(x, lyr.ffn1_w.to(f32), lyr.ffn1_b.to(f32)))
            x = ops.layer_norm(F.linear(f, lyr.ffn2_w.to(f32), lyr.ffn2_b.to(f32)) + x, lyr.ln2_g, lyr.ln2_b, self.eps)
        pooled = torch.tanh(F.linear(cls_rows(x), self.pool_w.to(f32), self.pool_b.to(f32)))
        return F.linear(pooled, self.cls_w.to(f32), self.cls_b.to(f32))


class ErnieStudent(ErnieEncoder):
    """A trainable ``ErnieEncoder``: the Transformer student of the NLP distillation.

    Same layers and parameter names as ``ErnieEncoder``, so a trained student's ``state_dict()`` loads into an
    ``ErnieEncoder`` of the same configuration and can be served by ``teacher_server`` unchanged.  The parameters are
    fp32 master copies; on CUDA each forward casts the matrices to bf16 and runs the training kernels of
    ops/transformer.py (attention and its backward, LayerNorm and embedding-LayerNorm with their backward, FFN1 with
    the GELU training epilogue and FFN2's gelu'-epilogue dgrad, residual gradients fused into the dgrad GEMMs).  On CPU
    the forward is the encoder's float32 reference under torch autograd.

    Dropout (keyword-only ``hidden_dropout`` / ``attention_dropout``, default 0; only while ``self.training``) sits
    where BERT puts it.  Each site draws one (seed, offset) pair of 4 offset units from the default CUDA generator of
    the device (``ops.transformer.dropout_keep_reference`` is the mask), in this order per forward:
      1. the embedding-LayerNorm output (hidden), index row * C + col, in the embedding-LayerNorm kernel;
      then per layer
      2. the attention probabilities (attention), index ((b H + h) L + i) L + j, in the attention kernels;
      3. the attention output branch before its residual add (hidden), index row * C + col, in the output projection's
         GEMM epilogue;
      4. the FFN output branch before its residual add (hidden), index row * C + col, in FFN2's GEMM epilogue;
      and last
      5. the pooled [CLS] features before the classifier (hidden), index b * C + col, through ``ops.dropout``.
    A step thus advances the generator offset by 4 * (2 + 3 * layers).  A site with p = 0 draws nothing and runs the
    p = 0 kernels; on CPU the sites are ``F.dropout``.  Dropout adds no parameters or buffers.

    ``forward`` also takes the token ids alone: positions are then 0 .. L - 1, segments 0 and the mask ``ids != 0``.

    ``forward_packed`` trains on a batch packed to its real tokens (``pack_sequences``): every GEMM, LayerNorm and
    attention tile runs on the T real rows only, and the [CLS] rows are rows cu_seqlens[:-1].  Its dropout sites and
    their order are those above, with packed indices: the hidden sites (1, 3, 4) at packed row * C + col, the attention
    probabilities (2) at ((b H + h) 512 + i) 512 + j (a fixed stride, so the sequences' index ranges are disjoint), the
    pooled features (5) at b * C + col; a step advances the offset by the same 4 * (2 + 3 * layers).  The padded
    ``forward`` is the shape-stable entry point: one graph per (B, L), where a packed step's graph is fixed to its T and
    cu_seqlens."""

    def __init__(self, *args, hidden_dropout=0.0, attention_dropout=0.0, **kwargs):
        super().__init__(*args, **kwargs)
        for p in (hidden_dropout, attention_dropout):
            if not 0.0 <= float(p) < 1.0:
                raise ValueError("ErnieStudent: dropout probabilities must satisfy 0 <= p < 1, got %r" % p)
        self.hidden_dropout, self.attention_dropout = float(hidden_dropout), float(attention_dropout)
        self.requires_grad_(True)

    def enable_fp8(self, scaling="block"):
        raise ValueError("ErnieStudent trains in bf16; load its state dict into an ErnieEncoder to serve it in FP8")

    def forward(self, input_ids, position_ids=None, segment_ids=None, input_mask=None):
        """ids int64 [B, L] (and optionally the other three feeds, [B, L]).  Returns fp32 logits [B, num_labels]."""
        b, l = input_ids.shape[0], input_ids.shape[1]
        ids = input_ids.reshape(b, l).long()
        pos = (torch.arange(l, device=ids.device).expand(b, l) if position_ids is None
               else position_ids.reshape(b, l).long())
        seg = torch.zeros_like(ids) if segment_ids is None else segment_ids.reshape(b, l).long()
        keep = (ids != 0) if input_mask is None else (input_mask.reshape(b, l) != 0)
        c = self.hidden
        hd, ad = (self.hidden_dropout, self.attention_dropout) if self.training else (0.0, 0.0)
        if not self.word_emb.is_cuda:
            if hd > 0.0 or ad > 0.0:
                return self._forward_dropout_cpu(ids, pos, seg, keep, hd, ad)
            return self._forward_reference(ids, pos, seg, lambda qkv: ops.attention(qkv, keep, b, l, self.heads,
                                                                                    self.head_dim),
                                           lambda x: x.view(b, l, c)[:, 0])
        mask = keep.to(torch.uint8).contiguous()
        x = ops.embedding_layernorm_trainable(ids, pos, seg, self.word_emb, self.pos_emb, self.seg_emb, self.emb_ln_g,
                                              self.emb_ln_b, self.eps, dropout_p=hd)
        for lyr in self.layers:
            h = ops.attention_block(x, lyr.qkv_w, lyr.qkv_b, lyr.out_w, lyr.out_b, mask, b, l, self.heads,
                                    attn_dropout=ad, hidden_dropout=hd)
            x = ops.layer_norm_trainable(h, lyr.ln1_g, lyr.ln1_b, self.eps)
            h = ops.gelu_ffn(x, lyr.ffn1_w, lyr.ffn1_b, lyr.ffn2_w, lyr.ffn2_b, dropout_p=hd)
            x = ops.layer_norm_trainable(h, lyr.ln2_g, lyr.ln2_b, self.eps)
        bf = torch.bfloat16
        pooled = torch.tanh(ops.linear_bf16(x.view(b, l, c)[:, 0], self.pool_w.to(bf), self.pool_b))
        pooled = ops.dropout(pooled, hd)
        n = self.num_labels
        pad = max(CLS_PAD, -(-n // CLS_PAD) * CLS_PAD) - n          # TMA-describable classifier rows, as the encoder
        logits = ops.linear_bf16(pooled, F.pad(self.cls_w, (0, 0, 0, pad)).to(bf), F.pad(self.cls_b, (0, pad)))
        return logits[:, :n].float()


    def forward_packed(self, ids, pos, seg, cu_seqlens, max_len, key_mask=None):
        """The training forward over packed sequences, with the arguments ``pack_sequences`` returns: ids / pos / seg
        int64 [T], ``cu_seqlens`` int32 [B + 1], ``max_len`` (host int) the longest length, ``key_mask`` uint8 [T] or
        None.  Returns fp32 logits [B, num_labels] with a gradient; the padded ``forward`` of the same batch up to the
        order of floating-point sums.  On CUDA the inputs are expected on the model's device; nothing reads back to the
        host under CUDA-graph capture, so a step can be captured for a fixed T and cu_seqlens.  Under
        ``torch.no_grad()`` at p = 0 the logits are those of ``ErnieEncoder.forward_packed``."""
        dev = self.word_emb.device
        ids, pos, seg, cu_seqlens = (t.to(dev) for t in (ids, pos, seg, cu_seqlens))
        key_mask = None if key_mask is None else key_mask.to(dev)
        hd, ad = (self.hidden_dropout, self.attention_dropout) if self.training else (0.0, 0.0)
        x = ops.embedding_layernorm_trainable(ids, pos, seg, self.word_emb, self.pos_emb, self.seg_emb, self.emb_ln_g,
                                              self.emb_ln_b, self.eps, dropout_p=hd)
        for lyr in self.layers:
            h = ops.attention_block_varlen(x, lyr.qkv_w, lyr.qkv_b, lyr.out_w, lyr.out_b, cu_seqlens, max_len,
                                           self.heads, key_mask, attn_dropout=ad, hidden_dropout=hd)
            x = ops.layer_norm_trainable(h, lyr.ln1_g, lyr.ln1_b, self.eps)
            h = ops.gelu_ffn(x, lyr.ffn1_w, lyr.ffn1_b, lyr.ffn2_w, lyr.ffn2_b, dropout_p=hd)
            x = ops.layer_norm_trainable(h, lyr.ln2_g, lyr.ln2_b, self.eps)
        cls = x.index_select(0, cu_seqlens[:-1].long())
        if not self.word_emb.is_cuda:
            pooled = ops.dropout(torch.tanh(F.linear(cls, self.pool_w, self.pool_b)), hd)
            return F.linear(pooled, self.cls_w, self.cls_b)
        bf = torch.bfloat16
        pooled = ops.dropout(torch.tanh(ops.linear_bf16(cls, self.pool_w.to(bf), self.pool_b)), hd)
        n = self.num_labels
        pad = max(CLS_PAD, -(-n // CLS_PAD) * CLS_PAD) - n
        logits = ops.linear_bf16(pooled, F.pad(self.cls_w, (0, 0, 0, pad)).to(bf), F.pad(self.cls_b, (0, pad)))
        return logits[:, :n].float()

    def _forward_dropout_cpu(self, ids, pos, seg, keep, hd, ad):
        """The float32 training forward on CPU with dropout at the documented sites (F.dropout masks)."""
        b, l = ids.shape
        x = ops.embedding_layernorm_trainable(ids, pos, seg, self.word_emb, self.pos_emb, self.seg_emb, self.emb_ln_g,
                                              self.emb_ln_b, self.eps, dropout_p=hd)
        for lyr in self.layers:
            h = ops.attention_block(x, lyr.qkv_w, lyr.qkv_b, lyr.out_w, lyr.out_b, keep, b, l, self.heads,
                                    attn_dropout=ad, hidden_dropout=hd)
            x = ops.layer_norm_trainable(h, lyr.ln1_g, lyr.ln1_b, self.eps)
            h = ops.gelu_ffn(x, lyr.ffn1_w, lyr.ffn1_b, lyr.ffn2_w, lyr.ffn2_b, dropout_p=hd)
            x = ops.layer_norm_trainable(h, lyr.ln2_g, lyr.ln2_b, self.eps)
        pooled = ops.dropout(torch.tanh(F.linear(x.view(b, l, self.hidden)[:, 0], self.pool_w, self.pool_b)), hd)
        return F.linear(pooled, self.cls_w, self.cls_b)


def ernie_base(num_labels=2):
    """ERNIE 1.0 base: vocabulary 18000, hidden 768, 12 layers, 12 heads, FFN 3072, 513 positions, 2 segment types."""
    return ErnieEncoder(18000, 768, 12, 12, 3072, 513, 2, num_labels)


def ernie_student(num_labels=2, dropout=0.0):
    """The Transformer student: the teacher's vocabulary (18000) and feeds, hidden 384, 4 layers, 6 heads, FFN 1536;
    ``dropout`` sets both its hidden and attention dropout (BERT trains with 0.1)."""
    return ErnieStudent(18000, 384, 4, 6, 1536, 513, 2, num_labels, hidden_dropout=dropout, attention_dropout=dropout)


def ernie_tiny(num_labels=2):
    """A 2-layer, 128-wide configuration with the same structure (tests, examples)."""
    return ErnieEncoder(1000, 128, 2, 2, 512, 513, 2, num_labels)
