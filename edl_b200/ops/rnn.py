"""Bidirectional LSTM layer on the recurrence kernels of csrc/lstm.cu (the BiLSTM student of the NLP distillation).

``lstm(x, lengths, params)`` has the semantics of ``torch.nn.LSTM(batch_first=True, bidirectional=True)`` with one
layer, run on right-padded sequences through ``pack_padded_sequence(..., enforce_sorted=False)``: past a sample's
length its state is not updated, its output is 0 and no gradient flows; a sample of length 0 gives zeros everywhere.

On CUDA (H = 128, E % 8 == 0) the work is:
  forward   xproj = X W_ih^T + (b_ih + b_hh) for both directions as one ``gemm_bf16`` (rows of W_ih in the kernel's
            thread order), then one persistent recurrence launch for the whole sequence;
  backward  one recurrence launch that writes dgates, then dX = [dgates_f | dgates_r] [W_ih_f ; W_ih_r] as one
            ``gemm_bf16`` with K = 8H, dW_ih and dW_hh through ``_wgrad`` (the side-stream weight-gradient hand-off),
            and the bias gradient as a column sum of dgates.
Everything is time-major inside (row t * B + b): with one zero block before and after the hidden states, h_{t-1} of
both directions is a plain view, so dW_hh needs no new GEMM.  ``y`` is returned as a [B, L, 2H] view of that buffer.
Nothing reads the lengths back to the host, so a step can be captured in a CUDA graph.

CPU tensors run ``lstm_reference``, an fp32 loop over time with the same semantics (autograd included); CUDA shapes
the kernels do not take run the same reference through ``count_fallback``."""
from __future__ import annotations

import torch

from .gemm import _grad_sink, _wgrad, gemm_bf16

HIDDEN = 128


def _count(reason):
    from . import count_fallback

    count_fallback(reason)


# ---------------------------------------------------------------------------------------------------------- reference
def _run_direction(xp, lengths, w_hh, reverse):
    """One direction over the pre-projected inputs ``xp`` [B, L, 4H]: returns (out [B, L, H], h_n [B, H])."""
    b, L, _ = xp.shape
    h = xp.new_zeros(b, w_hh.shape[1])
    c = torch.zeros_like(h)
    ar = torch.arange(b, device=xp.device)
    outs = []
    for s in range(L):
        active = (s < lengths).unsqueeze(1)
        t = (lengths - 1 - s).clamp(min=0) if reverse else torch.full_like(lengths, s)
        g = xp[ar, t] + h @ w_hh.t()
        i, f, gg, o = g.chunk(4, 1)
        cn = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        hn = torch.sigmoid(o) * torch.tanh(cn)
        c = torch.where(active, cn, c)
        h = torch.where(active, hn, h)
        outs.append(torch.where(active, hn, torch.zeros_like(hn)))
    out = torch.stack(outs, 1)                                  # step-major: out[:, s] belongs to t(s)
    if reverse:
        tt = torch.arange(L, device=xp.device)
        src = (lengths.unsqueeze(1) - 1 - tt).clamp(min=0)      # time t was computed at step len - 1 - t
        out = torch.gather(out, 1, src.unsqueeze(2).expand(-1, -1, out.shape[2]))
        out = torch.where((tt < lengths.unsqueeze(1)).unsqueeze(2), out, torch.zeros_like(out))
    return out, h


def lstm_reference(x, lengths, params):
    """fp32 math of ``lstm``: (y [B, L, 2H], h_n [2, B, H]) in x's dtype, differentiable by autograd."""
    xf = x.float()
    L = x.shape[1]
    lengths = lengths.to(x.device, torch.long).clamp(0, L)
    ys, hs = [], []
    for d in range(2):
        w_ih, w_hh, b_ih, b_hh = (p.float() for p in params[4 * d:4 * d + 4])
        xp = xf @ w_ih.t() + (b_ih + b_hh)
        # padded rows are never selected, but keep their (possibly non-finite) values out of the arithmetic
        xp = torch.where((torch.arange(L, device=x.device) < lengths.unsqueeze(1)).unsqueeze(2), xp,
                         torch.zeros_like(xp))
        y, h = _run_direction(xp, lengths, w_hh, d == 1)
        ys.append(y)
        hs.append(h)
    return torch.cat(ys, 2).to(x.dtype), torch.stack(hs, 0).to(x.dtype)


# ------------------------------------------------------------------------------------------------------------- kernels
def lstm_supported(x, params) -> bool:
    from . import native

    if not (x.is_cuda and x.dim() == 3 and params[1].shape == (4 * HIDDEN, HIDDEN)):
        return False
    b, L, e = x.shape
    return params[0].shape == (4 * HIDDEN, e) and native().lstm_supported(b, L, e, HIDDEN)


def _thread_order(h, device):
    """Row permutation of a [4H, *] gate matrix into the kernel's xproj column order (csrc/lstm.cu): column
    w * 256 + q * 64 + 4m + gate is gate ``gate`` of unit 64w + 4m + q."""
    c = torch.arange(4 * h, device=device)
    w, q, m, gate = c // 256, (c // 64) % 4, (c // 4) % 16, c % 4
    return gate * h + 64 * w + 4 * m + q


def lstm_forward_saved(x, lengths, params):
    """The kernel path's forward with everything it keeps: returns (hs, hn, gates, cs, xt, lengths32, whh) in the layouts
    of csrc/lstm.cu (``xt`` is X time-major [L * B, E] bf16, ``whh`` the bf16 [2, 4H, H] recurrent weights)."""
    from . import native, count_launch

    b, L, e = x.shape
    dev = x.device
    perm = _thread_order(HIDDEN, dev)
    xt = x.detach().to(torch.bfloat16).transpose(0, 1).reshape(L * b, e)
    w_cat = torch.cat([params[0].detach()[perm], params[4].detach()[perm]], 0).to(torch.bfloat16).contiguous()
    bias = torch.cat([(params[2].detach().float() + params[3].detach().float())[perm],
                      (params[6].detach().float() + params[7].detach().float())[perm]])
    xproj = gemm_bf16(xt, w_cat, col_shift=bias)
    whh = torch.stack([params[1].detach(), params[5].detach()]).to(torch.bfloat16).contiguous()
    len32 = lengths.detach().to(dev, torch.int32).contiguous()
    hs = torch.empty(((L + 2) * b, 2 * HIDDEN), device=dev, dtype=torch.bfloat16)
    hn = torch.empty((2, b, HIDDEN), device=dev, dtype=torch.bfloat16)
    gates = torch.empty((L * b, 2, HIDDEN, 4), device=dev, dtype=torch.bfloat16)
    cs = torch.empty((L * b, 2, HIDDEN), device=dev, dtype=torch.float32)
    native().lstm_fwd(xproj, whh, len32, hs, hn, gates, cs, L)
    count_launch()
    return hs, hn, gates, cs, xt, len32, whh, xproj


def lstm_backward_dgates(whh, len32, gates, cs, dy, dhn, L):
    """The backward recurrence: dgates bf16 [L * B, 8H] (time-major, nn.LSTM row order per direction)."""
    from . import native, count_launch

    b = len32.numel()
    dgates = torch.empty((L * b, 8 * HIDDEN), device=whh.device, dtype=torch.bfloat16)
    native().lstm_bwd(whh, len32, gates, cs, dy, dhn, dgates, L)
    count_launch()
    return dgates


class _LstmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, lengths, sinks, *params):
        b, L, e = x.shape
        hs, hn, gates, cs, xt, len32, whh, _ = lstm_forward_saved(x, lengths, params)
        ctx.save_for_backward(hs, gates, cs, xt, len32, whh, *params)
        ctx.shape, ctx.x_dtype = (b, L, e), x.dtype
        ctx.sinks = sinks
        y = hs[b:(L + 1) * b].view(L, b, 2 * HIDDEN).transpose(0, 1)
        return y.to(x.dtype), hn.to(x.dtype)

    @staticmethod
    def backward(ctx, dy, dhn):
        hs, gates, cs, xt, len32, whh, *params = ctx.saved_tensors
        b, L, e = ctx.shape
        H = HIDDEN
        if dy is not None:
            dy = dy.to(torch.bfloat16)
            if dy.stride(-1) != 1 or dy.stride(0) % 2 or dy.stride(1) % 2 or dy.data_ptr() % 4:
                dy = dy.contiguous()
        if dhn is not None:
            dhn = dhn.to(torch.bfloat16).contiguous()
        dg = lstm_backward_dgates(whh, len32, gates, cs, dy, dhn, L)
        dx = None
        if ctx.needs_input_grad[0]:
            w_cat = torch.cat([params[0], params[4]], 0).to(torch.bfloat16).contiguous()      # [8H, E]
            dx = gemm_bf16(dg, w_cat, b_mn_major=True).view(L, b, e).transpose(0, 1).to(ctx.x_dtype)
        grads = [None] * 8
        db = None
        for d in range(2):
            dgd = dg[:, 4 * H * d:4 * H * (d + 1)]
            w_ih, w_hh, b_ih, b_hh = params[4 * d:4 * d + 4]
            (s_ih, r_ih), (s_hh, r_hh) = ctx.sinks[4 * d], ctx.sinks[4 * d + 1]
            if ctx.needs_input_grad[3 + 4 * d]:
                g = _wgrad(dgd, xt, w_ih.shape, s_ih, r_ih)
                grads[4 * d] = None if g is None else g.to(w_ih.dtype)
            if ctx.needs_input_grad[4 + 4 * d]:
                hprev = hs[2 * b * d:2 * b * d + L * b, H * d:H * (d + 1)]      # h_{t-1} (forward), h_{t+1} (reverse)
                g = _wgrad(dgd, hprev, w_hh.shape, s_hh, r_hh)
                grads[4 * d + 1] = None if g is None else g.to(w_hh.dtype)
            if ctx.needs_input_grad[5 + 4 * d] or ctx.needs_input_grad[6 + 4 * d]:
                if db is None:
                    db = dg.float().sum(0)
                dbd = db[4 * H * d:4 * H * (d + 1)]
                for k, p in ((2, b_ih), (3, b_hh)):
                    if not ctx.needs_input_grad[3 + 4 * d + k]:
                        continue
                    sink, ready = ctx.sinks[4 * d + k]
                    if sink is not None:
                        sink.add_(dbd)
                        if ready is not None:
                            ready()
                    else:
                        grads[4 * d + k] = dbd.to(p.dtype)
        return (dx, None, None, *grads)


def lstm(x, lengths, params):
    """Bidirectional single-layer LSTM over right-padded sequences.

    ``x`` [B, L, E] (bf16 on CUDA), ``lengths`` integer [B] on x's device (clamped to [0, L]), ``params`` the eight
    tensors of a bidirectional ``nn.LSTM`` layer in its order and layout (weight_ih_l0, weight_hh_l0, bias_ih_l0,
    bias_hh_l0, then the _reverse set; any float dtype).  Returns (y [B, L, 2H], h_n [2, B, H]) in x's dtype; gradients
    come back in the parameters' dtype."""
    params = tuple(params)
    if len(params) != 8:
        raise ValueError("lstm: expected the 8 parameters of a bidirectional nn.LSTM layer, got %d" % len(params))
    if not x.is_cuda:
        return lstm_reference(x, lengths, params)
    if not lstm_supported(x, params):
        _count("lstm: no kernel for x %s %s, hidden %d (H = 128, E % 8 == 0): float32 loop on the library"
               % (tuple(x.shape), x.dtype, params[1].shape[1]))
        return lstm_reference(x, lengths, params)
    return _LstmFn.apply(x, lengths, tuple(_grad_sink(p) for p in params), *params)
