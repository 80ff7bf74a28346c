"""Fused NHWC BatchNorm (+residual add) (+ReLU), training and inference (csrc/bn.cu).

Replaces the reference's ``batch_norm(act=...)`` + ``elementwise_add(act='relu')`` Paddle ops
(example/distill/resnet/models/resnet_vd.py:167-173,254,276).  Activations are 4-D NCHW-shaped
tensors in ``channels_last`` memory format (i.e. NHWC in memory) or plain 2-D ``[M, C]``.
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn as nn


# SM-resident single-launch BN kernels (bn_fused.cu).  one fused launch
# costs about as much as the two streaming launches it replaces (both are latency- not bandwidth-bound
# at per-GPU batch 32), so the streaming pair stays the default; EDL_FUSED_BN=1 / set_fused_bn(True) enables it.
import os as _os

_FUSED = _os.environ.get("EDL_FUSED_BN", "0") == "1"


def set_fused_bn(enabled: bool) -> None:
    global _FUSED
    _FUSED = bool(enabled)


# ReLU after a residual add keeps its mask as bits (uint8 [M, C/8], written by the streaming apply kernel) instead of
# the bf16 output; a consumer 1x1 dgrad that carries this BN's reduction then stores the gradient already masked, and
# the backward needs neither the mask nor a separate residual gradient.  EDL_RELU_MASK=0 / set_relu_mask(False) saves
# the output as before.
_RELU_MASK = _os.environ.get("EDL_RELU_MASK", "1") == "1"


def set_relu_mask(enabled: bool) -> None:
    global _RELU_MASK
    _RELU_MASK = bool(enabled)


# True while torch.utils.checkpoint re-runs a block's forward during backward: that forward must not update the running
# statistics a second time.  A plain flag, not thread-local: the recompute runs on autograd's device threads.
_RECOMPUTING = False


@contextlib.contextmanager
def _recomputing():
    global _RECOMPUTING
    prev, _RECOMPUTING = _RECOMPUTING, True
    try:
        yield
    finally:
        _RECOMPUTING = prev


def checkpoint_context():
    """``context_fn`` for ``torch.utils.checkpoint.checkpoint(use_reentrant=False)``: the first forward runs as usual,
    the recomputed one leaves every ``BatchNormAct2d``'s running statistics alone."""
    return contextlib.nullcontext(), _recomputing()


def _mc(x: torch.Tensor) -> torch.Tensor:
    """View an activation as a contiguous [M, C] matrix (C fastest)."""
    if x.dim() == 2:
        assert x.is_contiguous()
        return x
    assert x.dim() == 4, "expected NCHW (channels_last) or [M, C]"
    if not x.is_contiguous(memory_format=torch.channels_last):
        x = x.contiguous(memory_format=torch.channels_last)
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1])


def _cl(x: torch.Tensor) -> torch.Tensor:
    if x.dim() == 4 and not x.is_contiguous(memory_format=torch.channels_last):
        return x.contiguous(memory_format=torch.channels_last)
    if x.dim() == 2 and not x.is_contiguous():
        return x.contiguous()
    return x


def _ref_forward(x, res, gamma, beta, rm, rv, relu, training, momentum, eps):
    """fp32 PyTorch reference (CPU path and test oracle)."""
    x2 = _mc(x).float()
    if training:
        mean = x2.mean(0)
        var = x2.var(0, unbiased=False)
        if rm is not None:
            m = x2.shape[0]
            with torch.no_grad():
                rm.mul_(1 - momentum).add_(momentum * mean)
                rv.mul_(1 - momentum).add_(momentum * var * (m / max(m - 1, 1)))
    else:
        mean, var = rm.float(), rv.float()
    rstd = torch.rsqrt(var + eps)
    y = (x2 - mean) * rstd * gamma.float() + beta.float()
    if res is not None:
        y = y + _mc(res).float()
    if relu:
        y = torch.relu(y)
    out = torch.empty_like(x)
    _mc(out).copy_(y.to(x.dtype))
    return out, mean, rstd


class BNBackwardHook:
    """Left by a train-mode BatchNorm on its output tensor (``y._edl_bn_hook``).  The consumer of ``y`` (a
    wgmma 1x1 / 3x3 convolution) computes d(loss)/dy in its dgrad kernel; with this hook that kernel's
    epilogue also accumulates the BN-backward reduction (sum dy_masked, sum dy_masked * xhat) into ``dsums``
    and sets ``done``, and the BN backward then skips its own reduction pass over (dy, x).  ``y`` (bf16 output) or
    ``mask`` (its ReLU mask bits) is set for ReLU after a residual add; with ``mask`` the epilogue stores the gradient
    already multiplied by the mask."""

    __slots__ = ("x", "y", "mask", "mean", "rstd", "gamma", "beta", "relu", "dsums", "done")

    def __init__(self):
        self.x = self.y = self.mask = self.mean = self.rstd = self.gamma = self.beta = self.dsums = None
        self.relu = False
        self.done = False

    def as_list(self, rows, channels):
        assert self.x.numel() == rows * channels
        return [self.x, self.mask if self.mask is not None else self.y, self.mean, self.rstd, self.gamma, self.beta,
                self.dsums]


def drop_bn_hook(t):
    """Call on a BatchNorm output that feeds MORE than one consumer without the fork mechanism of
    ``conv1x1``: no single dgrad kernel sees its complete gradient, so nobody may fuse the reduction."""
    if getattr(t, "_edl_bn_hook", None) is not None:
        t._edl_bn_hook = None
    return t


class _BNActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, res, gamma, beta, rm, rv, sums, ws, sink_g, sink_b, relu, momentum,
                eps, hook=None):
        from . import native, count_launch

        ctx.hook = None

        x = _cl(x)
        res = _cl(res) if res is not None else None
        ctx.relu = relu
        ctx.has_res = res is not None
        sink_g, ctx.ready = sink_g if isinstance(sink_g, tuple) else (sink_g, None)
        ctx.sinks = (sink_g, sink_b)
        # ws = (fwd_stats[2C] | None, bwd_sums[2C] | None, sync int32[2] | None): pre-zeroed arena slices
        fwd_ws, bwd_ws, sync_ws = ws if ws is not None else (None, None, None)
        ctx.bwd_ws, ctx.sync_ws = bwd_ws, sync_ws
        if not x.is_cuda:
            y, mean, rstd = _ref_forward(x, res, gamma, beta, rm, rv, relu, True, momentum, eps)
            ctx.save_for_backward(x, y, gamma, mean, rstd, beta)
            return y
        C = native()
        ch = gamma.numel()
        x2 = _mc(x)
        y = torch.empty_like(x)
        mean = torch.empty(ch, device=x.device, dtype=torch.float32)
        rstd = torch.empty(ch, device=x.device, dtype=torch.float32)
        res2 = _mc(res) if res is not None else None
        mask = None
        if sums is None and _FUSED and C.bn_fused_fits(x2.shape[0], ch, 2 if res is not None else 1):
            # statistics + normalise in ONE SM-resident kernel (tensor crosses HBM once)
            sums = fwd_ws if fwd_ws is not None else torch.zeros(2 * ch, device=x.device, dtype=torch.float32)
            sync = sync_ws[0:1] if sync_ws is not None else torch.zeros(1, device=x.device, dtype=torch.int32)
            C.bn_fwd_fused(x2, res2, _mc(y), sums, gamma, beta, rm, rv, mean, rstd, eps, momentum, relu, sync)
            count_launch()
        else:
            if sums is None:
                sums = fwd_ws if fwd_ws is not None else torch.zeros(2 * ch, device=x.device, dtype=torch.float32)
                C.bn_stats(x2, sums)
                count_launch()
            if relu and res is not None and _RELU_MASK and not _FUSED and C.bn_relu_mask_supported(x2.shape[0], ch):
                mask = torch.empty((x2.shape[0], ch // 8), device=x.device, dtype=torch.uint8)
            C.bn_apply(x2, res2, _mc(y), sums, gamma, beta, rm, rv, mean, rstd, eps, momentum, relu, mask)
            count_launch()
        # the ReLU mask is only needed when a residual was added (otherwise the backward kernels recompute it from x):
        # the mask bits when the apply kernel wrote them, else the saved output
        y_saved = y if (relu and res is not None and mask is None) else None
        ctx.save_for_backward(x, mask if mask is not None else y_saved, gamma, mean, rstd, beta)
        if hook is not None:
            # let the consumer's dgrad kernel carry this layer's backward reduction
            if bwd_ws is None:
                bwd_ws = ctx.bwd_ws = torch.zeros(2 * ch, device=x.device, dtype=torch.float32)
            hook.x, hook.y, hook.mask = x, y_saved, mask
            hook.mean, hook.rstd, hook.gamma, hook.beta = mean, rstd, gamma, beta
            hook.relu, hook.dsums = relu, bwd_ws
            ctx.hook = hook
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        x, y, gamma, mean, rstd, beta = ctx.saved_tensors
        relu, has_res = ctx.relu, ctx.has_res
        sink_g, sink_b = ctx.sinks
        dy = _cl(dy)
        if not x.is_cuda:
            x2, dy2 = _mc(x).float(), _mc(dy).float()
            if relu:
                dy2 = dy2 * (_mc(y).float() > 0)
            xhat = (x2 - mean) * rstd
            db = dy2.sum(0)
            dg = (dy2 * xhat).sum(0)
            m = x2.shape[0]
            dx2 = gamma.float() * rstd * (dy2 - db / m - xhat * dg / m)
            dx = torch.empty_like(x)
            _mc(dx).copy_(dx2.to(x.dtype))
            dres = None
            if has_res:
                dres = torch.empty_like(x)
                _mc(dres).copy_(dy2.to(x.dtype))
            dgo, dbo = dg.to(gamma.dtype), db.to(gamma.dtype)
            if sink_g is not None:
                sink_g.add_(dgo)
                sink_b.add_(dbo)
                dgo = dbo = None
                if ctx.ready is not None:
                    ctx.ready()
            return dx, dres, dgo, dbo, None, None, None, None, None, None, None, None, None, None
        C = native()
        ch = gamma.numel()
        dsums = ctx.bwd_ws
        if dsums is None:
            dsums = torch.zeros(2 * ch, device=x.device, dtype=torch.float32)
        x2, dy2 = _mc(x), _mc(dy)
        # y: the bf16 output, or the uint8 ReLU mask bits [M, C/8] (which the kernels take in its place)
        is_mask = y is not None and y.dtype == torch.uint8
        y2 = (y if is_mask else _mc(y)) if (relu and y is not None) else None
        # the consumer's dgrad epilogue reduced dy AND stored it multiplied by the mask: dy is the residual gradient
        premasked = is_mask and ctx.hook is not None and ctx.hook.done
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if (has_res and not premasked) else None
        if sink_g is not None:
            dg, db, acc = sink_g, sink_b, True
        else:
            dg = torch.empty_like(gamma)
            db = torch.empty_like(gamma)
            acc = False
        if premasked:
            count_launch(1)
            C.bn_bwd_apply(dy2, x2, None, gamma, beta, mean, rstd, dsums, _mc(dx), None, dg, db, False, acc)
            # dres aliases dy.  Whatever later adds into this buffer in place (autograd accumulating gradients) runs
            # on this stream after the kernel just enqueued, which has then read dy.
            dres = dy if has_res else None
        elif _FUSED and not is_mask and C.bn_fused_fits(x2.shape[0], ch, 3 if y2 is not None else 2):
            sync = ctx.sync_ws[1:2] if ctx.sync_ws is not None else torch.zeros(1, device=x.device,
                                                                               dtype=torch.int32)
            C.bn_bwd_fused(dy2, x2, y2, gamma, beta, mean, rstd, dsums, _mc(dx),
                           _mc(dres) if has_res else None, dg, db, relu, acc, sync)
            count_launch()
        else:
            if ctx.hook is not None and ctx.hook.done:
                count_launch(1)      # the reduction already rode in the consumer's dgrad epilogue
            else:
                C.bn_bwd_reduce(dy2, x2, y2, gamma, beta, mean, rstd, dsums, relu)
                count_launch(2)
            C.bn_bwd_apply(dy2, x2, y2, gamma, beta, mean, rstd, dsums, _mc(dx),
                           _mc(dres) if has_res else None, dg, db, relu, acc)
        if sink_g is not None:
            dg = db = None
            if ctx.ready is not None:
                ctx.ready()
        return dx, dres, dg, db, None, None, None, None, None, None, None, None, None, None


def batch_norm_act(x, gamma, beta, running_mean=None, running_var=None, residual=None, relu=False,
                   training=True, momentum=0.1, eps=1e-5, sums=None, bwd_ws=None, sinks=None, ws=None):
    """y = act(BN(x) (+ residual)).  ``sums`` may carry per-channel (sum, sum^2) already produced
    by the conv/GEMM epilogue; ``bwd_ws`` is an optional pre-zeroed [2C] fp32 scratch; ``sinks`` is
    an optional ``(dgamma_view, dbeta_view[, ready_callback])`` tuple: the backward accumulates the
    parameter gradients straight into those views (flat gradient buckets) and then calls the callback."""
    if not training:
        scale = gamma.float() * torch.rsqrt(running_var.float() + eps)
        shift = beta.float() - running_mean.float() * scale
        return scale_shift_act(x, scale, shift, residual, relu)
    sink_g, sink_b, ready = (tuple(sinks) + (None,))[:3] if sinks is not None else (None, None, None)
    if ws is None and bwd_ws is not None:
        ws = (None, bwd_ws, None)
    hook = BNBackwardHook() if (x.is_cuda and x.dtype == torch.bfloat16 and torch.is_grad_enabled() and not _FUSED) else None
    y = _BNActFn.apply(x, residual, gamma, beta, running_mean, running_var, sums, ws,
                       (sink_g, ready), sink_b, relu, momentum, eps, hook)
    if hook is not None and hook.x is not None:
        y._edl_bn_hook = hook
    return y


def bn_stats_into(x, sums):
    """Accumulate per-channel (sum, sum^2) of ``x`` into the pre-zeroed fp32 ``sums`` [2C]."""
    from . import native, count_launch

    x = _cl(x)
    if x.is_cuda:
        native().bn_stats(_mc(x), sums)
        count_launch()
    else:
        x2 = _mc(x).float()
        c = x2.shape[1]
        sums[:c] += x2.sum(0)
        sums[c:] += (x2 * x2).sum(0)
    return sums


def scale_shift_act(x, scale, shift, residual=None, relu=False):
    """Inference-form folded BN: y = act(x * scale[c] + shift[c] (+ residual)); no autograd."""
    from . import native, count_launch

    x = _cl(x)
    if not x.is_cuda:
        y = _mc(x).float() * scale.float() + shift.float()
        if residual is not None:
            y = y + _mc(_cl(residual)).float()
        if relu:
            y = torch.relu(y)
        out = torch.empty_like(x)
        _mc(out).copy_(y.to(x.dtype))
        return out
    out = torch.empty_like(x)
    native().scale_shift_act(_mc(x), _mc(_cl(residual)) if residual is not None else None, _mc(out),
                             scale.float().contiguous(), shift.float().contiguous(), relu)
    count_launch()
    return out


class BatchNormAct2d(nn.Module):
    """BatchNorm2d with the activation (and an optional residual add) fused into the same kernels.

    Parameters are kept in fp32 (like AMP master copies); activations are bf16 channels_last."""

    def __init__(self, num_features, relu=False, momentum=0.1, eps=1e-5):
        super().__init__()
        self.num_features = num_features
        self.relu = relu
        self.momentum = momentum
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(num_features, dtype=torch.float32))
        self.bias = nn.Parameter(torch.zeros(num_features, dtype=torch.float32))
        self.register_buffer("running_mean", torch.zeros(num_features, dtype=torch.float32))
        self.register_buffer("running_var", torch.ones(num_features, dtype=torch.float32))
        self.ws = None      # optional (fwd_stats, bwd_sums, sync) arena slices, see trainer.StepArena

    def _sinks(self):
        sg = getattr(self.weight, "_edl_grad_sink", None)
        sb = getattr(self.bias, "_edl_grad_sink", None)
        if sg is None or sb is None or not torch.is_grad_enabled():
            return None
        cbs = [getattr(p, "_edl_grad_ready", None) for p in (self.weight, self.bias)]
        cbs = [c for c in cbs if c is not None]
        return sg, sb, (lambda: [c() for c in cbs]) if cbs else None

    def forward(self, x, residual=None, sums=None):
        # the kernels skip the running-statistics update when they get none (a recomputed forward)
        rm, rv = (None, None) if _RECOMPUTING else (self.running_mean, self.running_var)
        return batch_norm_act(x, self.weight, self.bias, rm, rv,
                              residual=residual, relu=self.relu, training=self.training,
                              momentum=self.momentum, eps=self.eps, sums=sums, ws=self.ws,
                              sinks=self._sinks())

    def extra_repr(self):
        return "%d, relu=%s, eps=%g, momentum=%g" % (self.num_features, self.relu, self.eps,
                                                     self.momentum)
