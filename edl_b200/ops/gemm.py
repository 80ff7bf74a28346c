"""wgmma GEMM front-end (csrc/gemm.cu): plain GEMM, Linear and NHWC 1x1 convolution with the
train-mode BatchNorm statistics fused into the GEMM epilogue.

Reference call sites are library ops: ``fluid.layers.conv2d`` (cuDNN) and ``fluid.layers.fc``
(cuBLAS) in example/distill/resnet/models/resnet_vd.py:153-162,135-141."""
from __future__ import annotations

from typing import Optional

import torch

from .bn import _cl

_NUM_SMS = 132


def gemm_bf16(a, b, out=None, a_mn_major=False, b_mn_major=False, col_scale=None, col_shift=None,
              relu=False, col_stats=None, add=None, bn=None, gelu=False):
    """D = op(A) @ op(B): see csrc/gemm.h for the operand conventions.  The weight-gradient form (both operands
    MN-major) is ``_wgrad_impl``.

    default        : A [M, K], B [N, K]  -> D [M, N] = A @ B^T
    b_mn_major     : B [K, N]            -> D = A @ B
    a_mn_major     : A [K, M]            -> D = A^T @ op(B)
    add given      : D = result + add (bf16 [M, N]) in the epilogue (gradient accumulation fused into dgrad).
    bn given       : a ``BNBackwardHook`` (ops/bn.py): D is the gradient of that BatchNorm's output and the
                     epilogue accumulates its backward reduction (sum dy, sum dy * xhat) into hook.dsums.
    gelu           : D = gelu(A @ B^T * col_scale + col_shift) with the erf form in fp32 (inference; both operands
                     K-major, no addend / ReLU / statistics)."""
    from . import native, count_launch

    if gelu and (a_mn_major or b_mn_major or add is not None or relu or col_stats is not None or bn is not None):
        raise ValueError("gemm_bf16: the GELU epilogue is a forward GEMM with an optional scale / shift only")
    if gelu and a.is_cuda and _tma_compatible(a, b, out, b.shape[0]) and not native().persistent_gemm_enabled():
        from . import count_fallback
        count_fallback("gemm_bf16: the GELU epilogue needs the persistent GEMM (disabled): fp32 matmul on the library")
        return _gemm_reference(a, b, out, False, False, col_scale, col_shift, False, None, None, True)
    m = a.shape[1] if a_mn_major else a.shape[0]
    n = b.shape[1] if b_mn_major else b.shape[0]
    if not a.is_cuda or not _tma_compatible(a, b, out, n):
        # CPU tensors, or CUDA shapes TMA cannot describe (row pitch / base not 16-byte aligned):
        # plain PyTorch math with identical semantics -- counted and logged when it happens on a GPU
        if a.is_cuda:
            from . import count_fallback
            count_fallback("gemm_bf16: operand not TMA-describable (pitch / base not 16-byte aligned or not bf16): "
                           "fp32 matmul on the library, %s x %s" % (tuple(a.shape), tuple(b.shape)))
        return _gemm_reference(a, b, out, a_mn_major, b_mn_major, col_scale, col_shift, relu, col_stats, add, gelu)
    if out is None:
        out = torch.empty((m, n), device=a.device, dtype=torch.bfloat16)
    if gelu:
        native().gemm_bf16_gelu(a, b, out, col_scale, col_shift)
        count_launch()
        return out
    if add is not None and not (native().persistent_gemm_enabled() and n % 8 == 0 and add.stride(-1) == 1
                                and add.stride(0) % 8 == 0 and add.data_ptr() % 16 == 0):
        # the fused addend lives in the persistent kernel's epilogue; otherwise one extra elementwise pass, which is
        # only the same operation when nothing follows the addition in the epilogue
        if col_scale is not None or col_shift is not None or relu or col_stats is not None:
            raise RuntimeError("gemm_bf16: an addend together with scale / shift / ReLU / statistics needs the persistent "
                               "kernel's fused addend (persistent GEMM on, N % 8 == 0, 16-byte aligned addend rows)")
        native().gemm_bf16(a, b, out, a_mn_major, b_mn_major, col_scale, col_shift, relu, col_stats, None, None, False)
        count_launch()
        out.add_(add)
        return out
    bn_list, bn_relu = (bn.as_list(m, n), bn.relu) if bn is not None else (None, False)
    native().gemm_bf16(a, b, out, a_mn_major, b_mn_major, col_scale, col_shift, relu, col_stats, add, bn_list, bn_relu)
    count_launch()
    if bn is not None:
        bn.done = True
    return out


def _gemm_reference(a, b, out, a_mn_major, b_mn_major, col_scale, col_shift, relu, col_stats, add, gelu):
    """gemm_bf16's semantics in fp32 PyTorch math (CPU tensors, shapes TMA cannot describe)."""
    n = b.shape[1] if b_mn_major else b.shape[0]
    af = a.float().t() if a_mn_major else a.float()
    bf = b.float() if b_mn_major else b.float().t()
    d = af @ bf
    if add is not None:
        d = d + add.float()
    if col_scale is not None:
        d = d * col_scale.float()
    if col_shift is not None:
        d = d + col_shift.float()
    if relu:
        d = torch.relu(d)
    if gelu:
        d = torch.nn.functional.gelu(d)
    d = d.to(torch.bfloat16)
    if col_stats is not None:
        col_stats[:n] += d.float().sum(0)
        col_stats[n:] += (d.float() ** 2).sum(0)
    if out is not None:
        out.copy_(d)
        return out
    return d


def _tma_compatible(a, b, out, n):
    for t in (a, b, out):
        if t is None:
            continue
        if t.dtype != torch.bfloat16 or t.stride(-1) != 1 or t.stride(0) % 8 != 0 or t.data_ptr() % 16 != 0:
            return False
    return out is not None or n % 8 == 0


def _split_k_for(m, n, k):
    """Split-K factor of the wgrad GEMM.  The split is chosen to fill ~one wave of SMs and never more: outputs
    with >= 132 tiles are not split at all (direct bf16 store), tiny outputs (stage-2 layers, 1-8
    tiles with K ~ 100k) take the full 132-way split because they have few elements to update."""
    tiles = ((m + 127) // 128) * ((n + 127) // 128 if n > 64 else 1)
    kb = (k + 63) // 64
    if tiles >= 48:
        # a third of the SMs already have a tile: no split, hence no partial tiles and no reduce kernel.  The weight
        # gradients run on the low-priority side stream and are not the critical path: a kernel that keeps 48-147 SMs
        # busy a little longer leaves the other SMs to the dgrad / BatchNorm chain, which is what limits the step
        return 1
    want = max(1, _NUM_SMS // tiles)
    return max(1, min(want, max(1, kb // 2)))


_SIDE = {"streams": [], "next": 0, "keep": []}


def set_wgrad_stream(streams):
    """Run the weight gradients that go into a gradient sink on ``streams`` (a list; the DP engine passes its
    weight-gradient streams): they then overlap the dgrad / BN-backward chain of the main stream.  ``None``
    disables the overlap."""
    _SIDE["streams"] = [st for st in streams or () if st is not None]
    _SIDE["next"] = 0
    _SIDE["keep"].clear()


def _side_stream():
    """The next weight-gradient stream (round-robin over the engine's side streams): consecutive layers' weight
    gradients are independent, two of them in flight shorten the side-stream tail that remains after the last
    dgrad of backward."""
    sts = _SIDE["streams"]
    if not sts:
        return None
    st = sts[_SIDE["next"] % len(sts)]
    _SIDE["next"] += 1
    return st


def release_wgrad_keepalive():
    """Drop the references that kept side-stream operands alive (call after the streams were joined)."""
    _SIDE["keep"].clear()



# TIMING EXPERIMENT ONLY (never set in a real run: the model does not learn): EDL_DEBUG_SKIP_WGRAD=1 drops every
# weight-gradient kernel of the wgmma / library conv paths, which bounds what faster wgrad kernels could buy.
_SKIP_WGRAD = __import__("os").environ.get("EDL_DEBUG_SKIP_WGRAD", "0") == "1"


_PART = {}
_STEM_SCRATCH = {}


def _splitk_partials(device, numel):
    """Per (device, stream) scratch of at least ``numel`` fp32 for the split-K partial tiles (csrc/gemm.h
    GemmArgs::partials).  It starts at 64 MB, more than the ResNet50_vd weight gradients at batch 32 need, so a
    training step never grows it; a larger request replaces it."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _PART.get(key)
    if buf is None or buf.numel() < numel:
        buf = _PART[key] = torch.empty(max(numel, 16 << 20), device=device, dtype=torch.float32)
    return buf


def _stem_scratch(device):
    """Per (device, stream) all-zero fp32 [1024] + int32 [1] of the stem weight gradient's in-kernel reduction
    (csrc/stem.cu), which leaves both zeroed again."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _STEM_SCRATCH.get(key)
    if buf is None:
        buf = _STEM_SCRATCH[key] = (torch.zeros(1024, device=device, dtype=torch.float32),
                                    torch.zeros(1, device=device, dtype=torch.int32))
    return buf


def _grad_sink(param):
    """``(sink, ready)`` of a parameter whose gradient goes straight into its window of the flat gradient bucket
    (parallel/flat.py) instead of ``param.grad``; ``(None, None)`` for any other parameter and outside autograd."""
    sink = getattr(param, "_edl_grad_sink", None) if torch.is_grad_enabled() else None
    return sink, (getattr(param, "_edl_grad_ready", None) if sink is not None else None)


def _deliver_wgrad(dy, x, sink, ready, compute):
    """One layer's weight gradient: ``compute(sink)`` adds it into ``sink``, ``compute(None)`` returns it.

    Without a sink it is computed here and returned to autograd.  With one it runs on the next weight-gradient
    stream, behind the work already queued on the current stream, ``ready()`` is called with that stream still
    current and None is returned; ``dy`` and ``x`` stay referenced until the engine has joined the streams
    (``release_wgrad_keepalive``)."""
    if sink is None:
        return compute(None)
    if _SKIP_WGRAD:
        if ready is not None:
            ready()
        return None
    side = _side_stream() if dy.is_cuda else None
    if side is not None:
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dy.device))
        side.wait_event(ev)
        _SIDE["keep"].append((dy, x))
    with torch.cuda.stream(side):        # None: stay on the current stream
        compute(sink)
        if ready is not None:
            ready()
    return None


def _wgrad(dy2, x2, weight_shape, sink, ready):
    """dW[Cout, Cin] = dy2[M, Cout]^T @ x2[M, Cin], written as bf16 straight into the (flat gradient bucket) sink --
    no memset / cast / add kernels around it."""
    return _deliver_wgrad(dy2, x2, sink, ready, lambda s: _wgrad_impl(dy2, x2, weight_shape, s))


def _wgrad_impl(dy2, x2, weight_shape, sink, split_k: Optional[int] = None):
    from . import native, count_launch

    cout, cin = dy2.shape[1], x2.shape[1]
    if dy2.is_cuda and _tma_compatible(dy2, x2, None, cin):
        split = split_k if split_k is not None else _split_k_for(cout, cin, dy2.shape[0])
        out = sink.view(cout, cin) if sink is not None else torch.empty((cout, cin), device=dy2.device,
                                                                        dtype=torch.bfloat16)
        block_n = 64 if cin <= 64 else 128      # the kernel's tile width (csrc/gemm.cu)
        tiles = ((cout + 127) // 128) * ((cin + block_n - 1) // block_n)
        partials = _splitk_partials(dy2.device, split * tiles * 128 * block_n) if split > 1 else None
        native().gemm_wgrad_bf16(dy2, x2, out, split, sink is not None, partials)
        count_launch()
        return None if sink is not None else out.view(weight_shape)
    if dy2.is_cuda:
        from . import count_fallback
        count_fallback("gemm_bf16: operand not TMA-describable (pitch / base not 16-byte aligned or not bf16): "
                       "fp32 matmul on the library, %s x %s" % (tuple(dy2.shape), tuple(x2.shape)))
    d = dy2.float().t() @ x2.float()
    if sink is None:
        return d.to(torch.bfloat16).view(weight_shape)
    sink.view(cout, cin).add_(d)


class _Conv1x1Fn(torch.autograd.Function):
    """``fork=True`` also returns the input as a second output: a tensor that feeds this convolution AND a
    second consumer (the residual branch) then receives ONE gradient, summed inside the dgrad epilogue,
    instead of two gradients that autograd adds with an extra elementwise kernel."""

    @staticmethod
    def forward(ctx, x, w, stats, sink, ready, fork=False, bn_hook=None):
        ctx.bn_hook = bn_hook
        x = _cl(x)
        n, cin, h, wd = x.shape
        cout = w.shape[0]
        x2 = x.permute(0, 2, 3, 1).reshape(-1, cin)
        w2 = w.reshape(cout, cin)
        y = torch.empty((n, cout, h, wd), device=x.device, dtype=x.dtype,
                        memory_format=torch.channels_last)
        y2 = y.permute(0, 2, 3, 1).reshape(-1, cout)
        gemm_bf16(x2, w2, out=y2, col_stats=stats)
        ctx.save_for_backward(x, w)
        ctx.sink, ctx.ready = sink, ready
        if fork:
            return y, x.view_as(x)
        return y

    @staticmethod
    def backward(ctx, dy, dfork=None):
        x, w = ctx.saved_tensors
        if dy is None:      # only the forked alias was used downstream
            return dfork, None, None, None, None, None, None
        dy = _cl(dy)
        n, cin, h, wd = x.shape
        cout = w.shape[0]
        dy2 = dy.permute(0, 2, 3, 1).reshape(-1, cout)
        x2 = x.permute(0, 2, 3, 1).reshape(-1, cin)
        w2 = w.reshape(cout, cin)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            add = None
            if dfork is not None:
                add = _cl(dfork).permute(0, 2, 3, 1).reshape(-1, cin)
            # dx is the gradient of the BatchNorm output that fed this conv: its backward reduction
            # rides in this epilogue when the producing BN left a hook on the tensor
            hook = ctx.bn_hook if _bn_fusable(ctx.bn_hook, x, cin) else None
            gemm_bf16(dy2, w2, out=dx.permute(0, 2, 3, 1).reshape(-1, cin), b_mn_major=True, add=add, bn=hook)
        dw = _wgrad(dy2, x2, w.shape, ctx.sink, ctx.ready) if ctx.needs_input_grad[1] else None
        return dx, dw, None, None, None, None, None


def conv1x1(x, weight, stats: Optional[torch.Tensor] = None, fork: bool = False):
    """NHWC 1x1 stride-1 convolution as a wgmma GEMM.  ``weight``: [Cout, 1, 1, Cin] or
    [Cout, Cin] bf16.  If ``stats`` (pre-zeroed fp32 [2*Cout]) is given, the epilogue accumulates
    per-channel sum / sum-of-squares of the output for the following train-mode BatchNorm."""
    return _Conv1x1Fn.apply(x, weight, stats, *_grad_sink(weight), fork, getattr(x, "_edl_bn_hook", None))


def _bn_fusable(hook, x, channels) -> bool:
    """The consumer's dgrad may carry the BN-backward reduction iff the hook belongs to exactly this input,
    the persistent kernels are on and the layout is what the fused epilogue expects."""
    from . import native

    return (hook is not None and FUSE_BN_BWD and not hook.done and x.is_cuda and hook.x.shape == x.shape
            and channels % 8 == 0 and native().persistent_gemm_enabled()
            and x.numel() * x.element_size() <= FUSE_BN_BWD_MAX_BYTES)


# ON by default (EDL_FUSE_BN_BWD=0 turns it off): the BatchNorm-backward reduction of a conv's input
# gradient rides in that conv's dgrad epilogue as a column-pair loop over the staged tiles (csrc/gemm_persist.cu).
# Validated at kernel level and at model level against the stand-alone reduction kernels with
# the run-to-run atomics noise as yardstick (tests/test_persist_gpu.py); removes 44 bn_bwd_reduce launches per
# ResNet50_vd step.
FUSE_BN_BWD = __import__("os").environ.get("EDL_FUSE_BN_BWD", "1") == "1"
# Upper bound on the activation size for which the reduction is fused (EDL_FUSE_BN_BWD_MAX_MB).  The fused epilogue
# prefetches the BN input / output tiles of ONE tile ahead (64 KB per SM in flight), which is latency-bound on the
# largest activations (51 MB at 56 x 56 x 256 x 32); the stand-alone streaming
# reduction reads them at full bandwidth.
FUSE_BN_BWD_MAX_BYTES = float(__import__("os").environ.get("EDL_FUSE_BN_BWD_MAX_MB", "1e9")) * (1 << 20)


class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias, relu, sink, ready, bias_sink, bias_ready):
        x = x.contiguous()
        y = gemm_bf16(x, w, col_shift=bias.float() if bias is not None else None, relu=relu)
        ctx.save_for_backward(x, w, y if relu else None)
        ctx.has_bias = bias is not None
        ctx.bias_dtype = bias.dtype if bias is not None else None
        ctx.sink, ctx.ready = sink, ready
        ctx.bias_sink, ctx.bias_ready = bias_sink, bias_ready
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        dy = dy.contiguous()
        if y is not None:
            dy = dy * (y > 0)
        dx = gemm_bf16(dy, w, b_mn_major=True) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            dw = _wgrad(dy, x, w.shape, ctx.sink, ctx.ready)
        db = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.float().sum(0).to(ctx.bias_dtype)
            if ctx.bias_sink is not None:
                # straight into the flat gradient bucket: no autograd AccumulateGrad node runs for this
                # parameter (those are pinned to the stream of their first use, which breaks graph capture
                # on another stream after eager steps)
                ctx.bias_sink.add_(db)
                if ctx.bias_ready is not None:
                    ctx.bias_ready()
                db = None
        return dx, dw, db, None, None, None, None, None


def linear_bf16(x, weight, bias=None, relu=False, gelu=False):
    """y = act(x @ weight^T + bias) on the wgmma GEMM (bias/activation fused in the epilogue).
    x [M, K] bf16, weight [N, K] bf16, bias [N] (any float dtype).  ``gelu``: the erf-form GELU epilogue, inference only
    (raises when a gradient would be required)."""
    if gelu:
        if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, weight, bias)):
            raise RuntimeError("linear_bf16(gelu=True) is inference only: no backward; run it under torch.no_grad()")
        return gemm_bf16(x.contiguous(), weight, col_shift=bias.float() if bias is not None else None, gelu=True)
    return _LinearFn.apply(x, weight, bias, relu, *_grad_sink(weight), *_grad_sink(bias))


def _gelu_gemm_ok(*ts):
    from . import native

    return (all(t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(-1) == 1 and t.stride(0) % 8 == 0
                and t.data_ptr() % 16 == 0 for t in ts) and native().persistent_gemm_enabled())


def gemm_bf16_gelu_train(x, w, bias=None):
    """The training forward of a GELU linear layer: returns (y, u) with u = bf16(x @ w^T + bias) and
    y = bf16(gelu(x @ w^T + bias)) (erf form, from the fp32 value, so y is what the inference epilogue stores).
    x [M, K], w [N, K] bf16, N % 8 == 0; one persistent GEMM whose epilogue writes both."""
    from . import native, count_launch, count_fallback

    m, n = x.shape[0], w.shape[0]
    if x.is_cuda and n % 8 == 0 and _gelu_gemm_ok(x, w):
        y = torch.empty((m, n), device=x.device, dtype=torch.bfloat16)
        u = torch.empty_like(y)
        native().gemm_bf16_gelu_train(x, w, y, u, bias.float().contiguous() if bias is not None else None)
        count_launch()
        return y, u
    if x.is_cuda:
        count_fallback("gemm_bf16_gelu_train: no kernel for %s x %s: fp32 matmul on the library"
                       % (tuple(x.shape), tuple(w.shape)))
    uf = x.float() @ w.float().t() + (bias.float() if bias is not None else 0.0)
    return torch.nn.functional.gelu(uf).to(x.dtype), uf.to(x.dtype)


def gelu_grad_reference(u):
    """gelu'(u) = Phi(u) + u phi(u) in fp32."""
    uf = u.float()
    return 0.5 * (1.0 + torch.erf(uf * 0.7071067811865476)) + uf * 0.3989422804014327 * torch.exp(-0.5 * uf * uf)


def gemm_bf16_gelu_grad(dy, w, u):
    """dU = (dy @ w) * gelu'(u) in fp32, stored bf16: the dgrad of the layer after a GELU, dy [M, N2], w [N2, N] bf16
    (that layer's weight), u [M, N] the saved pre-activation.  One persistent dgrad GEMM; gelu'(u) is applied in its
    epilogue, which reads u through the fused-addend path."""
    from . import native, count_launch, count_fallback

    m, n = dy.shape[0], w.shape[1]
    if dy.is_cuda and n % 8 == 0 and _gelu_gemm_ok(dy, w, u):
        du = torch.empty((m, n), device=dy.device, dtype=torch.bfloat16)
        native().gemm_bf16_gelu_grad(dy, w, du, u)
        count_launch()
        return du
    if dy.is_cuda:
        count_fallback("gemm_bf16_gelu_grad: no kernel for %s x %s: fp32 matmul on the library"
                       % (tuple(dy.shape), tuple(w.shape)))
    return ((dy.float() @ w.float()) * gelu_grad_reference(u)).to(dy.dtype)


# EDL_PAIR_WGRAD=0: the library's weight gradient for the 32-channel stem convolutions as well
PAIR_WGRAD = __import__("os").environ.get("EDL_PAIR_WGRAD", "1") == "1"


def _pair_wgrad_ok(x, dy, w, cfg) -> bool:
    from . import native

    if not (PAIR_WGRAD and x.is_cuda and x.dtype == torch.bfloat16 and tuple(cfg) == (1, 1, 1) and w.dim() == 4):
        return False
    cout, kh, kw, cin = w.shape
    n, c, h, wd = x.shape
    return (kh == 3 and kw == 3 and cin == 32 and c == 32 and wd % 2 == 0 and cout % 32 == 0
            and native().conv3x3_wgrad_supported(n, h, wd // 2, 64, 2 * cout))


def _count_lib_conv(x, what, w_krsc, stride, groups):
    if x.is_cuda:
        from . import count_fallback
        cout, kh, kw, cin = w_krsc.shape
        count_fallback("conv %s on cuDNN: %dx%d stride %d groups %d, %d -> %d channels" % (what, kh, kw, stride, groups,
                                                                                      cin * groups, cout))


def _lib_dgrad(dy, x, w, cfg):
    """Input gradient of the convolution ``cfg`` = (stride, padding, groups), KRSC weight ``w``, on the library."""
    stride, padding, groups = cfg
    _count_lib_conv(x, "dgrad", w, stride, groups)
    return torch.ops.aten.convolution_backward(dy, x, w.permute(0, 3, 1, 2), None, [stride, stride], [padding, padding],
                                               [1, 1], False, [0, 0], groups, [True, False, False])[0]


def _lib_wgrad(dy, x, w, cfg, sink):
    """Weight gradient (KRSC) of the same convolution on the library: added into ``sink``, or returned without one."""
    stride, padding, groups = cfg
    _count_lib_conv(x, "wgrad", w, stride, groups)
    gw = torch.ops.aten.convolution_backward(dy, x, w.permute(0, 3, 1, 2), None, [stride, stride], [padding, padding],
                                             [1, 1], False, [0, 0], groups, [False, True, False])[1].permute(0, 2, 3, 1)
    if sink is None:
        return gw.contiguous()
    sink.view(w.shape).add_(gw)


class _ConvLibFn(torch.autograd.Function):
    """k x k / strided / grouped convolution on the library kernel (cuDNN) with the backward split in
    two: dgrad stays on the critical path, wgrad runs on the side stream next to the wgmma wgrad
    GEMMs and lands in the flat gradient bucket (sink) without going through ``param.grad``.
    ``w`` is stored KRSC ([Cout, kh, kw, Cin/groups]); the library sees a zero-copy NCHW-shaped view."""

    @staticmethod
    def forward(ctx, x, w, stride, padding, groups, sink, ready):
        wv = w.permute(0, 3, 1, 2)
        _count_lib_conv(x, "fprop", w, stride, groups)
        y = torch.ops.aten.convolution(x, wv, None, [stride, stride], [padding, padding], [1, 1], False, [0, 0], groups)
        ctx.save_for_backward(x, w)
        ctx.cfg = (stride, padding, groups)
        ctx.sink, ctx.ready = sink, ready
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dx = _lib_dgrad(dy, x, w, ctx.cfg) if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            # 32-input-channel 3x3 / stride 1 layer (the stem's conv1_2 / conv1_3): weight gradient in pixel-pair form
            # on the wgmma kernel even when fprop / dgrad stay on the library (these two layers are the END of
            # backward, where nothing hides a slow kernel)
            pair = _pair_wgrad_ok(x, dy, w, ctx.cfg)
            dw = _deliver_wgrad(dy, x, ctx.sink, ctx.ready, lambda sink: (
                _pair_wgrad(x, dy, w, sink) if pair else _lib_wgrad(dy, x, w, ctx.cfg, sink)))
        return dx, dw, None, None, None, None, None


def conv_lib(x, weight_krsc, stride=1, padding=0, groups=1):
    return _ConvLibFn.apply(x, weight_krsc, stride, padding, groups, *_grad_sink(weight_krsc))


def conv3x3_supported(x, weight_krsc, dgrad=False) -> bool:
    from . import native

    if not (x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16):
        return False
    n, _, h, w = x.shape
    cout, kh, kw, cin = weight_krsc.shape
    return kh == 3 and kw == 3 and native().conv3x3_supported(n, h, w, cin, cout, dgrad, 1)


class _Conv3x3Fn(torch.autograd.Function):
    """3x3 / stride 1 / pad 1 convolution on the wgmma implicit-GEMM kernel (csrc/conv3x3.cu): fprop
    with the BatchNorm statistics in its epilogue, dgrad on the same kernel with mirrored taps; the
    weight gradient uses the library kernel on the side stream (off the critical path)."""

    @staticmethod
    def forward(ctx, x, w, stats, sink, ready, bn_hook=None):
        from . import native, count_launch

        ctx.bn_hook = bn_hook
        x = _cl(x)
        n, _, h, wd = x.shape
        y = torch.empty((n, w.shape[0], h, wd), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
        native().conv3x3(x, w, y, False, stats, None, False)
        count_launch()
        ctx.save_for_backward(x, w)
        ctx.sink, ctx.ready = sink, ready
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        x, w = ctx.saved_tensors
        dy = _cl(dy)
        cfg = (1, 1, 1)
        dx = None
        if ctx.needs_input_grad[0]:
            if conv3x3_supported(dy, w, dgrad=True):
                dx = torch.empty_like(x)
                # (mask bits are a 1x1 dgrad feature; a residual BN does not feed a 3x3 convolution in these models)
                hook = ctx.bn_hook if _bn_fusable(ctx.bn_hook, x, x.shape[1]) and ctx.bn_hook.mask is None else None
                if hook is not None:
                    native().conv3x3(dy, w, dx, True, None, hook.as_list(dx.numel() // dx.shape[1], dx.shape[1]), hook.relu)
                    hook.done = True
                else:
                    native().conv3x3(dy, w, dx, True, None, None, False)
                count_launch()
            else:
                dx = _lib_dgrad(dy, x, w, cfg)
        dw = None
        if ctx.needs_input_grad[1]:
            own = OWN_WGRAD3 and conv3x3_wgrad_supported(x, w)
            dw = _deliver_wgrad(dy, x, ctx.sink, ctx.ready, lambda sink: (
                conv3x3_wgrad(x, dy, w.shape, sink) if own else _lib_wgrad(dy, x, w, cfg, sink)))
        return dx, dw, None, None, None, None


# EXPERIMENTAL until it has been validated on a GPU (written after the round-1 GPU budget was spent):
# EDL_OWN_WGRAD3=1 routes the 3x3 weight gradient through csrc/conv3x3_wgrad.cu instead of the library kernel.
OWN_WGRAD3 = __import__("os").environ.get("EDL_OWN_WGRAD3", "0") == "1"


def conv3x3_wgrad_supported(x, weight_krsc) -> bool:
    from . import native

    if not (x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16 and x.dim() == 4):
        return False
    n, c, h, w = x.shape
    cout, kh, kw, cin = weight_krsc.shape
    return kh == 3 and kw == 3 and cin == c and native().conv3x3_wgrad_supported(n, h, w, cin, cout)


def conv3x3_wgrad_split(n, h, w, cin, cout, s2=False) -> int:
    """Split-K factor ``conv3x3_wgrad`` uses when it is not given one; (n, h, w) is the geometry of dy."""
    from . import native

    if s2:                               # always the version-1 kernel (its pixel-block plan, 64-wide Cin tiles)
        kblocks, ctas = native().conv3x3_wgrad_s2_kblocks(n, h, w), native().conv3x3_wgrad_tiles(cin, cout)
    else:
        kblocks = native().conv3x3_wgrad_kblocks(n, h, w)
        ctas = native().conv3x3_wgrad_ctas(cin, cout)
    # one wave of CTAs, at least two pixel blocks per CTA; no split once a third of the SMs have a CTA (same rule as
    # the 1x1 wgrad split)
    return 1 if ctas >= 48 else max(1, min(max(1, _NUM_SMS // ctas), max(1, kblocks // 2)))


def conv3x3_wgrad(x, dy, weight_shape, sink=None, split_k: Optional[int] = None):
    """dW [Cout, 3, 3, Cin] of the 3x3 / stride 1 / pad 1 convolution on the wgmma kernel
    (csrc/conv3x3_wgrad.cu).  With ``sink`` (a flat bf16 window of the gradient bucket) the result is ADDED
    into it and ``None`` is returned; otherwise a new tensor is returned."""
    from . import native, count_launch

    x, dy = _cl(x), _cl(dy)
    cout, _, _, cin = weight_shape
    n, _, h, w = dy.shape                 # stride 2: x is twice as large; the pixel blocks tile dy
    s2 = x.shape[2] != h
    tiles = native().conv3x3_wgrad_tiles(cin, cout)
    if split_k is None:
        split_k = conv3x3_wgrad_split(n, h, w, cin, cout, s2)
    if sink is not None:
        out, acc = sink.view(weight_shape), True
    else:
        out, acc = torch.empty(tuple(weight_shape), device=x.device, dtype=torch.bfloat16), False
    partials = _splitk_partials(x.device, split_k * tiles * 128 * 192) if split_k > 1 else None
    native().conv3x3_wgrad(x, dy, out, int(split_k), acc, partials)
    count_launch(2 if split_k > 1 else 1)
    return None if sink is not None else out


def conv3x3(x, weight_krsc, stats: Optional[torch.Tensor] = None):
    """NHWC 3x3 stride-1 pad-1 convolution; ``stats`` (pre-zeroed fp32 [2*Cout]) receives the per-channel
    sum / sum of squares of the output for the following train-mode BatchNorm."""
    return _Conv3x3Fn.apply(x, weight_krsc, stats, *_grad_sink(weight_krsc), getattr(x, "_edl_bn_hook", None))


# 3x3 / pad 1 / STRIDE 2 forward convolutions (student: first block of stages 2-4; teacher: the grouped ones, which
# round 1 ran as "stride 1 then subsample" = 4x the MMA work) on the persistent wgmma kernel; the input is sampled
# by the TMA traversal stride (csrc/gemm_persist.cu).  On by default (EDL_CONV3_S2=0: off).
CONV3_S2 = __import__("os").environ.get("EDL_CONV3_S2", "1") == "1"


def conv3x3_s2_supported(x, weight_krsc, groups=1) -> bool:
    from . import native

    if not (x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16 and x.dim() == 4):
        return False
    n, c, h, w = x.shape
    cout, kh, kw, cin_g = weight_krsc.shape
    return (kh == 3 and kw == 3 and cin_g * groups == c and h % 2 == 0 and w % 2 == 0 and w // 2 <= 128
            and native().persistent_gemm_enabled()
            and native().conv3x3_supported(n, h // 2, w // 2, c, cout, False, groups))


def _conv3x3_s2_launch(x, weight_krsc, stats, scale, shift, relu, groups):
    from . import native, count_launch

    x = _cl(x)
    n, _, h, w = x.shape
    y = torch.empty((n, weight_krsc.shape[0], h // 2, w // 2), device=x.device, dtype=x.dtype,
                    memory_format=torch.channels_last)
    native().conv3x3_s2(x, weight_krsc, y, stats, scale, shift, relu, groups)
    count_launch()
    return y


@torch.no_grad()
def conv3x3_s2_infer(x, weight_krsc, scale=None, shift=None, relu=False, groups=1):
    """Inference 3x3 / pad 1 / stride 2 convolution (dense or grouped) with the folded-BN epilogue."""
    return _conv3x3_s2_launch(x, weight_krsc, None, scale, shift, relu, groups)


# Backward of the stride-2 3x3 convolutions on our own kernels (EDL_OWN_S2_BWD=1; OFF by default):
#   dgrad: four stride-1 wgmma launches over dy, one per parity class of the input pixel (1 + 2 + 2 + 4 taps = the
#          nine tap-MMAs of the forward pass), each storing through a strided tensor map.  (Zero-inserting
#          dy with csrc/pool.cu:dilate2_kernel and running the plain stride-1 dgrad costs 4x the MMAs.);
#   wgrad: the version-1 weight-gradient kernel with X read through the TMA traversal stride (csrc/conv3x3_wgrad.cu).
OWN_S2_BWD = __import__("os").environ.get("EDL_OWN_S2_BWD", "0") == "1"


def _s2_dgrad_supported(x, w) -> bool:
    from . import native

    n, c, h, wd = x.shape
    cout = w.shape[0]
    return (OWN_S2_BWD and x.is_cuda and h % 2 == 0 and wd % 2 == 0
            and native().conv3x3_dgrad_s2_supported(n, h // 2, wd // 2, c, cout))


def _s2_wgrad_supported(x, w) -> bool:
    from . import native

    n, c, h, wd = x.shape
    return (OWN_S2_BWD and x.is_cuda and h % 2 == 0 and wd % 2 == 0
            and native().conv3x3_wgrad_s2_supported(n, h // 2, wd // 2, c, w.shape[0]))


class _Conv3x3S2Fn(torch.autograd.Function):
    """Training form of the stride-2 3x3 convolution: forward on the wgmma kernel (BN statistics in its epilogue),
    input gradient = stride-1 wgmma dgrad of the zero-inserted output gradient, weight gradient on the wgmma
    wgrad kernel through a strided tensor map (side stream, straight into the gradient bucket)."""

    @staticmethod
    def forward(ctx, x, w, stats, sink, ready):
        x = _cl(x)
        y = _conv3x3_s2_launch(x, w, stats, None, None, False, 1)
        ctx.save_for_backward(x, w)
        ctx.cfg = (2, 1, 1)
        ctx.sink, ctx.ready = sink, ready
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        x, w = ctx.saved_tensors
        dy = _cl(dy)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            if _s2_dgrad_supported(x, w):
                # four stride-1 launches (1 + 2 + 2 + 4 taps), one per parity class of the input pixel, each storing
                # through a strided tensor map (csrc/gemm_persist.cu:conv3x3_dgrad_s2_persistent)
                dx = torch.empty_like(x)
                native().conv3x3_dgrad_s2(dy, w, dx)
                count_launch(4)
            else:
                dx = _lib_dgrad(dy, x, w, ctx.cfg)
        if ctx.needs_input_grad[1]:
            own = _s2_wgrad_supported(x, w)
            dw = _deliver_wgrad(dy, x, ctx.sink, ctx.ready, lambda sink: (
                conv3x3_wgrad(x, dy, w.shape, sink) if own else _lib_wgrad(dy, x, w, ctx.cfg, sink)))
        return dx, dw, None, None, None


def conv3x3_s2(x, weight_krsc, stats: Optional[torch.Tensor] = None):
    return _Conv3x3S2Fn.apply(x, weight_krsc, stats, *_grad_sink(weight_krsc))


# ---------------------------------------------------------------------------------------------------------------
# 1x1 / pad 0 / stride 2 convolutions (the projection shortcuts of plain ResNet): output pixel (h, w) reads input pixel
# (2h, 2w), i.e. the centre tap of the stride-2 3x3 convolution above -- fprop on the persistent kernel through the same
# strided input map, dgrad as one dgrad-mode launch storing the even-even pixels of a zero-filled dX, wgrad on the
# version-1 weight-gradient kernel with one tap (csrc/gemm_persist.cu, csrc/conv3x3_wgrad.cu).

def conv1x1_s2_supported(x, weight_krsc) -> bool:
    from . import native

    if not (x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16 and x.dim() == 4):
        return False
    n, c, h, w = x.shape
    if weight_krsc.dim() == 4 and tuple(weight_krsc.shape[1:3]) != (1, 1):
        return False
    cout, cin = weight_krsc.shape[0], weight_krsc.shape[-1]
    return (cin == c and c % 64 == 0 and h % 2 == 0 and w % 2 == 0 and w // 2 <= 128
            and native().conv1x1_s2_supported(n, h // 2, w // 2, c, cout, False))


def _conv1x1_s2_launch(x, weight, stats, scale, shift, relu):
    from . import native, count_launch

    x = _cl(x)
    n, _, h, w = x.shape
    y = torch.empty((n, weight.shape[0], h // 2, w // 2), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
    native().conv1x1_s2(x, weight, y, False, stats, scale, shift, relu)
    count_launch()
    return y


@torch.no_grad()
def conv1x1_s2_infer(x, weight_krsc, scale=None, shift=None, relu=False):
    """Inference 1x1 / stride 2 convolution with the folded-BN scale / shift and the ReLU in the epilogue."""
    return _conv1x1_s2_launch(x, weight_krsc, None, scale, shift, relu)


def conv1x1_s2_wgrad_split(n, ho, wo, cin, cout) -> int:
    """Split-K factor of the 1x1 / stride-2 weight gradient: the rule of ``conv3x3_wgrad_split`` over its tiles (one CTA
    per 128 x 64 tile instead of three)."""
    from . import native

    kblocks, ctas = native().conv3x3_wgrad_s2_kblocks(n, ho, wo), native().conv3x3_wgrad_tiles(cin, cout) // 3
    return 1 if ctas >= 48 else max(1, min(max(1, _NUM_SMS // ctas), max(1, kblocks // 2)))


def conv1x1_s2_wgrad(x, dy, weight_shape, sink=None, split_k: Optional[int] = None):
    """dW [Cout, 1, 1, Cin] of the 1x1 / stride 2 convolution; with ``sink`` added into it (returns None)."""
    from . import native, count_launch

    x, dy = _cl(x), _cl(dy)
    cout, cin = weight_shape[0], weight_shape[-1]
    n, _, ho, wo = dy.shape
    if split_k is None:
        split_k = conv1x1_s2_wgrad_split(n, ho, wo, cin, cout)
    if sink is not None:
        out, acc = sink.view(weight_shape), True
    else:
        out, acc = torch.empty(tuple(weight_shape), device=x.device, dtype=torch.bfloat16), False
    tiles = native().conv3x3_wgrad_tiles(cin, cout) // 3
    partials = _splitk_partials(x.device, split_k * tiles * 128 * 64) if split_k > 1 else None
    native().conv1x1_s2_wgrad(x, dy, out, int(split_k), acc, partials)
    count_launch(2 if split_k > 1 else 1)
    return None if sink is not None else out


class _Conv1x1S2Fn(torch.autograd.Function):
    """Training form of the 1x1 / stride 2 convolution (BN statistics in the fprop epilogue).  The input gradient is a
    dense tensor, zero at the three pixel parities the convolution skips, so a forked input adds it like any other."""

    @staticmethod
    def forward(ctx, x, w, stats, sink, ready):
        x = _cl(x)
        y = _conv1x1_s2_launch(x, w, stats, None, None, False)
        ctx.save_for_backward(x, w)
        ctx.cfg = (2, 0, 1)
        ctx.sink, ctx.ready = sink, ready
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        x, w = ctx.saved_tensors
        dy = _cl(dy)
        n, c, h, wd = x.shape
        cout = w.shape[0]
        dx = dw = None
        if ctx.needs_input_grad[0]:
            if native().conv1x1_s2_supported(n, h // 2, wd // 2, c, cout, True):
                dx = torch.empty_like(x)
                native().conv1x1_s2(dy, w, dx, True, None, None, None, False)
                count_launch()
            else:
                dx = _lib_dgrad(dy, x, w, ctx.cfg)
        if ctx.needs_input_grad[1]:
            own = native().conv3x3_wgrad_s2_supported(n, h // 2, wd // 2, c, cout)
            dw = _deliver_wgrad(dy, x, ctx.sink, ctx.ready, lambda sink: (
                conv1x1_s2_wgrad(x, dy, w.shape, sink) if own else _lib_wgrad(dy, x, w, ctx.cfg, sink)))
        return dx, dw, None, None, None


def conv1x1_s2(x, weight_krsc, stats: Optional[torch.Tensor] = None):
    """NHWC 1x1 / pad 0 / stride 2 convolution, weight [Cout, 1, 1, Cin]; ``stats`` (pre-zeroed fp32 [2*Cout]) receives
    the per-channel sum / sum of squares of the output for the following train-mode BatchNorm."""
    return _Conv1x1S2Fn.apply(x, weight_krsc, stats, *_grad_sink(weight_krsc))


# The first stem convolution (3 -> 32 channels, 3x3 / stride 2) runs on the direct kernel of csrc/stem.cu with the
# BatchNorm statistics fused in.  On by default (EDL_OWN_STEM1=0: library kernel).
OWN_STEM1 = __import__("os").environ.get("EDL_OWN_STEM1", "1") == "1"


def stem7_supported(x, weight_krsc) -> bool:
    """7x7 / stride 2 / pad 3 convolution of a 3-channel image (the teacher's stem) as im2col + wgmma GEMM."""
    return (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] == 3
            and weight_krsc.dtype == torch.bfloat16 and tuple(weight_krsc.shape[1:]) == (7, 7, 3)
            and weight_krsc.shape[0] % 8 == 0)


_STEM7_W = {}


@torch.no_grad()
def stem7_infer(x, weight_krsc, scale=None, shift=None, relu=False):
    """y = act(conv7x7/s2/p3(x, w) * scale + shift) for x [N,3,H,W] (channels_last bf16), w KRSC [Cout,7,7,3]:
    ``stem7_im2col`` writes the windows as rows of a [N*Ho*Wo, 160] matrix ((r, s, c) order = the KRSC weight order, 13 zero
    columns of padding) and the persistent GEMM applies the folded BatchNorm and the ReLU in its epilogue.  The reference's
    teacher runs this layer through the serving library (start_local_teacher.sh:24-30)."""
    from . import native, count_launch

    x = _cl(x)
    n, _, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    cout = weight_krsc.shape[0]
    # the padded weight is cached per weight tensor (held, so that its address cannot be reused by another tensor and
    # alias a stale entry) and version
    hit = _STEM7_W.get("w")
    if hit is not None and hit[0] is weight_krsc and hit[1] == weight_krsc._version:
        wp = hit[2]
    else:
        wp = torch.zeros((cout, 160), device=x.device, dtype=torch.bfloat16)
        wp[:, :147] = weight_krsc.reshape(cout, 147)
        _STEM7_W["w"] = (weight_krsc, weight_krsc._version, wp)
    a = torch.empty((n * ho * wo, 160), device=x.device, dtype=torch.bfloat16)
    native().stem7_im2col(x, a)
    count_launch()
    y = torch.empty((n, cout, ho, wo), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
    gemm_bf16(a, wp, out=y.permute(0, 2, 3, 1).reshape(-1, cout), col_scale=scale, col_shift=shift, relu=relu)
    return y


def _stem7_padded(weight_krsc):
    """The [Cout, 160] GEMM weight of a 7x7 stem, rebuilt from ``weight_krsc`` on EVERY call: one copy of the 147 real
    columns into a buffer kept on the parameter (its 13 pad columns stay zero).  The copy is part of a captured graph, so
    a replay reads the weight the optimizer last wrote -- a cache keyed on ``weight._version`` (``stem7_infer``) would not
    see the in-place updates of a replayed optimizer step."""
    cout = weight_krsc.shape[0]
    buf = getattr(weight_krsc, "_edl_stem7_padded", None)
    if buf is None or buf.device != weight_krsc.device or buf.shape[0] != cout:
        buf = torch.zeros((cout, 160), device=weight_krsc.device, dtype=torch.bfloat16)
        weight_krsc._edl_stem7_padded = buf
    buf[:, :147].copy_(weight_krsc.detach().reshape(cout, 147))
    return buf


def stem7_wgrad(dy, a, weight_shape, sink=None, split_k: Optional[int] = None):
    """dW [Cout, 7, 7, 3] of the 7x7 stem from its output gradient and saved im2col matrix ``a`` [M, 160]: the split-K
    weight-gradient GEMM over the padded width, storing only the 147 real columns (KRSC order = [Cout, 147]); with
    ``sink`` added into it (returns None)."""
    from . import native, count_launch

    dy = _cl(dy)
    cout = weight_shape[0]
    dy2 = dy.permute(0, 2, 3, 1).reshape(-1, cout)
    split = split_k if split_k is not None else _split_k_for(cout, 160, dy2.shape[0])
    out = sink.view(cout, 147) if sink is not None else torch.empty((cout, 147), device=dy.device, dtype=torch.bfloat16)
    tiles = (cout + 127) // 128 * 2            # 128-column tiles over the 160 columns
    partials = _splitk_partials(dy.device, split * tiles * 128 * 128) if split > 1 else None
    native().gemm_wgrad_bf16(dy2, a, out, split, sink is not None, partials)
    count_launch(2 if split > 1 else 1)
    return None if sink is not None else out.view(weight_shape)


class _Stem7Fn(torch.autograd.Function):
    """Training form of the 7x7 / stride 2 / pad 3 stem: ``stem7_im2col`` + the persistent GEMM with the BN statistics
    in its epilogue; the im2col matrix is kept for the weight gradient.  The input is the image: no dgrad."""

    @staticmethod
    def forward(ctx, x, w, stats, sink, ready):
        from . import native, count_launch

        x = _cl(x)
        n, _, h, wd = x.shape
        ho, wo = (h - 1) // 2 + 1, (wd - 1) // 2 + 1
        cout = w.shape[0]
        wp = _stem7_padded(w)
        a = torch.empty((n * ho * wo, 160), device=x.device, dtype=torch.bfloat16)
        native().stem7_im2col(x, a)
        count_launch()
        y = torch.empty((n, cout, ho, wo), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
        gemm_bf16(a, wp, out=y.permute(0, 2, 3, 1).reshape(-1, cout), col_stats=stats)
        ctx.save_for_backward(x, w, a)
        ctx.sink, ctx.ready = sink, ready
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, a = ctx.saved_tensors
        dx = dw = None
        if ctx.needs_input_grad[0]:      # nobody asks for the gradient of the images; kept for completeness
            dx = _lib_dgrad(_cl(dy), x, w, (2, 3, 1))
        if ctx.needs_input_grad[1]:
            dw = _deliver_wgrad(dy, a, ctx.sink, ctx.ready, lambda sink: stem7_wgrad(dy, a, w.shape, sink))
        return dx, dw, None, None, None


def stem7(x, weight_krsc, stats: Optional[torch.Tensor] = None):
    """7x7 / stride 2 / pad 3 convolution of a 3-channel image (plain ResNet's stem), weight KRSC [Cout, 7, 7, 3];
    ``stats`` (pre-zeroed fp32 [2*Cout]) receives the BN statistics of the output.  ``stem7_supported`` states what is
    accepted."""
    return _Stem7Fn.apply(x, weight_krsc, stats, *_grad_sink(weight_krsc))


def stem_conv_supported(x, weight_krsc) -> bool:
    return (x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16 and x.dim() == 4
            and x.shape[1] == 3 and tuple(weight_krsc.shape) == (32, 3, 3, 3))


class _StemConvFn(torch.autograd.Function):
    """conv3x3 / stride 2 / pad 1, 3 -> 32 channels: forward on the direct kernel (+ BN statistics); the weight gradient
    (and, if anybody asks for it, the input gradient) on the library kernels like every other k x k convolution."""

    @staticmethod
    def forward(ctx, x, w, stats, sink, ready):
        from . import native, count_launch

        x = _cl(x)
        n, _, h, wd = x.shape
        y = torch.empty((n, 32, (h - 1) // 2 + 1, (wd - 1) // 2 + 1), device=x.device, dtype=x.dtype,
                        memory_format=torch.channels_last)
        native().stem_conv3x3s2(x, w, y, stats)
        count_launch()
        ctx.save_for_backward(x, w)
        ctx.cfg = (2, 1, 1)
        ctx.sink, ctx.ready = sink, ready
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        x, w = ctx.saved_tensors
        dy = _cl(dy)
        dx = None
        if ctx.needs_input_grad[0]:      # nobody asks for the gradient of the images; kept for completeness
            dx = _lib_dgrad(dy, x, w, ctx.cfg)
        dw = None
        if ctx.needs_input_grad[1]:
            def wgrad(sink):
                if not (x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0 and x.shape[3] <= 4096):
                    return _lib_wgrad(dy, x, w, ctx.cfg, sink)
                ws, counters = _stem_scratch(x.device)
                out = sink.view(w.shape) if sink is not None else torch.empty_like(w)
                native().stem_wgrad(x, dy, out, ws, counters, sink is not None)
                count_launch()
                return None if sink is not None else out

            dw = _deliver_wgrad(dy, x, ctx.sink, ctx.ready, wgrad)
        return dx, dw, None, None, None


def stem_conv(x, weight_krsc, stats: Optional[torch.Tensor] = None):
    return _StemConvFn.apply(x, weight_krsc, stats, *_grad_sink(weight_krsc))


# ---------------------------------------------------------------------------------------------------------------
# 3x3 / stride 1 convolutions with 32 input channels (the stem's conv1_2 / conv1_3) in "pixel-pair" form on the
# 64-channel wgmma kernels (csrc/misc.cu:pair_weight_expand_kernel explains the transform).  EDL_OWN_STEM23=1.
OWN_STEM23 = __import__("os").environ.get("EDL_OWN_STEM23", "0") == "1"


def _pair_view(t):
    """NHWC [N, H, W, C] seen as [N, H, W/2, 2C] (zero-copy), returned in the NCHW-shaped channels_last form."""
    n, c, h, w = t.shape
    return t.as_strided((n, 2 * c, h, w // 2), (h * w * c, 1, w * c, 2 * c))


def _unpair_view(t2):
    n, c2, h, w2 = t2.shape
    return t2.as_strided((n, c2 // 2, h, 2 * w2), (h * w2 * c2, 1, w2 * c2, c2 // 2))


def _pair_wgrad(x, dy, w, sink):
    """Weight gradient of a 3x3 / stride 1 convolution with 32 input channels in pixel-pair form: the 64-channel wgmma
    weight gradient over pixel pairs, folded back to ``w``'s [Cout, 3, 3, 32] (added into ``sink``, or returned)."""
    from . import native, count_launch

    dw2 = conv3x3_wgrad(_pair_view(_cl(x)), _pair_view(_cl(dy)), (2 * w.shape[0], 3, 3, 64), None)
    out = sink.view(w.shape) if sink is not None else torch.empty_like(w)
    native().pair_weight_fold(dw2, out, sink is not None)
    count_launch()
    return None if sink is not None else out


def conv3x3_pair_supported(x, weight_krsc) -> bool:
    from . import native

    if not (OWN_STEM23 and x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16 and x.dim() == 4):
        return False
    n, c, h, w = x.shape
    cout, kh, kw, cin = weight_krsc.shape
    return (kh == 3 and kw == 3 and cin == 32 and c == 32 and w % 2 == 0 and cout % 32 == 0
            and native().conv3x3_supported(n, h, w // 2, 64, 2 * cout, False, 1)
            and native().conv3x3_supported(n, h, w // 2, 2 * cout, 64, True, 1))


class _Conv3x3PairFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, stats, sink, ready):
        from . import native, count_launch

        C = native()
        x = _cl(x)
        n, _, h, wd = x.shape
        cout = w.shape[0]
        w2 = torch.empty((2 * cout, 3, 3, 64), device=x.device, dtype=x.dtype)
        C.pair_weight_expand(w.contiguous(), w2)
        x2 = _pair_view(x)
        y2 = torch.empty((n, 2 * cout, h, wd // 2), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
        s2 = torch.zeros(4 * cout, device=x.device, dtype=torch.float32) if stats is not None else None
        C.conv3x3(x2, w2, y2, False, s2, None, False)
        count_launch(2)
        if stats is not None:
            C.fold_pair_stats(s2, stats)
            count_launch()
        ctx.save_for_backward(x, w, w2)
        ctx.sink, ctx.ready = sink, ready
        return _unpair_view(y2)

    @staticmethod
    def backward(ctx, dy):
        from . import native, count_launch

        C = native()
        x, w, w2 = ctx.saved_tensors
        dy = _cl(dy)
        x2, dy2 = _pair_view(x), _pair_view(dy)
        dx = None
        if ctx.needs_input_grad[0]:
            dx2 = torch.empty_like(x2)
            C.conv3x3(dy2, w2, dx2, True, None, None, False)
            count_launch()
            dx = _unpair_view(dx2)
        dw = None
        if ctx.needs_input_grad[1]:
            dw = _deliver_wgrad(dy, x, ctx.sink, ctx.ready, lambda sink: _pair_wgrad(x, dy, w, sink))
        return dx, dw, None, None, None


def conv3x3_pair(x, weight_krsc, stats: Optional[torch.Tensor] = None):
    return _Conv3x3PairFn.apply(x, weight_krsc, stats, *_grad_sink(weight_krsc))


def conv3x3_infer_supported(x, weight_krsc, groups=1) -> bool:
    from . import native

    if not (x.is_cuda and x.dtype == torch.bfloat16 and weight_krsc.dtype == torch.bfloat16 and x.dim() == 4):
        return False
    n, c, h, w = x.shape
    cout, kh, kw, cin_g = weight_krsc.shape
    return (kh == 3 and kw == 3 and cin_g * groups == c
            and native().conv3x3_supported(n, h, w, c, cout, False, groups))


@torch.no_grad()
def conv3x3_infer(x, weight_krsc, scale=None, shift=None, relu=False, groups=1):
    """Inference 3x3 / stride 1 / pad 1 convolution (dense or grouped) on the persistent wgmma kernel with
    the folded-BatchNorm scale / shift and the ReLU in its epilogue.  The grouped form is what the
    ResNeXt teacher needs."""
    from . import native, count_launch

    x = _cl(x)
    n, _, h, w = x.shape
    y = torch.empty((n, weight_krsc.shape[0], h, w), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
    native().conv3x3_infer(x, weight_krsc, y, scale, shift, relu, groups)
    count_launch()
    return y
