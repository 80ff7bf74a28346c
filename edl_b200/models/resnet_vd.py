"""ResNet-vd family (the distillation *student*), NHWC / bf16, built from the fused sm_90a ops.

Architecture follows the reference definition example/distill/resnet/models/resnet_vd.py:43-143,
213-291 (3x3x3 deep stem, stride on the 3x3 of the bottleneck, avg-pool + 1x1 "vd" shortcut) --
re-expressed as ConvBNAct units whose 1x1 convolutions run on the wgmma GEMM with the BatchNorm
statistics reduced in the GEMM epilogue, and whose BN-apply / residual-add / ReLU are one kernel.
"""
from __future__ import annotations

import functools
import math
import os
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..ops.bn import BatchNormAct2d, checkpoint_context


class ConvBNAct(nn.Module):
    """conv (no bias) -> train-mode BN -> (+ residual) -> (ReLU), as 2-3 kernels.

    The weight is stored KRSC (``[Cout, kh, kw, Cin]``), i.e. already in the layout the NHWC
    implicit GEMM consumes; torch/cuDNN sees it through a zero-copy ``permute`` view."""

    def __init__(self, cin, cout, k, stride=1, relu=True, groups=1, impl="auto"):
        super().__init__()
        self.cin, self.cout, self.k, self.stride, self.groups = cin, cout, k, stride, groups
        self.weight = nn.Parameter(torch.empty(cout, k, k, cin // groups))
        std = math.sqrt(2.0 / (k * k * cin // groups))
        nn.init.normal_(self.weight, 0.0, std)
        self.bn = BatchNormAct2d(cout, relu=relu)
        self.impl = impl
        self.fwd_stats: Optional[torch.Tensor] = None  # arena slice [2*cout], zeroed every step
        self.split_backward = os.environ.get("EDL_SPLIT_CONV_BWD", "1") == "1"
        self.own_conv3 = os.environ.get("EDL_OWN_CONV3", "1") == "1"

    def _use_gemm(self, x):
        if self.impl == "cudnn":
            return False
        return (self.k == 1 and self.stride == 1 and self.groups == 1 and x.is_cuda
                and x.dtype == torch.bfloat16 and self.cin % 8 == 0 and self.cout % 8 == 0)

    def conv(self, x, want_stats, fork=False):
        op = None
        if self._use_gemm(x):
            op = functools.partial(ops.conv1x1, fork=fork)
        elif (self.k == 3 and self.stride == 1 and self.groups == 1 and self.impl != "cudnn" and self.own_conv3
                and ops.conv3x3_supported(x, self.weight)):
            # own wgmma implicit-GEMM 3x3 (csrc/conv3x3.cu) with the BN statistics in its epilogue
            op = ops.conv3x3
        elif (self.k == 3 and self.stride == 1 and self.groups == 1 and self.cin == 32 and self.impl != "cudnn"
                and self.own_conv3 and ops.conv3x3_pair_supported(x, self.weight)):
            # EDL_OWN_STEM23=1: 32-channel stem convolutions in pixel-pair form on the wgmma 3x3 kernels
            op = ops.conv3x3_pair
        elif (self.k == 3 and self.stride == 2 and self.cin == 3 and self.cout == 32 and self.impl != "cudnn"
                and ops.gemm.OWN_STEM1 and ops.stem_conv_supported(x, self.weight)):
            # experimental (EDL_OWN_STEM1=1): direct kernel for the K = 27 stem convolution, statistics fused
            op = ops.stem_conv
        elif (self.k == 3 and self.stride == 2 and self.groups == 1 and self.impl != "cudnn" and self.own_conv3
                and ops.gemm.CONV3_S2 and ops.conv3x3_s2_supported(x, self.weight)):
            # experimental (EDL_CONV3_S2=1): stride-2 fprop on the wgmma kernel, statistics in its epilogue
            op = ops.conv3x3_s2
        elif (self.k == 1 and self.stride == 2 and self.groups == 1 and self.impl != "cudnn"
                and ops.conv1x1_s2_supported(x, self.weight)):
            # plain ResNet's projection shortcuts: 1x1 / stride 2 on the persistent kernel (the stride-2 3x3's centre tap)
            op = ops.conv1x1_s2 if (want_stats or torch.is_grad_enabled()) else ops.conv1x1_s2_infer
        elif (self.k == 7 and self.stride == 2 and self.cin == 3 and self.impl != "cudnn"
                and ops.stem7_supported(x, self.weight)):
            # plain ResNet's 7x7 stem: im2col + persistent GEMM (statistics in its epilogue), split-K GEMM weight gradient
            op = ops.stem7
        if op is not None:
            stats = None
            if want_stats:
                stats = self.fwd_stats if self.fwd_stats is not None else torch.zeros(
                    2 * self.cout, device=x.device, dtype=torch.float32)
            return op(x, self.weight, stats), stats
        if self.split_backward and torch.is_grad_enabled() and self.weight.requires_grad:
            # library conv whose wgrad half runs on the side stream (ops/gemm.py:_ConvLibFn)
            return ops.conv_lib(x, self.weight, self.stride, (self.k - 1) // 2, self.groups), None
        w = self.weight.permute(0, 3, 1, 2)
        if x.is_cuda:
            ops.count_fallback("conv fprop on cuDNN (inference / frozen weight): %dx%d stride %d, %d -> %d channels" % (
                self.k, self.k, self.stride, self.cin, self.cout))
        y = F.conv2d(x, w, None, self.stride, (self.k - 1) // 2, 1, self.groups)
        return y, None

    def can_fork(self, x):
        """True if forward(x, fork=True) can hand back an alias of ``x`` whose gradient is summed inside
        this convolution's dgrad epilogue (wgmma 1x1 path, training)."""
        return self._use_gemm(x) and torch.is_grad_enabled() and x.requires_grad

    def forward(self, x, residual=None, fork=False):
        y, stats = self.conv(x, self.training, fork)
        xa = None
        if fork:
            y, xa = y
        # stats is None for library convs: the BN op then computes them itself (SM-resident fused
        # kernel when the tensor fits, else the streaming stats kernel into its arena slice)
        out = self.bn(y, residual=residual, sums=stats)
        return (out, xa) if fork else out


class Bottleneck(nn.Module):
    def __init__(self, cin, width, stride, if_first, impl):
        super().__init__()
        cout = width * 4
        self.a = ConvBNAct(cin, width, 1, 1, True, impl=impl)
        self.b = ConvBNAct(width, width, 3, stride, True, impl=impl)
        self.c = ConvBNAct(width, cout, 1, 1, True, impl=impl)  # ReLU applied after the residual add
        self.pool = False
        self.short = None
        if cin != cout or stride != 1 or if_first:
            # vd shortcut: 2x2 avg-pool (ceil) then 1x1 conv; the very first block keeps a plain 1x1
            self.pool = not if_first and stride != 1
            self.short = ConvBNAct(cin, cout, 1, stride if (if_first or not self.pool) else 1, False,
                                   impl=impl)

    def forward(self, x):
        # x has two consumers (conv a and the shortcut): route the shortcut through the alias returned by
        # conv a so that both gradients are summed in a's dgrad epilogue
        if self.a.can_fork(x):
            y, xs = self.a(x, fork=True)
        else:
            ops.drop_bn_hook(x)          # two consumers, no fork: nobody sees x's complete gradient
            y, xs = self.a(x), x
        if self.short is not None:
            s = ops.avg_pool_2x2(xs) if self.pool else xs
            s = self.short(s)
        else:
            s = xs
        y = self.b(y)
        return self.c(y, residual=s)


class BasicBlock(nn.Module):
    def __init__(self, cin, width, stride, if_first, impl):
        super().__init__()
        self.a = ConvBNAct(cin, width, 3, stride, True, impl=impl)
        self.b = ConvBNAct(width, width, 3, 1, True, impl=impl)
        self.pool = False
        self.short = None
        if cin != width or stride != 1 or if_first:
            self.pool = not if_first and stride != 1
            self.short = ConvBNAct(cin, width, 1, stride if (if_first or not self.pool) else 1,
                                   False, impl=impl)

    def forward(self, x):
        ops.drop_bn_hook(x)              # x feeds conv a (3x3) and the shortcut
        if self.short is not None:
            s = ops.avg_pool_2x2(x) if self.pool else x
            s = self.short(s)
        else:
            s = x
        return self.b(self.a(x), residual=s)


class FCHead(nn.Module):
    """Classifier parameters (uniform +-1/sqrt(fan_in) like the reference, resnet_vd.py:133-141)."""

    def __init__(self, cin, class_dim):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(class_dim, cin))
        self.bias = nn.Parameter(torch.zeros(class_dim, dtype=torch.float32))
        stdv = 1.0 / math.sqrt(cin)
        nn.init.uniform_(self.weight, -stdv, stdv)


_DEPTHS = {18: [2, 2, 2, 2], 34: [3, 4, 6, 3], 50: [3, 4, 6, 3], 101: [3, 4, 23, 3],
           152: [3, 8, 36, 3], 200: [3, 12, 48, 3]}


class ResNetVd(nn.Module):
    def __init__(self, layers=50, class_dim=1000, impl="auto", width_mult=1.0, recompute=False):
        super().__init__()
        # recompute: drop every residual block's inner activations after forward and re-run the block
        # during backward (reference: dist_strategy.forward_recompute + model.checkpoints = the block
        # outputs, example/distill/resnet/train_with_fleet.py:328-331).  Trades ~1/3 more compute for
        # ~3x less activation memory; off on the benchmark path (180 GB of HBM3e do not need it).
        self.recompute = recompute
        assert layers in _DEPTHS, "supported layers are %s" % sorted(_DEPTHS)
        depth = _DEPTHS[layers]
        bottleneck = layers >= 50
        w = [int(c * width_mult) for c in (64, 128, 256, 512)]
        s0, s1 = max(8, int(32 * width_mult)), max(8, int(64 * width_mult))
        self.stem = nn.Sequential(ConvBNAct(3, s0, 3, 2, True, impl=impl),
                                  ConvBNAct(s0, s0, 3, 1, True, impl=impl),
                                  ConvBNAct(s0, s1, 3, 1, True, impl=impl))
        blocks: List[nn.Module] = []
        cin = s1
        for stage, n in enumerate(depth):
            for i in range(n):
                stride = 2 if i == 0 and stage != 0 else 1
                if_first = stage == 0 and i == 0
                if bottleneck:
                    blocks.append(Bottleneck(cin, w[stage], stride, if_first, impl))
                    cin = w[stage] * 4
                else:
                    blocks.append(BasicBlock(cin, w[stage], stride, if_first, impl))
                    cin = w[stage]
        self.blocks = nn.Sequential(*blocks)
        # registered last (as a child module) so that reverse registration order == the order in
        # which gradients become ready during backward (see parallel/flat.py)
        self.fc = FCHead(cin, class_dim)
        self.feat_dim = cin
        self.impl = impl

    @property
    def fc_weight(self):
        return self.fc.weight

    @property
    def fc_bias(self):
        return self.fc.bias

    def forward(self, x):
        x = self.stem(x)
        x = ops.max_pool_3x3_s2(x)
        if self.recompute and self.training and torch.is_grad_enabled():
            from torch.utils.checkpoint import checkpoint
            for blk in self.blocks:
                x = checkpoint(blk, x, use_reentrant=False, context_fn=checkpoint_context)
        else:
            x = self.blocks(x)
        x = ops.global_avg_pool(x)
        if x.is_cuda and x.dtype == torch.bfloat16 and self.impl != "cudnn":
            return ops.linear_bf16(x, self.fc_weight, self.fc_bias)
        return F.linear(x, self.fc_weight, self.fc_bias.to(x.dtype))

    def conv_bn_units(self):
        return [m for m in self.modules() if isinstance(m, ConvBNAct)]


def to_train_dtype(model: nn.Module, dtype=torch.bfloat16, device=None):
    """Cast conv/fc weights to ``dtype`` while BN parameters, biases and running stats stay fp32."""
    for m in model.modules():
        for name, p in list(m.named_parameters(recurse=False)):
            keep_fp32 = isinstance(m, BatchNormAct2d) or (name.endswith("bias") and not isinstance(m, nn.Conv2d))
            p.data = p.data.to(device=device, dtype=torch.float32 if keep_fp32 else dtype)
        for name, b in list(m.named_buffers(recurse=False)):
            m._buffers[name] = b.to(device=device)
    return model


def ResNet18_vd(**kw): return ResNetVd(18, **kw)
def ResNet34_vd(**kw): return ResNetVd(34, **kw)
def ResNet50_vd(**kw): return ResNetVd(50, **kw)
def ResNet101_vd(**kw): return ResNetVd(101, **kw)
def ResNet152_vd(**kw): return ResNetVd(152, **kw)
def ResNet200_vd(**kw): return ResNetVd(200, **kw)
