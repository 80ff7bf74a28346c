"""ResNeXt (the distillation *teacher*: ResNeXt101_32x16d_wsl), inference-only, NHWC / bf16.

The reference never contains this network -- it downloads a pre-exported Paddle Serving model
(README.md:51-57, example/distill/resnet/scripts/start_local_teacher.sh:19-30); the architecture is
the public WSL / torchvision ResNeXt (groups 32, width-per-group 16, depths 3-4-23-3; 194.0 M
params, 72.3 GFLOP/img -- SURVEY App. F.2).

Inference formulation: every BatchNorm is folded into a per-output-channel (scale, shift), so a
layer is  conv -> *scale + shift (+ residual) -> ReLU :
  * 1x1 convolutions run on the wgmma GEMM with scale/shift/ReLU fused in the epilogue
    (``ops.gemm_bf16(col_scale=, col_shift=, relu=)``),
  * grouped 3x3 convolutions use the library conv followed by the fused scale-shift-(add)-ReLU kernel,
  * the block's last 1x1 adds the shortcut and applies ReLU in one fused kernel.
"""
import math
import os
from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops


class FoldedConv(nn.Module):
    """conv (+ folded BN scale/shift) (+ residual) (+ ReLU) for inference."""

    def __init__(self, cin, cout, k, stride=1, groups=1, relu=True):
        super().__init__()
        self.cin, self.cout, self.k, self.stride, self.groups, self.relu = cin, cout, k, stride, groups, relu
        self.weight = nn.Parameter(torch.empty(cout, k, k, cin // groups), requires_grad=False)   # KRSC
        nn.init.normal_(self.weight, 0.0, math.sqrt(2.0 / (k * k * cin // groups)))
        # folded BN: scale = gamma / sqrt(var + eps), shift = beta - mean * scale  (random-init teacher:
        # gamma=1, beta=0, running stats (0, 1) => identity; real weights load through load_bn())
        self.register_buffer("scale", torch.ones(cout, dtype=torch.float32))
        self.register_buffer("shift", torch.zeros(cout, dtype=torch.float32))
        self.own_conv3 = os.environ.get("EDL_OWN_CONV3", "1") == "1"
        self._fp8 = None             # None (bf16), "tensor" or "block": the enabled fp8 mode of a 1x1 convolution
        self._fp8_cache = None

    def load_bn(self, gamma, beta, mean, var, eps=1e-5):
        s = gamma.float() * torch.rsqrt(var.float() + eps)
        self.scale.copy_(s)
        self.shift.copy_(beta.float() - mean.float() * s)
        self._w_scaled = None

    def _scaled_weight(self):
        """bf16 [Cout, Cin] weights with the folded-BN scale multiplied in (cached; inference weights are frozen)."""
        key = (self.weight.data_ptr(), self.weight._version, self.scale._version)
        if getattr(self, "_w_scaled", None) is None or self._w_scaled[0] != key:
            w = (self.weight.view(self.cout, self.cin).float() * self.scale.float()[:, None]).to(self.weight.dtype)
            self._w_scaled = (key, w.contiguous())
        return self._w_scaled[1]

    def _residual_fusable(self, residual, y):
        return (ops.native().persistent_gemm_enabled() and residual.shape == y.shape and residual.dtype == y.dtype
                and residual.is_contiguous(memory_format=torch.channels_last) and self.cout % 8 == 0
                and residual.data_ptr() % 16 == 0)

    # ---- fp8 (e4m3) mode of the 1x1 convolutions: see ops/fp8.py -------------------------------
    def _widened_groups(self):
        """(weight [Cout, 3, 3, 64], groups) with neighbouring groups merged into 64-input-channel block-diagonal
        groups, or None when the layer does not need it (>= 64 channels per group) or does not fit the scheme."""
        cout, kh, kw, cin_g = self.weight.shape
        if cin_g >= 64 or 64 % cin_g != 0 or self.groups % (64 // cin_g) != 0:
            return None
        cached = getattr(self, "_w64", None)
        if cached is not None and cached[0].device == self.weight.device and cached[2] == self.weight._version:
            return cached[0], cached[1]
        merge = 64 // cin_g                       # original groups per widened group
        cout_g = cout // self.groups
        w = self.weight.detach()
        w64 = torch.zeros((cout, kh, kw, 64), dtype=w.dtype, device=w.device)
        sub = (torch.arange(cout, device=w.device) // cout_g) % merge        # position of o's group inside its block
        for j in range(merge):
            rows = (sub == j).nonzero().flatten()
            w64[rows, :, :, j * cin_g:(j + 1) * cin_g] = w[rows]
        self._w64 = (w64.contiguous(), self.groups // merge, self.weight._version)
        return self._w64[0], self._w64[1]

    def fp8_eligible(self):
        return self.k == 1 and self.groups == 1 and self.cin % 16 == 0 and self.cout % 8 == 0

    def begin_calibration(self):
        self._amax = torch.zeros(1, dtype=torch.float32, device=self.weight.device)

    def finish_calibration(self, margin: float = 1.0):
        """Freeze the activation scale from the recorded max|x|; the weights are quantised per output channel."""
        from ..ops.fp8 import E4M3_MAX

        amax = float(self._amax.item()) if getattr(self, "_amax", None) is not None else 0.0
        self._amax = None
        if not self.fp8_eligible() or amax <= 0.0:
            return False
        self.act_scale = torch.full((1,), amax * margin / E4M3_MAX, dtype=torch.float32, device=self.weight.device)
        self._fp8 = "tensor"
        self._fp8_cache = None                  # a recalibration: deq_scale carries the new activation scale
        self._fp8_weights()
        return True

    def enable_fp8_blocks(self):
        """Block-scaled fp8: the weights are quantised per 128x128 block; the input is scaled per row and 128-channel
        block when the layer runs, so there is nothing to calibrate and no host synchronisation."""
        if not self.fp8_eligible():
            return False
        self._fp8 = "block"
        self._fp8_weights()
        return True

    def _fp8_weights(self):
        """(e4m3 weights, their scales, ones, zeros) of the enabled fp8 mode, quantised from the current weight on its
        device: rebuilt after a load (``load_state_dict``, ``load_bn``) or a move (``.to()``), like ``_scaled_weight``.
        Per-tensor: per-output-channel weight scales with the calibrated activation scale and the folded-BN scale
        multiplied in (``deq_scale``, so it is also keyed on the activation scale); block: one scale per 128x128
        block."""
        from ..ops.fp8 import quantize_weight_blocks, quantize_weight_rows

        w, s = self.weight, self.scale
        key = (self._fp8, w.device, w.data_ptr(), w._version, s.data_ptr(), s._version)
        if self._fp8 == "tensor":
            if self.act_scale.device != w.device:
                self.act_scale = self.act_scale.to(w.device)
            key += (self.act_scale.data_ptr(), self.act_scale._version)
        if self._fp8_cache is None or self._fp8_cache[0] != key:
            w2 = w.detach().view(self.cout, self.cin)
            if self._fp8 == "block":
                q, ws = quantize_weight_blocks(w2)
            else:
                q, ws = quantize_weight_rows(w2)
                ws = (self.act_scale * ws.to(q.device) * s).contiguous()     # act * weight * folded BN
            self._fp8_cache = (key, (q, ws, torch.ones_like(s), torch.zeros_like(s)))
        return self._fp8_cache[1]

    @property
    def w8(self):
        """Per-tensor mode: e4m3 weights [Cout, Cin] (None in the other modes)."""
        return self._fp8_weights()[0] if self._fp8 == "tensor" else None

    @property
    def deq_scale(self):
        return self._fp8_weights()[1] if self._fp8 == "tensor" else None

    @property
    def w8_blocks(self):
        """Block mode: e4m3 weights [Cout, Cin] (None in the other modes)."""
        return self._fp8_weights()[0] if self._fp8 == "block" else None

    @property
    def w_block_scales(self):
        return self._fp8_weights()[1] if self._fp8 == "block" else None

    def forward(self, x, residual=None):
        fast = (x.is_cuda and x.dtype == torch.bfloat16 and self.k == 1 and self.groups == 1
                and self.cin % 8 == 0 and self.cout % 8 == 0)
        if getattr(self, "_amax", None) is not None and self.fp8_eligible():
            self._amax.copy_(torch.maximum(self._amax, x.detach().float().abs().max()))
        if fast:
            if self.stride != 1:
                x = x[:, :, ::self.stride, ::self.stride].contiguous(memory_format=torch.channels_last)
            n, c, h, w = x.shape
            x2 = x.permute(0, 2, 3, 1).reshape(-1, c)
            y = torch.empty((n, self.cout, h, w), device=x.device, dtype=x.dtype, memory_format=torch.channels_last)
            y2 = y.permute(0, 2, 3, 1).reshape(-1, self.cout)
            if self._fp8 == "block":
                from ..ops.fp8 import gemm_fp8_blockscaled, quantize_e4m3_blocks

                w8, sb, ones, zeros = self._fp8_weights()
                x8, sa = quantize_e4m3_blocks(x2)
                if residual is None:
                    gemm_fp8_blockscaled(x8, sa, w8, sb, self.scale, self.shift, self.relu, out=y2)
                    return y
                gemm_fp8_blockscaled(x8, sa, w8, sb, self.scale, self.shift, False, out=y2)
                return ops.scale_shift_act(y, ones, zeros, residual, self.relu)
            if self._fp8 == "tensor":
                from ..ops.fp8 import gemm_fp8, quantize_e4m3

                w8, deq_scale, ones, zeros = self._fp8_weights()
                x8 = quantize_e4m3(x2, self.act_scale)
                if residual is None:
                    gemm_fp8(x8, w8, deq_scale, self.shift, self.relu, out=y2)
                    return y
                gemm_fp8(x8, w8, deq_scale, self.shift, False, out=y2)
                return ops.scale_shift_act(y, ones, zeros, residual, self.relu)
            if residual is None:
                ops.gemm_bf16(x2, self.weight.view(self.cout, self.cin), out=y2, col_scale=self.scale,
                              col_shift=self.shift, relu=self.relu)
                return y
            if FUSE_RESIDUAL and self._residual_fusable(residual, y):
                # y = relu(x W'^T + residual + shift) in ONE kernel: the folded-BN scale lives in the weights
                # (W' = scale[:, None] * W), the residual tile is fetched by TMA into the epilogue's staging
                # buffer (the addend path of the persistent GEMM) -- no separate scale/shift/add/ReLU pass
                ops.gemm_bf16(x2, self._scaled_weight(), out=y2, col_shift=self.shift, relu=self.relu,
                              add=residual.permute(0, 2, 3, 1).reshape(-1, self.cout))
                return y
            ops.gemm_bf16(x2, self.weight.view(self.cout, self.cin), out=y2)
            return ops.scale_shift_act(y, self.scale, self.shift, residual, self.relu)
        if self.k == 3 and residual is None and self.own_conv3 and self.groups > 1 and x.is_cuda:
            wide = self._widened_groups()
            if wide is not None:
                # 16 / 32 channels per group (ResNeXt101_32x16d stages 1-2): four / two neighbouring groups share one
                # 64-channel block-diagonal group, so the 64-wide k-blocks of the wgmma kernel apply (zeros in the
                # off-diagonal blocks: 4x / 2x the MMAs of layers that are memory-bound anyway)
                w64, g64 = wide
                if self.stride == 2 and ops.gemm.CONV3_S2 and ops.conv3x3_s2_supported(x, w64, g64):
                    return ops.conv3x3_s2_infer(x, w64, self.scale, self.shift, self.relu, g64)
                if self.stride in (1, 2) and ops.conv3x3_infer_supported(x, w64, g64):
                    y = ops.conv3x3_infer(x, w64, self.scale, self.shift, self.relu, g64)
                    if self.stride == 2:
                        y = y[:, :, ::2, ::2].contiguous(memory_format=torch.channels_last)
                    return y
        if (self.k == 3 and residual is None and self.own_conv3 and self.stride == 2 and ops.gemm.CONV3_S2
                and ops.conv3x3_s2_supported(x, self.weight, self.groups)):
            # experimental (EDL_CONV3_S2=1): true stride-2 kernel, a quarter of the MMAs of the path below
            return ops.conv3x3_s2_infer(x, self.weight, self.scale, self.shift, self.relu, self.groups)
        if (self.k == 3 and residual is None and self.own_conv3 and self.stride in (1, 2)
                and ops.conv3x3_infer_supported(x, self.weight, self.groups)):
            # dense or grouped 3x3 on the persistent wgmma kernel, folded BN + ReLU in its epilogue
            y = ops.conv3x3_infer(x, self.weight, self.scale, self.shift, self.relu, self.groups)
            if self.stride == 2:
                # 3x3 / pad 1 / stride 2 == the stride-1 result sampled at even positions.  4x the MMA work
                # of a strided kernel
                y = y[:, :, ::2, ::2].contiguous(memory_format=torch.channels_last)
            return y
        if (self.k == 7 and self.stride == 2 and self.groups == 1 and residual is None and OWN_STEM7
                and ops.stem7_supported(x, self.weight)):
            return ops.stem7_infer(x, self.weight, self.scale, self.shift, self.relu)
        if x.is_cuda:
            ops.count_fallback("teacher conv on cuDNN: %dx%d stride %d groups %d, %d -> %d channels" % (
                self.k, self.k, self.stride, self.groups, self.weight.shape[3] * self.groups, self.weight.shape[0]))
        y = F.conv2d(x, self.weight.permute(0, 3, 1, 2), None, self.stride, (self.k - 1) // 2, 1, self.groups)
        return ops.scale_shift_act(y, self.scale, self.shift, residual, self.relu)


# On by default (EDL_TEACHER_FUSE_RES=0: off): folds the residual add
# of every block's last 1x1 convolution into its GEMM epilogue.
FUSE_RESIDUAL = __import__("os").environ.get("EDL_TEACHER_FUSE_RES", "1") == "1"
# 7x7 stem as im2col + wgmma GEMM instead of the library convolution (EDL_TEACHER_OWN_STEM7=0: library)
OWN_STEM7 = __import__("os").environ.get("EDL_TEACHER_OWN_STEM7", "1") == "1"


class ResNeXtBlock(nn.Module):
    def __init__(self, cin, planes, stride, groups, width_per_group, downsample):
        super().__init__()
        width = int(planes * (width_per_group / 64.0)) * groups
        cout = planes * 4
        self.c1 = FoldedConv(cin, width, 1)
        self.c2 = FoldedConv(width, width, 3, stride, groups)
        self.c3 = FoldedConv(width, cout, 1, relu=True)           # ReLU after the residual add
        self.ds = FoldedConv(cin, cout, 1, stride, relu=False) if downsample else None

    def forward(self, x):
        s = self.ds(x) if self.ds is not None else x
        return self.c3(self.c2(self.c1(x)), residual=s)


class ResNeXt(nn.Module):
    def __init__(self, depths: List[int], groups=32, width_per_group=16, class_dim=1000, base=64):
        super().__init__()
        self.stem = FoldedConv(3, base, 7, 2)
        blocks, cin = [], base
        for stage, n in enumerate(depths):
            planes = base << stage
            for i in range(n):
                stride = 2 if (i == 0 and stage > 0) else 1
                blocks.append(ResNeXtBlock(cin, planes, stride, groups, width_per_group, downsample=(i == 0)))
                cin = planes * 4
        self.blocks = nn.Sequential(*blocks)
        self.fc_weight = nn.Parameter(torch.empty(class_dim, cin), requires_grad=False)
        self.fc_bias = nn.Parameter(torch.zeros(class_dim, dtype=torch.float32), requires_grad=False)
        nn.init.uniform_(self.fc_weight, -1.0 / math.sqrt(cin), 1.0 / math.sqrt(cin))

    @torch.no_grad()
    def enable_fp8(self, calib_batch: Optional[torch.Tensor] = None, margin: float = 1.0, scaling: str = "tensor") -> int:
        """Switch every eligible 1x1 convolution to the e4m3 wgmma GEMM.  Returns the number of converted layers.

        ``scaling="tensor"``: calibrate one activation scale per layer on ``calib_batch`` (one bf16 forward).
        ``scaling="block"``: per-128-channel-block activation scales computed from each block's own max|x| when
        the layer runs, per-128x128-block weight scales; needs no batch, runs no forward and never syncs."""
        convs = [m for m in self.modules() if isinstance(m, FoldedConv)]
        if scaling == "block":
            return sum(1 for c in convs if c.enable_fp8_blocks())
        if scaling != "tensor":
            raise ValueError("enable_fp8: scaling must be 'tensor' or 'block', got %r" % (scaling,))
        if calib_batch is None:
            raise ValueError("enable_fp8(scaling='tensor') needs a calibration batch")
        for c in convs:
            c._fp8 = None                                   # calibrate on the bf16 forward
            c.begin_calibration()
        self.forward_features(calib_batch)
        return sum(1 for c in convs if c.finish_calibration(margin))

    @torch.no_grad()
    def forward_features(self, x):
        """Everything up to the classifier: pooled [N, feat] features (the distill link fuses the FC
        GEMM with the NVLink ship of its output, distill/device_feed.py:ship_linear)."""
        x = self.stem(x)
        x = ops.max_pool_3x3_s2(x) if x.is_cuda else F.max_pool2d(x, 3, 2, 1)
        x = self.blocks(x)
        return ops.global_avg_pool(x)

    @torch.no_grad()
    def forward(self, x, return_logits=True):
        x = self.forward_features(x)
        if x.is_cuda and x.dtype == torch.bfloat16:
            logits = ops.gemm_bf16(x, self.fc_weight, col_shift=self.fc_bias)
        else:
            logits = F.linear(x, self.fc_weight, self.fc_bias.to(x.dtype))
        return logits if return_logits else torch.softmax(logits.float(), -1)


def ResNeXt101_32x16d(class_dim=1000):
    """The WSL teacher: 194 M parameters, 72.3 GFLOP / image at 224x224."""
    return ResNeXt([3, 4, 23, 3], 32, 16, class_dim)


def ResNeXt50_32x4d(class_dim=1000):
    return ResNeXt([3, 4, 6, 3], 32, 4, class_dim)


def ResNeXt_tiny(class_dim=16):
    """2-2-2-2 / 8 groups x 4: unit-test sized."""
    return ResNeXt([1, 1, 1, 1], 8, 4, class_dim, base=32)


def to_inference_dtype(model, dtype=torch.bfloat16, device=None):
    for m in model.modules():
        for name, p in list(m.named_parameters(recurse=False)):
            keep = name.endswith("bias")
            p.data = p.data.to(device=device, dtype=torch.float32 if keep else dtype)
        for name, b in list(m.named_buffers(recurse=False)):
            m._buffers[name] = b.to(device=device)
    return model.eval()
