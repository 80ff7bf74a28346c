#!/usr/bin/env python
"""Measure the per-launch cost of back-to-back vs alternating kernels with different shared-memory
footprints inside CUDA graphs (is an L1/smem carveout re-partition taxing every kernel boundary?).

    python tools/launch_overhead.py [--policy]
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from edl_b200 import ops  # noqa: E402

if "--policy" in sys.argv:
    ops.native().set_smem_carveout_policy(True)
dev = "cuda"
N = 200
c = 256
x = torch.randn(32, c, 14, 14, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
x2 = x.permute(0, 2, 3, 1).reshape(-1, c)
y = torch.empty_like(x)
y2 = y.permute(0, 2, 3, 1).reshape(-1, c)
sums = torch.zeros(2 * c, device=dev)
C = ops.native()
C.bn_stats(x2, sums)
g, b = torch.ones(c, device=dev), torch.zeros(c, device=dev)
mean, rstd = torch.empty(c, device=dev), torch.empty(c, device=dev)
w = torch.randn(256, 256, device=dev).bfloat16()
out = torch.empty(x2.shape[0], 256, device=dev, dtype=torch.bfloat16)
t = torch.randn(1 << 20, device=dev)


def A():   # TMA-ring BN apply, 65 KB dynamic smem
    C.bn_apply(x2, None, y2, sums, g, b, None, None, mean, rstd, 1e-5, 0.1, True)


def B():   # plain elementwise, no smem
    t.add_(1.0)


def G():   # wgmma GEMM, 99 KB dynamic smem
    C.gemm_bf16(x2, w, out, False, False, None, None, False, None, None, None, False)


def D():   # cuDNN conv
    torch.nn.functional.conv2d(x, w.view(256, 256, 1, 1))


def timed(seq, name):
    for f in seq:
        f()
    torch.cuda.synchronize()
    gph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for f in seq:
            f()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    with torch.cuda.graph(gph):
        for _ in range(N // len(seq)):
            for f in seq:
                f()
    gph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        gph.replay()
    e1.record()
    torch.cuda.synchronize()
    per = e0.elapsed_time(e1) * 1e3 / (5 * (N // len(seq)) * len(seq))
    print("%-28s %7.2f us per kernel" % (name, per), flush=True)
    return per


print("policy prefer-max-shared:", "--policy" in sys.argv)
a = timed([A], "A x N  (bn_apply stream)")
b_ = timed([B], "B x N  (aten add_)")
g_ = timed([G], "G x N  (wgmma gemm)")
d_ = timed([D], "D x N  (cudnn conv1x1)")
ab = timed([A, B], "A,B alternating")
ag = timed([A, G], "A,G alternating")
gb = timed([G, B], "G,B alternating")
gd = timed([G, D], "G,D alternating")
print("expected A,B = %.2f  measured %.2f | expected A,G = %.2f measured %.2f | expected G,B %.2f measured %.2f | G,D exp %.2f meas %.2f" % (
    (a + b_) / 2, ab, (a + g_) / 2, ag, (g_ + b_) / 2, gb, (g_ + d_) / 2, gd))
