#!/usr/bin/env python
"""Teacher (ResNeXt101_32x16d) forward time and per-kernel breakdown.

    python tools/teacher_prof.py [--fp8 [--fp8-scaling tensor|block]] [--batch 32]
    python tools/teacher_prof.py --modes bf16,fp8-tensor,fp8-block --batch 16,32 --rounds 5

With several modes, one model per mode (same seeded weights) is captured in a CUDA graph and the modes are
timed in turn, ``--rounds`` times, so that drift of the shared machine hits all of them alike; the median and
minimum ms per batch are reported, then a torch.profiler kernel table per mode.  tensor-fp8 calibrates on the
random input batch, as teacher_server --fp8 does."""
import argparse
import copy
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from edl_b200.models.resnext import ResNeXt101_32x16d, to_inference_dtype  # noqa: E402

MODES = ("bf16", "fp8-tensor", "fp8-block")

ap = argparse.ArgumentParser()
ap.add_argument("--fp8", action="store_true", help="single mode: fp8 1x1 convolutions (see --fp8-scaling)")
ap.add_argument("--fp8-scaling", choices=("tensor", "block"), default="tensor")
ap.add_argument("--modes", default=None, help="comma-separated subset of %s, timed alternately" % (",".join(MODES),))
ap.add_argument("--batch", default="32", help="batch size, or a comma-separated list")
ap.add_argument("--rounds", type=int, default=1, help="timing windows per mode (alternating)")
ap.add_argument("--iters", type=int, default=10, help="forwards per timing window")
ap.add_argument("--no-graph", action="store_true")
ap.add_argument("--no-profile", action="store_true")
args = ap.parse_args()
if args.modes is not None:
    modes = args.modes.split(",")
    for md in modes:
        if md not in MODES:
            ap.error("unknown mode %r" % (md,))
else:
    modes = ["fp8-" + args.fp8_scaling if args.fp8 else "bf16"]
dev = "cuda"

smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
print("gpu:", smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name())

torch.manual_seed(0)
base = ResNeXt101_32x16d()
models = {}
for md in modes:
    models[md] = to_inference_dtype(copy.deepcopy(base) if len(modes) > 1 else base, torch.bfloat16, dev).eval()
del base
enabled = set()   # fp8 modes are switched on (tensor mode: calibrated) with the first batch only


def run_batch(batch):
    torch.manual_seed(1)
    x = torch.randn(batch, 3, 224, 224, device=dev).bfloat16().contiguous(memory_format=torch.channels_last)
    runs, outs = {}, {}
    with torch.no_grad():
        for md in modes:
            m = models[md]
            if md not in enabled and md == "fp8-tensor":
                print("%s layers: %d" % (md, m.enable_fp8(x)))
            elif md not in enabled and md == "fp8-block":
                print("%s layers: %d" % (md, m.enable_fp8(scaling="block")))
            enabled.add(md)
            for _ in range(3):
                m(x)
            torch.cuda.synchronize()
            if args.no_graph:
                runs[md] = (lambda m=m: m(x))
                outs[md] = m(x)
            else:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    y = m(x)
                runs[md] = g.replay
                g.replay()
                outs[md] = y
            torch.cuda.synchronize()
        if "bf16" in outs:
            ref = outs["bf16"].float()
            for md in modes:
                if md != "bf16":
                    o = outs[md].float()
                    cos = torch.nn.functional.cosine_similarity(o.flatten(), ref.flatten(), dim=0).item()
                    top1 = (o.argmax(-1) == ref.argmax(-1)).float().mean().item()
                    print("%s vs bf16 logits: cosine %.5f, top-1 agreement %.3f" % (md, cos, top1))
        times = {md: [] for md in modes}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for md in modes:
                run = runs[md]
                run()
                e0.record()
                for _ in range(args.iters):
                    run()
                e1.record()
                torch.cuda.synchronize()
                times[md].append(e0.elapsed_time(e1) / args.iters)
        for md in modes:
            med, mn = statistics.median(times[md]), min(times[md])
            print("batch %d %-10s forward median %.2f ms (min %.2f) = %.0f img/s, %.0f TFLOP/s" % (
                batch, md, med, mn, batch / med * 1e3, 72.3e9 * batch / med / 1e9))
        if not args.no_profile:
            from torch.profiler import ProfilerActivity, profile
            for md in modes:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(3):
                        runs[md]()
                    torch.cuda.synchronize()
                print("== batch %d %s ==" % (batch, md))
                print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25, max_name_column_width=100))
    del runs, outs
    torch.cuda.empty_cache()


for b in [int(v) for v in args.batch.split(",")]:
    run_batch(b)
