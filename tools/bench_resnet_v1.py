"""Plain ResNet50 (models/resnet.py) training step on our kernels against the same model on the library convolutions.

    python tools/bench_resnet_v1.py [--rounds 5] [--steps 50] [--batch 32] [--kineto PATH]

Two models from the same seed, ``impl="auto"`` (7x7 stem and 1x1 / stride-2 projections on the wgmma kernels) and
``impl="cudnn"``, each a ``StudentTrainer`` step captured in a CUDA graph on synthetic data, timed with CUDA events in
alternating rounds.  Prints one JSON line: ms / step (median and min over the rounds) and the peak memory each model's
step adds, with the card's name, power limit and maximum SM clock read in the same run.

``--kineto PATH``: a separate profiled pass over the layers this path owns -- the stem's fprop and weight gradient and
each projection's fprop, dgrad and weight gradient at the workload's shapes -- writing the per-call kernel time of our
kernels next to the library kernels they replace, with FLOPs and minimum bytes from the shapes and each kernel's share
of the bound that limits it (989 TFLOP/s dense BF16, 3.35 TB/s HBM3: H100 SXM data sheet)."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_FLOPS = 989e12
PEAK_BYTES = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True)
    name, power, clock = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def make_trainer(impl, batch, seed=0):
    import torch
    from edl_b200.models import to_train_dtype
    from edl_b200.models.resnet import ResNet
    from edl_b200.trainer import StudentTrainer

    torch.manual_seed(seed)
    m = to_train_dtype(ResNet(50, impl=impl), torch.bfloat16, "cuda").train()
    tr = StudentTrainer(m, batch_size=batch, image_shape=(3, 224, 224), num_classes=1000, lr=0.1, use_graph=True)
    g = torch.Generator(device="cuda").manual_seed(seed)
    tr.static_x.copy_(torch.randn(tr.static_x.shape, device="cuda", generator=g))
    tr.static_t.copy_(torch.softmax(torch.randn(tr.static_t.shape, device="cuda", generator=g), -1))
    return tr


def time_steps(tr, steps):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        tr.step_device()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


# ------------------------------------------------------------------------------------------------ per-layer pass
def layer_cases(batch):
    """(name, pass, flops, min_bytes, ours, library) at the workload's shapes; the callables take no argument."""
    import torch
    from edl_b200 import ops
    from edl_b200.ops import gemm as G

    C = ops.native()
    cl = torch.channels_last
    cases = []

    def conv_bwd(dy, x, w, stride, pad, mask):
        return lambda: torch.ops.aten.convolution_backward(dy, x, w, None, [stride] * 2, [pad] * 2, [1, 1], False, [0, 0],
                                                           1, mask)

    # 7x7 / stride 2 / pad 3 stem, 3 -> 64
    x = torch.randn(batch, 3, 224, 224, device="cuda").bfloat16().contiguous(memory_format=cl)
    w = (torch.randn(64, 7, 7, 3, device="cuda") * 0.05).bfloat16()
    wn = w.permute(0, 3, 1, 2).contiguous(memory_format=cl)
    m = batch * 112 * 112
    dy = torch.randn(batch, 64, 112, 112, device="cuda").bfloat16().contiguous(memory_format=cl)
    a = torch.empty((m, 160), device="cuda", dtype=torch.bfloat16)
    C.stem7_im2col(x, a)
    flops = 2.0 * m * 64 * 147
    # minimum bytes of ANY stem convolution: the image, the weight and the output once (the im2col route moves its
    # [M, 160] matrix on top: written and read in fprop, read again in the weight gradient)
    cases.append(("stem 7x7/2 3->64", "fprop", flops, x.numel() * 2 + w.numel() * 2 + m * 64 * 2,
                  lambda x=x, w=w: ops.stem7(x, w), lambda x=x, wn=wn: torch.nn.functional.conv2d(x, wn, None, 2, 3)))
    cases.append(("stem 7x7/2 3->64", "wgrad", flops, x.numel() * 2 + m * 64 * 2 + w.numel() * 2,
                  lambda dy=dy, a=a, w=w: G.stem7_wgrad(dy, a, w.shape), conv_bwd(dy, x, wn, 2, 3, [False, True, False])))
    # 1x1 / stride 2 projections of ResNet50
    for cin, cout, s in ((256, 512, 56), (512, 1024, 28), (1024, 2048, 14)):
        x = torch.randn(batch, cin, s, s, device="cuda").bfloat16().contiguous(memory_format=cl)
        w = (torch.randn(cout, 1, 1, cin, device="cuda") * 0.05).bfloat16()
        wn = w.permute(0, 3, 1, 2).contiguous(memory_format=cl)
        ho = s // 2
        dy = torch.randn(batch, cout, ho, ho, device="cuda").bfloat16().contiguous(memory_format=cl)
        dx = torch.empty_like(x)
        flops = 2.0 * batch * ho * ho * cin * cout
        xs, wb, yb = x.numel() * 2 // 4, w.numel() * 2, dy.numel() * 2      # the sampled quarter of x is all a pass needs
        name = "proj 1x1/2 %d->%d @%d" % (cin, cout, s)
        cases.append((name, "fprop", flops, xs + wb + yb, lambda x=x, w=w: ops.conv1x1_s2(x, w),
                      lambda x=x, wn=wn: torch.nn.functional.conv2d(x, wn, None, 2, 0)))
        cases.append((name, "dgrad", flops, yb + wb + x.numel() * 2,
                      lambda dy=dy, w=w, dx=dx: C.conv1x1_s2(dy, w, dx, True, None, None, None, False),
                      conv_bwd(dy, x, wn, 2, 0, [True, False, False])))
        cases.append((name, "wgrad", flops, xs + yb + wb, lambda x=x, dy=dy, w=w: G.conv1x1_s2_wgrad(x, dy, w.shape),
                      conv_bwd(dy, x, wn, 2, 0, [False, True, False])))
    return cases


def kernel_us(fn, reps):
    """Device time per call (us) of the kernels ``fn`` launches, and their names, from one profiled run of ``reps`` calls."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total, names = 0.0, {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0 and e.key and not e.key.startswith(("cudaDeviceSynchronize", "Activity Buffer")):
            total += t
            names[e.key] = names.get(e.key, 0.0) + t / reps
    return total / reps, names


def kineto_pass(path, batch, reps=20):
    rows = []
    lines = ["per-call kernel time at batch %d (torch.profiler, %d calls each); bound = max(FLOPs / 989 TFLOP/s, "
             "min bytes / 3.35 TB/s)" % (batch, reps), "",
             "%-28s %-6s %8s %9s %9s %9s %9s %8s %8s" % ("layer", "pass", "GFLOP", "min MB", "bound us", "ours us",
                                                          "lib us", "ours %", "lib %")]
    detail = []
    for name, what, flops, nbytes, ours, lib in layer_cases(batch):
        bound_us = max(flops / PEAK_FLOPS, nbytes / PEAK_BYTES) * 1e6
        limit = "compute" if flops / PEAK_FLOPS >= nbytes / PEAK_BYTES else "memory"
        t_o, k_o = kernel_us(ours, reps)
        t_l, k_l = kernel_us(lib, reps)
        rows.append({"layer": name, "pass": what, "gflop": flops / 1e9, "min_mb": nbytes / 1e6, "bound_us": bound_us,
                     "limit": limit, "ours_us": t_o, "lib_us": t_l, "ours_share": bound_us / t_o, "lib_share": bound_us / t_l})
        lines.append("%-28s %-6s %8.2f %9.1f %9.1f %9.1f %9.1f %7.0f%% %7.0f%%  (%s-bound)" % (
            name, what, flops / 1e9, nbytes / 1e6, bound_us, t_o, t_l, 100 * bound_us / t_o, 100 * bound_us / t_l, limit))
        detail.append("%s %s\n  ours:    %s\n  library: %s" % (name, what, "; ".join(
            "%s %.1f us" % (k[:70], v) for k, v in sorted(k_o.items(), key=lambda kv: -kv[1])), "; ".join(
            "%s %.1f us" % (k[:70], v) for k, v in sorted(k_l.items(), key=lambda kv: -kv[1]))))
    with open(path, "w") as fh:
        fh.write("\n".join(lines) + "\n\nkernels per call\n" + "\n".join(detail) + "\n")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--kineto", type=str, default="")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_resnet_v1 needs a CUDA device")
    from edl_b200 import ops

    info = card()
    trainers, peak = {}, {}
    for impl in ("auto", "cudnn"):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ops.reset_fallbacks()
        tr = make_trainer(impl, args.batch)
        tr.step_device()                              # warm-up steps, capture and one replay
        torch.cuda.synchronize()
        peak[impl] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        trainers[impl] = (tr, sorted(ops.fallbacks()))
    times = {impl: [] for impl in trainers}
    for _ in range(args.rounds):
        for impl, (tr, _) in trainers.items():
            times[impl].append(time_steps(tr, args.steps))
    out = {"card": info, "model": "ResNet50", "batch": args.batch, "rounds": args.rounds, "steps": args.steps}
    for impl, (tr, fb) in trainers.items():
        t = times[impl]
        out[impl] = {"ms_step_median": statistics.median(t), "ms_step_min": min(t), "ms_rounds": t,
                     "img_s_median": args.batch * 1000.0 / statistics.median(t), "peak_mib": peak[impl],
                     "library_convolutions": [k for k in fb if "conv" in k]}
    if args.kineto:
        del trainers
        torch.cuda.empty_cache()
        out["layers"] = kineto_pass(args.kineto, args.batch)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
