"""The BiLSTM student's recurrent layer: ``ops.lstm`` (csrc/lstm.cu) against ``torch.nn.LSTM`` (cuDNN), same device.

    python tools/bench_lstm.py                 # H = E = 128, B in {32, 128}, L in {64, 128, 256}: one JSON line each

Workload: one bidirectional layer, right-padded batches whose lengths come from a fixed seed in [L/4, L].  "ours" is
``ops.lstm`` on bf16 inputs; "cudnn" is ``nn.LSTM`` over ``pack_padded_sequence(enforce_sorted=False)`` with the same
weights in bf16 (fp16 when the library refuses bf16 for RNNs; the line says which).  Both arms are CUDA-graph replays
of the forward alone and of forward + backward (gradients of sum(y * w) + sum(h_n * w')), timed in alternating
device-timed windows; the median window is reported as microseconds per time step (per L).  Agreement: the largest
absolute difference of y and h_n between the arms."""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from edl_b200 import ops  # noqa: E402

H = E = 128


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit"] = q[0].strip()
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def graph(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn()
    return g, out


def time_alternating(graphs, windows, reps):
    """Median over ``windows`` of the device time of ``reps`` back-to-back replays, arms alternating per window."""
    res = {k: [] for k in graphs}
    for _ in range(windows):
        for k, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                g.replay()
            b.record()
            b.synchronize()
            res[k].append(a.elapsed_time(b) * 1e3 / reps)
    return {k: sorted(v)[len(v) // 2] for k, v in res.items()}


def cudnn_dtype(lstm, x, lengths):
    for dt in (torch.bfloat16, torch.float16):
        try:
            m = lstm.to(dt)
            m.flatten_parameters()          # one contiguous weight buffer: no compaction inside each call
            pk = pack_padded_sequence(x.to(dt), lengths.cpu(), batch_first=True, enforce_sorted=False)
            m(pk)
            torch.cuda.synchronize()
            return m, dt
        except RuntimeError:
            continue
    raise RuntimeError("nn.LSTM accepts neither bf16 nor fp16 on this device")


def run(b, L, windows, reps):
    dev = torch.device("cuda", 0)
    gen = torch.Generator().manual_seed(b * 1000 + L)
    lengths = torch.randint(L // 4, L + 1, (b,), generator=gen).to(dev)
    torch.manual_seed(0)
    ref = torch.nn.LSTM(E, H, batch_first=True, bidirectional=True).to(dev)
    with torch.no_grad():
        for p in ref.parameters():
            p.copy_(p.to(torch.bfloat16))
    params = [p.detach().to(torch.bfloat16).clone().requires_grad_(True) for p in ref.parameters()]
    x = torch.randn(b, L, E, device=dev).to(torch.bfloat16)
    m, dt = cudnn_dtype(ref, x, lengths)
    xr = x.to(dt)
    wy = torch.randn(b, L, 2 * H, device=dev)
    wh = torch.randn(2, b, H, device=dev)
    len_cpu = lengths.cpu()        # pack_padded_sequence takes host lengths (outside the graphs)

    def ours_fwd():
        with torch.no_grad():
            return ops.lstm(x, lengths, params)

    def ours_fb():
        xg = x.detach().requires_grad_(True)
        y, hn = ops.lstm(xg, lengths, params)
        torch.autograd.backward([y, hn], [wy.to(y.dtype), wh.to(hn.dtype)])
        return y, hn

    sorted_idx = torch.sort(lengths, descending=True).indices
    unsorted_idx = torch.argsort(sorted_idx)
    sorted_len = len_cpu[sorted_idx.cpu()]

    def cudnn(xx):
        # pack_padded_sequence(enforce_sorted=False) with its host-side sort done once, outside the graph: the graph
        # holds the device gather into length order, the packing, the LSTM, the unpacking and the gather back
        pk = pack_padded_sequence(xx.index_select(0, sorted_idx), sorted_len, batch_first=True)
        out, (hn, _) = m(pk)
        y, _ = pad_packed_sequence(out, batch_first=True, total_length=L)
        return y.index_select(0, unsorted_idx), hn.index_select(1, unsorted_idx)

    def cudnn_fwd():
        with torch.no_grad():
            return cudnn(xr)

    def cudnn_fb():
        xg = xr.detach().requires_grad_(True)
        y, hn = cudnn(xg)
        torch.autograd.backward([y, hn], [wy.to(y.dtype), wh.to(hn.dtype)])
        return y, hn

    ops.reset_fallbacks()
    gs, outs = {}, {}
    for k, fn in (("ours_fwd", ours_fwd), ("cudnn_fwd", cudnn_fwd), ("ours_fwd_bwd", ours_fb),
                  ("cudnn_fwd_bwd", cudnn_fb)):
        gs[k], outs[k] = graph(fn)
    t = time_alternating(gs, windows, reps)
    gs["ours_fwd"].replay()
    gs["cudnn_fwd"].replay()
    torch.cuda.synchronize()
    (y0, h0), (y1, h1) = outs["ours_fwd"], outs["cudnn_fwd"]
    return {
        "bench": "bilstm_layer", "card": card(), "B": b, "L": L, "E": E, "H": H,
        "lengths": "seeded in [L/4, L], mean %.1f" % float(lengths.float().mean()),
        "cudnn_dtype": str(dt).replace("torch.", ""),
        "us_per_step": {k: round(v / L, 3) for k, v in t.items()},
        "us_total": {k: round(v, 1) for k, v in t.items()},
        "fwd_ratio_cudnn_over_ours": round(t["cudnn_fwd"] / t["ours_fwd"], 3),
        "fwd_bwd_ratio_cudnn_over_ours": round(t["cudnn_fwd_bwd"] / t["ours_fwd_bwd"], 3),
        "max_abs_diff_y": float((y0.float() - y1.float()).abs().max()),
        "max_abs_diff_hn": float((h0.float() - h1.float()).abs().max()),
        "library_fallbacks": ops.fallbacks(),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, nargs="*", default=[32, 128])
    ap.add_argument("--lengths", type=int, nargs="*", default=[64, 128, 256])
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    for b in args.batch:
        for L in args.lengths:
            print(json.dumps(run(b, L, args.windows, args.reps)), flush=True)


if __name__ == "__main__":
    main()
