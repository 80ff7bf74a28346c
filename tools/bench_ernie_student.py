#!/usr/bin/env python
"""Time the Transformer student (models/ernie.py ErnieStudent) on one GPU: one training step (forward, backward,
AdamW) at B = 32, L = 128 with the student configuration (hidden 384, 4 layers, 6 heads, FFN 1536, vocabulary 18000)
on the package's kernels, against the same bf16 model in torch (cuBLAS linears, F.scaled_dot_product_attention with
the key mask, F.layer_norm, F.gelu), both as CUDA-graph replays; and the attention backward alone against SDPA's
backward, eager.  With ``--dropout p`` it times instead three training steps with hidden and attention dropout: ours at
p, ours at 0, and the bf16 torch model with F.dropout at the same sites and SDPA's dropout_p = p.  With ``--packed
MIN_LEN`` the sample lengths are drawn uniformly from [MIN_LEN, seq] (fixed seed) and it times three steps on that
batch and the same weights: ours padded (``forward``), ours packed (``forward_packed`` on ``pack_sequences`` of the
batch) and torch padded; it also reports the real-token fraction and the host time of ``pack_sequences`` per batch.
All GPU times come from CUDA events.  Prints the GPU name and power limit with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from edl_b200 import ops  # noqa: E402
from edl_b200.models.ernie import ernie_student, pack_sequences  # noqa: E402


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def torch_encoder(m, ids, keep, p=0.0):
    """The student's layers in bf16 torch: cuBLAS linears, SDPA with the key mask, F.layer_norm, F.gelu; with p > 0,
    F.dropout at ErnieStudent's hidden sites and SDPA's dropout_p = p on the probabilities."""
    b, l = ids.shape
    c, nh = m.hidden, m.heads
    d = (lambda t: F.dropout(t, p, True)) if p > 0 else (lambda t: t)
    pos = torch.arange(l, device=ids.device)
    x = F.embedding(ids, m.word_emb) + F.embedding(pos, m.pos_emb) + m.seg_emb[0]
    x = d(F.layer_norm(x, (c,), m.emb_ln_g, m.emb_ln_b, m.eps))
    am = keep.view(b, 1, 1, l)
    for lyr in m.layers:
        q, k, v = F.linear(x, lyr.qkv_w, lyr.qkv_b).view(b, l, 3, nh, c // nh).unbind(2)
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=am,
                                           dropout_p=p)
        x = F.layer_norm(d(F.linear(o.transpose(1, 2).reshape(b, l, c), lyr.out_w, lyr.out_b)) + x, (c,), lyr.ln1_g,
                         lyr.ln1_b, m.eps)
        x = F.layer_norm(d(F.linear(F.gelu(F.linear(x, lyr.ffn1_w, lyr.ffn1_b)), lyr.ffn2_w, lyr.ffn2_b)) + x, (c,),
                         lyr.ln2_g, lyr.ln2_b, m.eps)
    return F.linear(d(torch.tanh(F.linear(x[:, 0], m.pool_w, m.pool_b))), m.cls_w, m.cls_b).float()


def graph_time(fn, warmup, iters):
    """Milliseconds per replay of ``fn`` captured in a CUDA graph (after ``warmup`` eager calls on a side stream)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(warmup):
        g.replay()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / iters


def event_time(fn, warmup, iters):
    """Milliseconds per eager call of ``fn``, CUDA events around ``iters`` calls."""
    for _ in range(warmup):
        fn()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return a.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--seq", type=int, default=128)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--dropout", type=float, default=None, help="time training steps with this dropout instead")
    ap.add_argument("--packed", type=int, default=None, metavar="MIN_LEN",
                    help="lengths uniform in [MIN_LEN, seq]: time the padded step, the packed step and torch")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ernie_student: needs a GPU")
    if args.packed is not None and not 1 <= args.packed <= args.seq:
        sys.exit("bench_ernie_student: --packed MIN_LEN needs 1 <= MIN_LEN <= --seq")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    b, l = args.batch, args.seq
    ids = torch.randint(1, 18000, (b, l), device=dev)
    if args.packed is None:
        lens = torch.randint(l // 2, l + 1, (b, 1), device=dev)
    else:                                                # a fixed batch whatever the device's RNG state
        lens = torch.randint(args.packed, l + 1, (b, 1), generator=torch.Generator().manual_seed(1234)).to(dev)
    ids[torch.arange(l, device=dev).unsqueeze(0) >= lens] = 0
    label = torch.randint(0, 2, (b,), device=dev)
    keep = ids != 0

    ours = ernie_student().to(dev)
    opt = torch.optim.AdamW(ours.parameters(), 1e-4, capturable=True)
    ref = ernie_student().to(dev).to(torch.bfloat16)
    ref.load_state_dict({k: v.to(torch.bfloat16) for k, v in ours.state_dict().items()})
    ropt = torch.optim.AdamW(ref.parameters(), 1e-4, capturable=True)

    def step_ours():
        opt.zero_grad(set_to_none=False)
        F.cross_entropy(ours(ids), label).backward()
        opt.step()

    def step_torch():
        ropt.zero_grad(set_to_none=False)
        F.cross_entropy(torch_encoder(ref, ids, keep), label).backward()
        ropt.step()

    if args.dropout is not None:
        return bench_dropout(args, ours, opt, ref, ropt, ids, label, keep)
    if args.packed is not None:
        return bench_packed(args, ours, opt, step_ours, step_torch, ids, label)
    ops.reset_fallbacks()
    t_ours = graph_time(step_ours, args.warmup, args.iters)
    fallbacks = ops.fallbacks()
    t_torch = graph_time(step_torch, args.warmup, args.iters)

    # attention backward alone: one layer's shapes
    h = 6
    qkv = torch.randn(b * l, 3 * h * 64, device=dev).to(torch.bfloat16)
    mask = keep.to(torch.uint8).contiguous()
    do = torch.randn(b * l, h * 64, device=dev).to(torch.bfloat16)
    out, lse = ops.transformer.attention_forward_saved(qkv, mask, b, l, h)
    t_abwd = event_time(lambda: ops.transformer.attention_backward(qkv, mask, out, lse, do, b, l, h),
                        args.warmup, args.iters * 4)
    q, k, v = (qkv.view(b, l, 3, h, 64)[:, :, i].transpose(1, 2).detach().requires_grad_(True) for i in range(3))
    o = F.scaled_dot_product_attention(q, k, v, attn_mask=keep.view(b, 1, 1, l))
    g_o = do.view(b, l, h, 64).transpose(1, 2)
    t_sdpa = event_time(lambda: torch.autograd.grad(o, (q, k, v), g_o, retain_graph=True), args.warmup,
                        args.iters * 4)
    name, limit = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": limit, "batch": b, "seq": l,
                      "train_step_ms": {"ours": round(t_ours, 3), "torch_bf16": round(t_torch, 3)},
                      "attention_bwd_us": {"ours": round(t_abwd * 1e3, 1), "sdpa": round(t_sdpa * 1e3, 1)},
                      "fallbacks": fallbacks}))


def bench_dropout(args, ours, opt, ref, ropt, ids, label, keep):
    """Training steps with dropout p against the same steps at p = 0 and against torch with dropout, CUDA-graph
    replays, the three alternated over five rounds (the median of each is printed)."""
    p = args.dropout

    def step_ours(q):
        def fn():
            ours.hidden_dropout = ours.attention_dropout = q
            opt.zero_grad(set_to_none=False)
            F.cross_entropy(ours(ids), label).backward()
            opt.step()
        return fn

    def step_torch():
        ropt.zero_grad(set_to_none=False)
        F.cross_entropy(torch_encoder(ref, ids, keep, p), label).backward()
        ropt.step()

    ops.reset_fallbacks()
    arms = {"ours_p": step_ours(p), "ours_0": step_ours(0.0), "torch_bf16_p": step_torch}
    times = {k: [] for k in arms}
    for _ in range(5):
        for k, fn in arms.items():
            times[k].append(graph_time(fn, args.warmup, args.iters))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    name, limit = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": limit, "batch": args.batch, "seq": args.seq, "dropout": p,
                      "train_step_ms": {k: round(v, 3) for k, v in med.items()},
                      "dropout_overhead": round(med["ours_p"] / med["ours_0"] - 1.0, 4),
                      "fallbacks": ops.fallbacks()}))


def bench_packed(args, ours, opt, step_ours, step_torch, ids, label):
    """The padded step, the packed step and torch's padded step on one batch, CUDA-graph replays alternated over five
    rounds (medians); the packed step's graph is fixed to this batch's T and cu_seqlens."""
    b, l = ids.shape
    feeds = (ids.cpu(), torch.arange(l).expand(b, l), torch.zeros(b, l, dtype=torch.int64), (ids != 0).cpu())
    n_pack = 200
    t0 = time.perf_counter()
    for _ in range(n_pack):
        pk = pack_sequences(*feeds)
    pack_ms = (time.perf_counter() - t0) * 1e3 / n_pack
    dev = ids.device
    pk = tuple(t.to(dev) if torch.is_tensor(t) else t for t in pk)
    tokens = pk[0].numel()

    def step_packed():
        opt.zero_grad(set_to_none=False)
        F.cross_entropy(ours.forward_packed(*pk), label).backward()
        opt.step()

    ops.reset_fallbacks()
    arms = {"ours_padded": step_ours, "ours_packed": step_packed, "torch_bf16_padded": step_torch}
    times = {k: [] for k in arms}
    for _ in range(5):
        for k, fn in arms.items():
            times[k].append(graph_time(fn, args.warmup, args.iters))
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    name, limit = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": limit, "batch": b, "seq": l, "min_len": args.packed,
                      "tokens": tokens, "token_fraction": round(tokens / (b * l), 4),
                      "train_step_ms": {k: round(v, 3) for k, v in med.items()},
                      "packed_speedup_vs_padded": round(med["ours_padded"] / med["ours_packed"], 3),
                      "pack_sequences_host_ms": round(pack_ms, 3), "fallbacks": ops.fallbacks()}))


if __name__ == "__main__":
    main()
