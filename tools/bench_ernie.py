"""ERNIE-base teacher forward: the package's kernels against the same bf16 weights on torch.

    python tools/bench_ernie.py                      # B = 16, L = 128 and 256, one JSON line per length
    python tools/bench_ernie.py --profile DIR        # separately: a torch.profiler per-kernel table (no timing)

Workload: ``ernie_base`` with random weights, batch 16, right-padded masks whose lengths come from a fixed seed (in
[L/4, L], the spread of a batch padded to its longest sample).  "ours" is a CUDA-graph replay of
``ErnieEncoder.forward`` on the wgmma GEMM (bias / residual / GELU epilogues), the attention, LayerNorm and
embedding-LayerNorm kernels; "packed" is a CUDA-graph replay of ``forward_packed`` on the same samples packed to their
real tokens (the varlen attention kernel, every other layer on T rows instead of B * L); "torch" is a CUDA-graph replay
of the padded forward in bf16 on cuBLAS linear, ``F.scaled_dot_product_attention`` and ``F.layer_norm``; "fp8" is a
CUDA-graph replay of ``forward_packed`` on a copy of the model after ``enable_fp8()`` (block-scaled e4m3 linear layers),
reported with its logits cosine and top-1 agreement against the bf16 packed arm (the classifier weights are scaled by 20
so that the random model's top-1 is decisive).  The four alternate in timed windows of device-timed replays.  FLOPs are counted from shapes: ``gflop`` over the full padded
length (what the padded forwards compute), ``gflop_real`` over the real tokens only (GEMM rows T, attention len_b^2 per
sequence), the work every arm has to do; the shares of peak are against the H100 SXM data-sheet dense bf16 rate
(989 TFLOP/s at 700 W), so they are end-to-end figures, not a kernel's."""
import argparse
import copy
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from edl_b200 import ops  # noqa: E402
from edl_b200.models import ernie  # noqa: E402

PEAK_BF16 = 989e12


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q[0].split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = "unknown (%s)" % type(e).__name__
    return info


def inputs(b, l, seed):
    gen = torch.Generator().manual_seed(seed)
    lens = torch.randint(l // 4, l + 1, (b,), generator=gen)
    mask = (torch.arange(l)[None] < lens[:, None]).float()
    ids = torch.randint(0, 18000, (b, l), generator=gen)
    seg = torch.zeros(b, l, dtype=torch.long)
    pos = torch.arange(l).expand(b, l).contiguous()
    return [t.cuda() for t in (ids, pos, seg, mask)]


def torch_forward(model):
    """The same forward in bf16 on the library, with the bf16 weights of the kernel path."""
    w = model._device_weights()
    word, pemb, semb, g0, b0 = w["emb"]
    c, h, eps = model.hidden, model.heads, model.eps
    bf = torch.bfloat16

    def fwd(ids, pos, seg, mask):
        b, l = ids.shape
        x = F.layer_norm(word[ids] + pemb[pos] + semb[seg], (c,), g0.to(bf), b0.to(bf), eps)
        keep = (mask != 0).view(b, 1, 1, l)
        for qkv_w, qkv_b, out_w, out_b, g1, be1, f1_w, f1_b, f2_w, f2_b, g2, be2 in w["layers"]:
            q, k, v = F.linear(x, qkv_w, qkv_b.to(bf)).view(b, l, 3, h, 64).permute(2, 0, 3, 1, 4)
            ctx = F.scaled_dot_product_attention(q, k, v, attn_mask=keep).transpose(1, 2).reshape(b, l, c)
            x = F.layer_norm(F.linear(ctx, out_w, out_b.to(bf)) + x, (c,), g1.to(bf), be1.to(bf), eps)
            x = F.layer_norm(F.linear(F.gelu(F.linear(x, f1_w, f1_b.to(bf))), f2_w, f2_b.to(bf)) + x, (c,), g2.to(bf),
                             be2.to(bf), eps)
        pool_w, pool_b, cls_w, cls_b = w["head"]
        pooled = torch.tanh(F.linear(x[:, 0], pool_w, pool_b.to(bf)))
        return F.linear(pooled, cls_w, cls_b.to(bf))[:, :model.num_labels].float()
    return fwd


def flops(model, b, l, lens=None):
    """(GEMM, attention) FLOPs of a batch of b sequences padded to l, or of the sequences of lengths ``lens`` alone."""
    c, f, n = model.hidden, model.layers[0].ffn1_w.shape[0], model.num_layers
    lens = [l] * b if lens is None else lens
    m = sum(lens)
    gemm = 2 * m * c * (3 * c + c + 2 * f) * n + 2 * b * c * (c + model.num_labels)
    attn = 4 * model.heads * sum(x * x for x in lens) * model.head_dim * n
    return gemm, attn


def split(avgs):
    """Device time (ms over the profiled replays) per kernel group of a profiler ``key_averages()``."""
    groups = (("fp8 GEMM, GELU -> e4m3 epilogue (FFN1)", ("gemm_fp8_wgmma_kernel", "Fp8BlockQParams")),
              ("fp8 GEMM, residual epilogue (out-proj, FFN2)", ("gemm_fp8_wgmma_kernel", ", 1>")),
              ("fp8 GEMM, bias epilogue (QKV)", ("gemm_fp8_wgmma_kernel",)),
              ("ctx quantiser", ("quantize_e4m3_blocks_kernel",)),
              ("LayerNorm (with e4m3 output)", ("layernorm_kernel<true>",)),
              ("LayerNorm", ("layernorm_kernel",)),
              ("bf16 GEMM", ("gemm",)),
              ("attention", ("attention",)))
    out = {}
    for e in avgs:
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if t <= 0:
            continue
        name = next((g for g, keys in groups if all(k in e.key for k in keys)), "other")
        out[name] = out.get(name, 0.0) + t / 1e3
    total = sum(out.values())
    return {k: {"ms": round(v, 4), "share": round(v / total, 4)} for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def capture(fn, args):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn(*args)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn(*args)
    return g, out


def timed(graph, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--lens", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--windows", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20, help="graph replays per timed window")
    ap.add_argument("--profile", default=None, help="directory: write a torch.profiler kernel table instead of timing")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ernie.py measures on a GPU; none found")
    torch.manual_seed(0)
    model = ernie.ernie_base().cuda().eval()
    with torch.no_grad():
        model.cls_w.mul_(20)                  # decisive logits for the FP8 arm's top-1 agreement
    model8 = copy.deepcopy(model)
    model8.enable_fp8()
    info = card()
    for l in args.lens:
        feed = inputs(args.batch, l, l)
        ops.reset_fallbacks()
        g_ours, out_ours = capture(model, feed)
        g_ref, out_ref = capture(torch.no_grad()(torch_forward(model)), feed)
        packed = ernie.pack_sequences(*(t.cpu() for t in feed))
        lens = packed[3].diff().tolist()
        packed = [p.cuda() if torch.is_tensor(p) else p for p in packed]
        g_pack, out_pack = capture(model.forward_packed, packed)
        g_fp8, out_fp8 = capture(model8.forward_packed, packed)
        g_ours.replay()
        g_ref.replay()
        g_pack.replay()
        g_fp8.replay()
        torch.cuda.synchronize()

        def cosine(a, b):
            return F.cosine_similarity(a.flatten()[None].double(), b.flatten()[None].double()).item()
        cos = cosine(out_ours, out_ref)
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            os.makedirs(args.profile, exist_ok=True)
            for name, g in (("ours", g_ours), ("packed", g_pack), ("torch", g_ref), ("fp8_packed", g_fp8)):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        g.replay()
                    torch.cuda.synchronize()
                avgs = prof.key_averages()
                table = avgs.table(sort_by="cuda_time_total", row_limit=25)
                with open(os.path.join(args.profile, "ernie_L%d_%s.txt" % (l, name)), "w") as fh:
                    fh.write(table)
                print("== L %d %s (5 replays) ==\n%s" % (l, name, table))
                print(json.dumps({"L": l, "arm": name, "card": info, "kernel_time_split": split(avgs)}), flush=True)
            continue
        for g in (g_ours, g_pack, g_ref, g_fp8):
            timed(g, 5)
        t_ours, t_pack, t_ref, t_fp8 = [], [], [], []
        for _ in range(args.windows):
            t_ours.append(timed(g_ours, args.reps))
            t_pack.append(timed(g_pack, args.reps))
            t_ref.append(timed(g_ref, args.reps))
            t_fp8.append(timed(g_fp8, args.reps))
        gemm, attn = flops(model, args.batch, l)
        real = sum(flops(model, args.batch, l, lens))
        best_o, best_p, best_r, best_8 = min(t_ours), min(t_pack), min(t_ref), min(t_fp8)
        med_o, med_p, med_r, med_8 = (sorted(t)[len(t) // 2] for t in (t_ours, t_pack, t_ref, t_fp8))
        print(json.dumps({
            "workload": "ernie_base forward, B %d, L %d, padded masks" % (args.batch, l),
            "card": info, "fallbacks": ops.fallbacks(), "logits_cosine_vs_torch": round(cos, 6),
            "real_tokens": sum(lens), "real_token_share": round(sum(lens) / (args.batch * l), 4),
            "packed_logits_cosine_vs_padded": round(cosine(out_pack, out_ours), 6),
            "packed_logits_max_abs_diff_vs_padded": float((out_pack - out_ours).abs().max()),
            "packed_logits_bitwise_equal_padded": bool(torch.equal(out_pack, out_ours)),
            "ours_seq_per_s": round(args.batch / med_o, 1), "packed_seq_per_s": round(args.batch / med_p, 1),
            "torch_seq_per_s": round(args.batch / med_r, 1),
            "ours_ms_median": round(med_o * 1e3, 4), "packed_ms_median": round(med_p * 1e3, 4),
            "torch_ms_median": round(med_r * 1e3, 4),
            "ours_ms_best": round(best_o * 1e3, 4), "packed_ms_best": round(best_p * 1e3, 4),
            "torch_ms_best": round(best_r * 1e3, 4),
            "speedup_median": round(med_r / med_o, 3), "packed_speedup_vs_padded_median": round(med_o / med_p, 3),
            "packed_speedup_vs_torch_median": round(med_r / med_p, 3),
            "gflop": round((gemm + attn) / 1e9, 2), "gemm_flop_share": round(gemm / (gemm + attn), 4),
            "gflop_real": round(real / 1e9, 2),
            "ours_tflops": round((gemm + attn) / med_o / 1e12, 1),
            "ours_share_of_bf16_peak": round((gemm + attn) / med_o / PEAK_BF16, 3),
            "torch_share_of_bf16_peak": round((gemm + attn) / med_r / PEAK_BF16, 3),
            "real_tflops": {k: round(real / t / 1e12, 1) for k, t in (("ours", med_o), ("packed", med_p),
                                                                      ("torch", med_r), ("fp8_packed", med_8))},
            "fp8_packed_seq_per_s": round(args.batch / med_8, 1), "fp8_packed_ms_median": round(med_8 * 1e3, 4),
            "fp8_packed_ms_best": round(best_8 * 1e3, 4),
            "fp8_speedup_vs_bf16_packed_median": round(med_p / med_8, 3),
            "fp8_logits_cosine_vs_bf16_packed": round(cosine(out_fp8, out_pack), 6),
            "fp8_top1_agreement_vs_bf16_packed": float((out_fp8.argmax(1) == out_pack.argmax(1)).float().mean()),
        }), flush=True)


if __name__ == "__main__":
    main()
