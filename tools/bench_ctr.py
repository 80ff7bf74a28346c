#!/usr/bin/env python
"""Dense against row-sparse embedding gradients for the CTR models on one GPU.

Both CTR-DNN and DeepFM are built twice at the reference's size (26 tables of [vocab, 10] fp32, batch 1000, one id
per slot), once with dense table gradients (the default: misc.cu scatter into a [V, D] gradient, FlatAdam over every
row) and once with ``sparse_grad=True`` (embedding.cu: row-sparse gradient, ``ops.SparseAdam`` over the looked-up
rows).  The two variants run in the same process, alternated round by round, on the same pre-generated batches; every
step (zero_grad, forward, backward, finish, optimizer) is timed with CUDA events after warm-up and the median is
reported per model and path, with the card name and its power limit.  The byte counts beside the times are computed
from shapes, not measured.

    python tools/bench_ctr.py [--steps 30] [--warmup 5] [--rounds 3] [--vocab 1000001] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from edl_b200 import ops  # noqa: E402
from edl_b200.models.ctr_dnn import CtrDnn, DeepFM  # noqa: E402
from edl_b200.parallel import ElasticDataParallel  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def shape_bytes(model, sparse, batch):
    """Per-step bytes of the embedding tables, from shapes.  Dense: the fp32 [V, D] gradient of every table is zeroed in
    the flat buffer, zeroed again as the kernel's scatter target and added into the flat buffer (5 passes), and Adam
    reads gradient, weights, m, v and writes weights, m, v (7 passes); on several ranks the whole gradient is
    all-reduced.  Sparse: one index (8 B) and one row (4 D B) per looked-up element; the optimizer reads and writes
    weights, m, v of at most that many rows (6 row passes) besides the gradient; on several ranks that gradient is what
    one rank contributes to the all-gather."""
    tables = [p for n, p in model.named_parameters() if n.startswith(("tables.", "first_order."))]
    uses = model.num_sparse // len(model.tables)
    if not sparse:
        tb = sum(p.numel() * 4 for p in tables)
        return {"table_grad_bytes": 5 * tb, "optimizer_bytes": 7 * tb, "exchanged_bytes_per_rank": tb}
    grad = sum(uses * batch * (8 + 4 * p.shape[1]) for p in tables)
    rows = sum(uses * batch * 4 * p.shape[1] for p in tables)
    return {"table_grad_bytes": grad, "optimizer_bytes": grad + 6 * rows, "exchanged_bytes_per_rank": grad}


class Runner:
    def __init__(self, cls, sparse, vocab, dev):
        torch.manual_seed(0)
        self.model = cls(sparse_feature_dim=vocab, sparse_grad=sparse).to(dev)
        self.dp = ElasticDataParallel(self.model, bucket_cap_mb=64)
        self.opts = [ops.FlatAdam(self.dp.flat, lr=1e-4)]
        if sparse:
            self.opts.append(ops.SparseAdam(self.dp.sparse_params, lr=1e-4))

    def step(self, dense, ids, label):
        self.dp.zero_grad()
        loss = F.cross_entropy(self.dp(dense, ids), label)
        loss.backward()
        self.dp.finish()
        for o in self.opts:
            o.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--vocab", type=int, default=1000001)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ctr needs a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gen = torch.Generator(device=dev).manual_seed(1)
    data = []
    for _ in range(args.steps):
        dense = torch.rand(args.batch, 13, generator=gen, device=dev)
        ids = torch.randint(0, args.vocab, (args.batch, 26, 1), generator=gen, device=dev)
        data.append((dense, ids, ((ids[:, 0, 0] % 2 == 1) ^ (dense[:, 0] > 0.5)).long()))
    result = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "batch": args.batch,
              "vocab": args.vocab, "steps": args.steps, "rounds": args.rounds, "models": {}}
    for name, cls in (("ctr_dnn", CtrDnn), ("deepfm", DeepFM)):
        runners = {"dense": Runner(cls, False, args.vocab, dev), "sparse": Runner(cls, True, args.vocab, dev)}
        times = {k: [] for k in runners}
        for k, r in runners.items():
            for i in range(args.warmup):
                r.step(*data[i % len(data)])
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for k, r in runners.items():
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
                ev[0].record()
                for i in range(args.steps):
                    r.step(*data[i])
                    ev[i + 1].record()
                torch.cuda.synchronize()
                times[k] += [ev[i].elapsed_time(ev[i + 1]) for i in range(args.steps)]
        entry = {}
        for k, r in runners.items():
            entry[k] = {"step_ms_median": statistics.median(times[k]), "step_ms_min": min(times[k]),
                        **shape_bytes(r.model, k == "sparse", args.batch)}
        entry["speedup"] = entry["dense"]["step_ms_median"] / entry["sparse"]["step_ms_median"]
        result["models"][name] = entry
        print("%-8s dense %.3f ms/step  sparse %.3f ms/step  (x%.1f)" % (
            name, entry["dense"]["step_ms_median"], entry["sparse"]["step_ms_median"], entry["speedup"]), flush=True)
        del runners
        torch.cuda.empty_cache()
    print(json.dumps(result))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
