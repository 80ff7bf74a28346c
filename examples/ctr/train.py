#!/usr/bin/env python
"""CTR-DNN elastic data-parallel training + embedding all-reduce bandwidth sweep
(BASELINE.json config 4; reference workload: example/ctr/ctr/train.py -- CPU parameter-server mode,
network in example/ctr/ctr/save_program.py:75-144: 26 x embedding[1 000 001, 10] (avg-pooled) + 13
dense -> FC400 x3 -> FC2, Adam 1e-4, batch 1000, AUC).

Here the model trains on GPUs with the embedding tables replicated and their (dense) gradients
all-reduced by the fused NVSwitch kernels like any other parameter (26 x 40 MB fp32 = 1.04 GB per
step at the reference's table size -- the "embedding all-reduce bandwidth sweep").

With ``--sparse`` the tables are row-sparse instead (``sparse_grad=True``, the reference's ``is_sparse=True``): a
step only exchanges and updates the rows its batch looked up (all-gathered, ``ops.SparseAdam``).

    python examples/ctr/train.py --steps 20                    # 1 GPU / CPU smoke
    python examples/ctr/train.py --sparse --vocab 1000001      # row-sparse tables at the reference's size
    torchrun --nproc-per-node 8 examples/ctr/train.py --sweep  # all-reduce bus bandwidth vs message size
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from edl_b200 import ops  # noqa: E402
from edl_b200.models.ctr_dnn import CtrDnn, DeepFM, auc  # noqa: E402
from edl_b200.parallel import ElasticDataParallel  # noqa: E402


def synthetic_batch(batch, vocab, dev, gen):
    dense = torch.rand(batch, 13, generator=gen, device=dev)
    sparse = torch.randint(0, vocab, (batch, 26, 1), generator=gen, device=dev)
    # a learnable rule so AUC moves: click iff (slot0 id parity) xor (dense0 > 0.5)
    label = ((sparse[:, 0, 0] % 2 == 1) ^ (dense[:, 0] > 0.5)).long()
    return dense, sparse, label


def sweep(dev, world, rank):
    """Bus bandwidth of the fused all-reduce for embedding-gradient sized messages."""
    from edl_b200.ops import native
    from edl_b200.parallel.symm import SymmetricPool

    sizes_mb = [1, 4, 16, 40, 128, 256, 512]
    pool = SymmetricPool((sizes_mb[-1] + 8) << 20, device=dev)
    out = []
    for mb in sizes_mb:
        n = (mb << 20) // 4
        sl = pool.alloc(n, torch.float32)
        sl.tensor.normal_()
        for algo in (["twoshot", "multimem"] if pool.has_multicast else ["twoshot"]):
            for nblocks in (32, 64):
                torch.cuda.synchronize()
                dist.barrier()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                for it in range(13):
                    if it == 3:
                        e0.record()
                    native().allreduce_twoshot(sl.data_ptrs, sl.sig_ptrs, sl.mc_ptr, rank, sl.tensor, n, 1.0 / world,
                                               None, None, algo == "multimem", nblocks, 30.0)
                e1.record()
                torch.cuda.synchronize()
                ms = torch.tensor([e0.elapsed_time(e1) / 10], device=dev, dtype=torch.float64)
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
                busbw = (mb << 20) * 2 * (world - 1) / world / (ms.item() * 1e-3) / 1e9
                out.append({"MB": mb, "algo": algo, "blocks": nblocks, "ms": ms.item(), "busbw_GBps": busbw})
                if rank == 0:
                    print("allreduce fp32 %4d MB %-8s blocks %2d: %8.3f ms  busbw %7.1f GB/s" % (
                        mb, algo, nblocks, ms.item(), busbw), flush=True)
        pool._off -= 0   # slices are bump-allocated; the pool is sized for the largest one only
        pool._off = pool._sig_total
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=1000)
    ap.add_argument("--vocab", type=int, default=100001, help="1000001 in the reference")
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--model", default="ctr_dnn", choices=["ctr_dnn", "deepfm"])
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--sparse", action="store_true", help="row-sparse embedding gradients + lazy Adam on the tables")
    ap.add_argument("--out", default="")
    ap.add_argument("--save", default="", help="rank 0 writes the trained model's state dict here (input of dumper.py)")
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    cuda = torch.cuda.is_available()
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))) if cuda else torch.device("cpu")
    if cuda:
        torch.cuda.set_device(dev)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl" if cuda else "gloo")
    result = {}
    if args.sweep:
        assert cuda and world > 1, "--sweep needs >= 2 GPUs"
        result["sweep"] = sweep(dev, world, rank)
    else:
        torch.manual_seed(0)
        model = (DeepFM if args.model == "deepfm" else CtrDnn)(sparse_feature_dim=args.vocab,
                                                                sparse_grad=args.sparse).to(dev)
        dp = ElasticDataParallel(model, bucket_cap_mb=64)
        opt = ops.FlatAdam(dp.flat, lr=args.lr)
        sparse_opt = ops.SparseAdam(dp.sparse_params, lr=args.lr) if args.sparse else None
        gen = torch.Generator(device=dev).manual_seed(100 + rank)
        scores, labels = [], []
        t0 = time.time()
        for step in range(args.steps):
            dense, sparse, label = synthetic_batch(args.batch, args.vocab, dev, gen)
            dp.zero_grad()
            logits = dp(dense, sparse)
            loss = ops.soft_cross_entropy(logits, label, "labels")
            loss.backward()
            dp.finish()
            opt.step()
            if sparse_opt is not None:
                sparse_opt.step()
            scores.append(torch.softmax(logits.detach().float(), -1)[:, 1])
            labels.append(label)
            if step % 10 == 0 and rank == 0:
                a = auc(torch.cat(scores[-10:]), torch.cat(labels[-10:]))
                print("step %d loss %.4f auc %.4f" % (step, float(loss), float(a)), flush=True)
        if cuda:
            torch.cuda.synchronize()
        result["examples_per_s"] = args.batch * world * args.steps / (time.time() - t0)
        result["grad_bytes_per_step"] = sum(g.grad.numel() * g.grad.element_size() for g in dp.flat.groups.values())
        if args.sparse:
            result["grad_bytes_per_step"] += dp.last_sparse_bytes     # indices + values this rank sent last step
        if rank == 0:
            print(json.dumps(result))
            if args.save:
                os.makedirs(os.path.dirname(os.path.abspath(args.save)), exist_ok=True)
                torch.save({"model": {k: v.detach().cpu() for k, v in model.state_dict().items()}}, args.save)
    if args.out and rank == 0:
        json.dump(result, open(args.out, "w"), indent=1)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
