#!/usr/bin/env python
"""Same-box distillation training: half of the GPUs train the ResNet50_vd student, the other half serve the
ResNeXt101_32x16d teacher through the NVSwitch-direct link (no RPC, no host copies of logits) -- the training-loop
version of ``bench.py --mode distill``.

    torchrun --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 examples/distill/resnet/train_device_link.py \
        --epochs 120 --steps_per_epoch 5004 --teacher_fp8 0

Ranks [0, N/2) are students (data-parallel among themselves), rank s is paired with teacher rank N/2 + s.  Student and
teacher are software-pipelined by one batch.  Teacher weights: ``--teacher_ckpt`` (a state dict of
``paddle_edl.models.resnext.ResNeXt101_32x16d``); random init if absent (no network access here).
"""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", ".."))
sys.path.insert(0, ROOT)

from edl_b200.checkpoint import LocalFS, TrainStatus, load_check_point, save_check_point  # noqa: E402
from edl_b200.distill.device_feed import DeviceDistillLink, pool_bytes_needed  # noqa: E402
from edl_b200.distill.device_trainer import DistillStudentTrainer, TeacherWorker, split_roles  # noqa: E402
from edl_b200.models import ResNetVd, to_train_dtype  # noqa: E402
from edl_b200.models.resnext import ResNeXt101_32x16d, to_inference_dtype  # noqa: E402
from edl_b200.ops.optim import cosine_decay_with_warmup, scaled_lr  # noqa: E402
from edl_b200.parallel.symm import SymmetricPool  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch_size", type=int, default=32, help="per student GPU")
    ap.add_argument("--epochs", type=int, default=120)
    ap.add_argument("--steps_per_epoch", type=int, default=100)
    ap.add_argument("--lr", type=float, default=0.1)
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--teacher_ckpt", default=None)
    ap.add_argument("--teacher_fp8", type=int, default=0)
    ap.add_argument("--teacher_fp8_scaling", choices=("tensor", "block"), default="tensor",
                    help="'tensor': one activation scale per layer from a random calibration batch; 'block': per-row, "
                         "per-128-channel scales computed as each layer runs (no calibration)")
    ap.add_argument("--checkpoint", default="./distill_link_ckpt")
    ap.add_argument("--fetch_steps", type=int, default=10)
    args = ap.parse_args()

    world, rank = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev)
    n_students, students, teachers = split_roles(world)
    sgroup = dist.new_group(ranks=students)
    dist.new_group(ranks=teachers)
    B = args.batch_size
    pool = SymmetricPool(pool_bytes_needed(B, slots=2) + (8 << 20), device=dev)
    is_student = rank < n_students
    peer = rank + n_students if is_student else rank - n_students
    link = DeviceDistillLink(pool, peer, "student" if is_student else "teacher", B, slots=2, temperature=args.temperature,
                             timeout_s=300.0)
    total_steps = args.epochs * args.steps_per_epoch

    if not is_student:
        tm = ResNeXt101_32x16d()
        if args.teacher_ckpt:
            tm.load_state_dict(torch.load(args.teacher_ckpt, map_location="cpu"))
        tm = to_inference_dtype(tm, torch.bfloat16, dev).eval()
        if args.teacher_fp8 and args.teacher_fp8_scaling == "block":
            tm.enable_fp8(scaling="block")
        elif args.teacher_fp8:
            calib = torch.randn(B, 3, 224, 224, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
            tm.enable_fp8(calib)
        worker = TeacherWorker(tm, link)
        for _ in range(total_steps + 1):          # +1: the student's priming step ships a batch without training
            worker.step()
        torch.cuda.synchronize(dev)
        dist.barrier()
        dist.destroy_process_group()
        return

    torch.manual_seed(0)
    model = to_train_dtype(ResNetVd(50), torch.bfloat16, dev).train()
    base_lr = scaled_lr(args.lr, B, n_students)
    tr = DistillStudentTrainer(model, B, link, lr=base_lr, group=sgroup)
    fs = LocalFS()
    tensors, ts, _ = load_check_point(args.checkpoint, fs, trainer_id=rank, map_location=dev)
    if tensors is not None:
        tr.load_state_dict(tensors)
    g = torch.Generator().manual_seed(1234 + rank)
    host = [torch.randn(B, 3, 224, 224, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).pin_memory()
            for _ in range(4)]                      # synthetic images; plug paddle_edl.utils.image_pipeline here
    step = 0
    tr.step(host[0])                                # priming step: batch 0 goes to the teacher, nothing to train on yet
    for epoch in range(args.epochs):
        t0 = time.time()
        for it in range(args.steps_per_epoch):
            tr.set_lr(cosine_decay_with_warmup(step, base_lr, args.steps_per_epoch, args.epochs))
            loss = tr.step(host[(step + 1) % 4])
            step += 1
            if it % args.fetch_steps == 0 and rank == 0:
                print("Pass %d, batch %d, loss %.5f, speed %.1f img/s" % (
                    epoch, it, float(loss), (it + 1) * B * n_students / max(1e-6, time.time() - t0)), flush=True)
        tr.consolidate()                 # student ranks: sharded optimizer state -> complete (collective of the students)
        if rank == 0 and epoch >= ts.next():
            save_check_point(args.checkpoint, tr.state_dict(), TrainStatus(epoch, step), fs, trainer_id=0)
    assert link.check_error() == 0, "the NVSwitch link reported a timeout"
    torch.cuda.synchronize(dev)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
