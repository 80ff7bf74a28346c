#!/usr/bin/env python
"""Sentence-classification distillation: BOW / TextCNN / BiLSTM / Transformer student, served sequence teacher, ``KL_T`` loss
with T=2 and a batch generator carrying token ids (reference: example/distill/nlp/distill.py:98-196,
model.py:54-135; the reference's teacher is an ERNIE served by Paddle Serving -- any served model
that returns ``logits`` works here; a TextCNN stands in when none is given)."""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))))
from paddle_edl.distill.distill_reader import DistillReader  # noqa: E402
from paddle_edl.distill.teacher_server import TeacherServer  # noqa: E402
from paddle_edl.models.small import BOW, BiLSTM, TextCNN, kl_distill_loss  # noqa: E402
from paddle_edl.models.ernie import ernie_student  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train import student_logits  # noqa: E402


def corpus(n, vocab, seq, seed):
    rng = np.random.RandomState(seed)
    for _ in range(n):
        y = rng.randint(0, 2)
        ids = rng.randint(2, vocab // 2, size=seq) + (vocab // 2 - 2) * y   # class-dependent vocabulary half
        ids[rng.randint(seq // 2, seq):] = 0                                 # padding
        yield ids.astype("int64"), np.array([y], dtype="int64")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="bow", choices=["bow", "cnn", "lstm", "ernie"])
    ap.add_argument("--teachers", default="")
    ap.add_argument("--T", type=float, default=2.0)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--vocab", type=int, default=2000)
    ap.add_argument("--dropout", type=float, default=0.0, help="hidden and attention dropout of --model ernie")
    ap.add_argument("--packed", action="store_true",
                    help="--model ernie: the student trains on each batch packed to its real tokens (the teacher still "
                         "receives the padded feeds)")
    ap.add_argument("--heads", type=int, default=6,
                    help="--model ernie: attention heads of the hidden-384 student (12: the MiniLM-shaped head dim 32)")
    args = ap.parse_args()
    if args.packed and args.model != "ernie":
        ap.error("--packed needs --model ernie")
    srv = None
    if not args.teachers:
        teacher = TextCNN(args.vocab).eval()
        srv = TeacherServer(teacher, ["ids"], ["logits"], {"ids": [64]}).start()
        args.teachers = srv.endpoint
    dev = torch.device("cpu")
    if args.model in ("lstm", "ernie"):  # these students run on the GPU when there is one
        dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
        # the Transformer student builds its four feeds from the ids (positions 0.., segment 0, mask ids != 0)
        student = (BiLSTM(args.vocab) if args.model == "lstm" else ernie_student(dropout=args.dropout,
                                                                                      heads=args.heads)).to(dev)
    else:
        student = BOW(args.vocab) if args.model == "bow" else TextCNN(args.vocab)
    opt = torch.optim.AdamW(student.parameters(), 1e-4 if args.model == "ernie" else 1e-3)   # a Transformer wants less

    def batch_gen():
        buf = []
        for s in corpus(512, args.vocab, 64, 1):
            buf.append(s)
            if len(buf) == 16:
                yield np.stack([b[0] for b in buf]), np.stack([b[1] for b in buf])
                buf = []

    dr = DistillReader(ins=["ids", "label"], predicts=["logits"])
    dr.set_teacher_batch_size(16)
    dr.set_fixed_teacher(args.teachers)
    reader = dr.set_batch_generator(batch_gen)
    for epoch in range(args.epochs):
        for i, (ids, label, t_logits) in enumerate(reader()):
            logits = student_logits(student, ids, dev, args.packed)
            loss = kl_distill_loss(logits, torch.from_numpy(t_logits).to(dev), args.T) + \
                torch.nn.functional.cross_entropy(logits, torch.from_numpy(label[:, 0]).to(dev))
            opt.zero_grad()
            loss.backward()
            opt.step()
            if i % 8 == 0:
                print("epoch %d step %d loss %.4f" % (epoch, i, float(loss)), flush=True)
    dr.stop()
    if srv:
        srv.stop()


if __name__ == "__main__":
    main()
