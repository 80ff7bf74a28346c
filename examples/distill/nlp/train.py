#!/usr/bin/env python
"""Train the small student (BOW / TextCNN / BiLSTM / Transformer) alone on hard labels -- the baseline the distilled student is
compared with (reference: example/distill/nlp/train.py)."""
import argparse
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.abspath(os.path.join(HERE, "..", "..", "..")))
from reader import TsvReader, batches, synthetic_corpus  # noqa: E402
from paddle_edl.models.small import BOW, BiLSTM, TextCNN  # noqa: E402
from paddle_edl.models.ernie import ernie_student, pack_sequences  # noqa: E402


def build_model(name, vocab, dropout=0.0):
    """(model, device): the LSTM and Transformer students run on the GPU when there is one (csrc/lstm.cu, the encoder
    kernels), the others on the CPU.  The Transformer student has the teacher's 18000-id vocabulary and builds its four
    feeds from the ids (positions 0.., segment 0, mask ids != 0); ``dropout`` is its hidden and attention dropout."""
    if name in ("lstm", "ernie"):
        dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
        return (BiLSTM(vocab) if name == "lstm" else ernie_student(dropout=dropout)).to(dev), dev
    return (BOW(vocab) if name == "bow" else TextCNN(vocab)), torch.device("cpu")


def student_logits(model, ids, dev, packed=False):
    """The student's logits for a padded id batch.  ``packed`` (Transformer student only): pack the batch to its real
    tokens (``pack_sequences`` of the feeds built from the ids: positions 0.., segment 0, mask ids != 0) and run
    ``forward_packed``, so no GEMM, LayerNorm or attention tile works on padding."""
    t = torch.from_numpy(ids)
    if not packed:
        return model(t.to(dev))
    b, l = t.shape
    ids_p, pos, seg, cu, max_len, key_mask = pack_sequences(t, torch.arange(l).expand(b, l), torch.zeros_like(t), t != 0)
    return model.forward_packed(ids_p.to(dev), pos.to(dev), seg.to(dev), cu.to(dev), max_len,
                                None if key_mask is None else key_mask.to(dev))


def evaluate(model, data, dev=torch.device("cpu")):
    model.eval()
    hit = n = 0
    with torch.no_grad():
        for ids, label in data:
            pred = model(torch.from_numpy(ids).to(dev)).argmax(-1).cpu()
            hit += int((pred == torch.from_numpy(label[:, 0])).sum())
            n += len(label)
    model.train()
    return hit / max(1, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="bow", choices=["bow", "cnn", "lstm", "ernie"])
    ap.add_argument("--train_tsv", default=None)
    ap.add_argument("--dev_tsv", default=None)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--vocab", type=int, default=2000)
    ap.add_argument("--seq_len", type=int, default=64)
    ap.add_argument("--samples", type=int, default=1024)
    ap.add_argument("--dropout", type=float, default=0.0, help="hidden and attention dropout of --model ernie")
    ap.add_argument("--packed", action="store_true",
                    help="--model ernie: train on each batch packed to its real tokens (forward_packed)")
    args = ap.parse_args()
    if args.packed and args.model != "ernie":
        ap.error("--packed needs --model ernie")
    if args.train_tsv:
        tr = TsvReader(args.train_tsv, seq_len=args.seq_len)
        dev = TsvReader(args.dev_tsv or args.train_tsv, vocab=tr.vocab, seq_len=args.seq_len)
        vocab = len(tr.vocab)
        train_iter = lambda ep: batches(tr.samples(), 16)       # noqa: E731
        dev_data = list(batches(dev.samples(), 16))
    else:
        vocab = args.vocab
        train_iter = lambda ep: batches(synthetic_corpus(args.samples, vocab, args.seq_len, ep), 16)   # noqa: E731
        dev_data = list(batches(synthetic_corpus(256, vocab, args.seq_len, 10_000), 16))
    model, dev = build_model(args.model, vocab, args.dropout)
    opt = torch.optim.AdamW(model.parameters(), 1e-4 if args.model == "ernie" else 1e-3)   # a Transformer wants less
    for ep in range(args.epochs):
        for ids, label in train_iter(ep):
            loss = torch.nn.functional.cross_entropy(student_logits(model, ids, dev, args.packed),
                                                     torch.from_numpy(label[:, 0]).to(dev))
            opt.zero_grad()
            loss.backward()
            opt.step()
        print("epoch %d loss %.4f dev acc %.4f" % (ep, float(loss), evaluate(model, dev_data, dev)), flush=True)


if __name__ == "__main__":
    main()
