"""Fused soft-label / hard-label cross-entropy, KL-with-temperature and top-k accuracy
(csrc/loss.cu).  Reference ops: ``softmax_with_cross_entropy(soft_label=True)`` on teacher scores,
``accuracy(k=1,5)`` (example/distill/resnet/train_with_fleet.py:254-275) and the ``KL``/``KL_T``
distill losses (example/distill/nlp/model.py:54-66)."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

_MODE = {"probs": 0, "logits": 1, "labels": 2}


def _ref_loss(logits, target, mode, s_temp, t_temp, label_smooth, kl, loss_scale):
    z = logits.float() / s_temp
    logp = F.log_softmax(z, dim=-1)
    c = z.shape[-1]
    if mode == 2:
        p = F.one_hot(target, c).float() * (1 - label_smooth) + label_smooth / c
    elif mode == 0:
        p = target.float()
    else:
        p = F.softmax(target.float() / t_temp, dim=-1)
    loss = -(p * logp).sum(-1)
    if kl:
        loss = loss + (p * torch.log(p.clamp_min(1e-30))).sum(-1)
    return loss.mean() * loss_scale


def _smoothed_onehot_plogp(c, label_smooth):
    """``sum_j p_j log p_j`` of a one-hot over ``c`` classes smoothed by ``label_smooth``."""
    off = label_smooth / c
    on = 1.0 - label_smooth + off
    return (on * math.log(on) if on > 0 else 0.0) + (c - 1) * off * math.log(off)


class _SoftCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, mode, s_temp, t_temp, label_smooth, kl, loss_scale):
        from . import native, count_launch

        C = native()
        logits = logits.contiguous()
        n = logits.shape[0]
        # the kernel adds every row's share into `loss`.  KL against a smoothed one-hot: the target's sum p log p is
        # the same constant for every row, so it is the starting value
        start = 0.0
        if mode == 2 and kl and label_smooth > 0:
            start = _smoothed_onehot_plogp(logits.shape[1], label_smooth) * loss_scale
        loss = torch.full((), start, device=logits.device, dtype=torch.float32)
        stats = torch.empty(n, 4, device=logits.device, dtype=torch.float32)
        tgt = target.contiguous()
        if mode == 2:
            C.soft_ce_fwd(logits, None, tgt, loss, stats, mode, s_temp, t_temp, label_smooth, kl,
                          loss_scale)
        else:
            C.soft_ce_fwd(logits, tgt, None, loss, stats, mode, s_temp, t_temp, label_smooth, kl,
                          loss_scale)
        count_launch()
        ctx.save_for_backward(logits, tgt, stats)
        ctx.cfg = (mode, s_temp, t_temp, label_smooth, loss_scale)
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        from . import native, count_launch

        logits, tgt, stats = ctx.saved_tensors
        mode, s_temp, t_temp, label_smooth, loss_scale = ctx.cfg
        dlogits = torch.empty_like(logits)
        go = grad_out.float().contiguous()
        if mode == 2:
            native().soft_ce_bwd(logits, None, tgt, stats, go, dlogits, mode, s_temp, t_temp,
                                 label_smooth, loss_scale)
        else:
            native().soft_ce_bwd(logits, tgt, None, stats, go, dlogits, mode, s_temp, t_temp,
                                 label_smooth, loss_scale)
        count_launch()
        return dlogits, None, None, None, None, None, None, None


def soft_cross_entropy(logits, target, target_kind="probs", student_temperature=1.0,
                       teacher_temperature=1.0, label_smoothing=0.0, kl=False, loss_scale=1.0):
    """Mean over rows of ``-sum_j p_j log softmax(logits / Ts)_j`` (+ ``sum p log p`` if ``kl``).

    target_kind: ``"probs"`` (teacher scores, the reference's ``soft_label=True`` path),
    ``"logits"`` (raw teacher logits, softmax with ``teacher_temperature`` applied inside the
    kernel -- what the NVSwitch logit-ship path delivers) or ``"labels"`` (int64 hard labels)."""
    mode = _MODE[target_kind]
    if logits.is_cuda:
        return _SoftCEFn.apply(logits, target, mode, float(student_temperature),
                               float(teacher_temperature), float(label_smoothing), bool(kl),
                               float(loss_scale))
    return _ref_loss(logits, target, mode, student_temperature, teacher_temperature,
                     label_smoothing, kl, loss_scale)


def topk_accuracy(logits, labels):
    """Returns a float32 tensor [2] = (top-1 hits, top-5 hits) summed over the batch."""
    from . import native, count_launch

    if logits.is_cuda:
        counts = torch.zeros(2, device=logits.device, dtype=torch.float32)
        native().topk_acc(logits.contiguous(), labels.contiguous(), counts)
        count_launch()
        return counts
    top5 = logits.float().topk(min(5, logits.shape[-1]), dim=-1).indices
    hit1 = (top5[:, 0] == labels).float().sum()
    hit5 = (top5 == labels[:, None]).any(-1).float().sum()
    return torch.stack([hit1, hit5])
