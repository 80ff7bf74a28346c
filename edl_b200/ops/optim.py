"""Flat-buffer fused optimizers (csrc/optim.cu) + LR schedules.

``FlatSGDMomentum`` is the H100 counterpart of the reference's ``Momentum(lr, 0.9, L2Decay(1e-4))``
(example/distill/resnet/train_with_fleet.py:106-122) and its AMP master-weight helpers
(example/distill/resnet/utils/fp16_utils.py:86-129): one kernel per dtype group updates fp32 master
weights + momentum and writes the bf16 model copy.  The learning rate lives in a device scalar so a
captured CUDA graph can be replayed while the host-side schedule (reference:
utils/learning_rate.py:39-95 cosine/piecewise with warm-up) only updates that scalar.
"""
from __future__ import annotations

import math
from typing import Optional

import torch


class _FlatOptimizerBase:
    def __init__(self, flat, lr: float):
        self.flat = flat
        dev = flat.device
        self.lr = float(lr)
        self.lr_t = torch.full((1,), float(lr), dtype=torch.float32, device=dev)
        self.grad_scale_t: Optional[torch.Tensor] = None  # device scalar multiplied into grads
        self.found_inf_t: Optional[torch.Tensor] = None   # device int flag: skip step when != 0
        self._found_inf_is_comm_error = False
        self.skip_dtype = None    # set by ElasticDataParallel.attach_optimizer: dtype -> "already updated this step"

    def set_lr(self, lr: float):
        self.lr = float(lr)
        self.lr_t.fill_(self.lr)

    def set_grad_scale(self, t: Optional[torch.Tensor]):
        self.grad_scale_t = t

    def set_found_inf(self, t: Optional[torch.Tensor], comm_error: bool = False):
        """``comm_error``: the flag is the fabric's error word (in-place elastic guard), not a gradient overflow
        flag -- the per-bucket fused optimizer may then still be used (its kernel checks the word itself)."""
        self.found_inf_t = t
        self._found_inf_is_comm_error = bool(comm_error) and t is not None

    def found_inf_is_comm_error(self) -> bool:
        return self.found_inf_t is None or self._found_inf_is_comm_error

    def zero_grad(self):
        self.flat.zero_grad()


class FlatSGDMomentum(_FlatOptimizerBase):
    def __init__(self, flat, lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=False,
                 decay_filter=None):
        super().__init__(flat, lr)
        self.momentum, self.weight_decay, self.nesterov = momentum, weight_decay, nesterov
        self.state = {}
        for dt, g in flat.groups.items():
            st = {"mom": torch.zeros(g.numel, dtype=torch.float32, device=flat.device), "wd_mask": None}
            if decay_filter is not None:
                mask = torch.zeros(g.numel, dtype=torch.float32, device=flat.device)
                for e in g.entries:
                    if decay_filter(e.name, e.param):
                        mask[e.offset:e.offset + e.numel] = 1.0
                st["wd_mask"] = mask
            self.state[dt] = st

    @torch.no_grad()
    def step(self):
        from . import native, count_launch

        for dt, g in self.flat.groups.items():
            if self.skip_dtype is not None and self.skip_dtype(dt):
                continue                 # updated bucket by bucket by the data-parallel engine (parallel/ddp.py)
            st = self.state[dt]
            master = g.master if g.master is not None else g.param
            lp = g.param if g.master is not None else None
            if g.param.is_cuda:
                native().sgd_momentum(lp, master, st["mom"], g.grad, st["wd_mask"], self.lr_t,
                                      self.grad_scale_t, self.found_inf_t, self.momentum,
                                      self.weight_decay, self.nesterov)
                count_launch()
            else:
                if self.found_inf_t is not None and int(self.found_inf_t.item()) != 0:
                    continue
                grad = g.grad.float()
                if self.grad_scale_t is not None:
                    grad = grad * self.grad_scale_t
                wd = self.weight_decay if st["wd_mask"] is None else self.weight_decay * st["wd_mask"]
                grad = grad + wd * master
                st["mom"].mul_(self.momentum).add_(grad)
                upd = grad + self.momentum * st["mom"] if self.nesterov else st["mom"]
                master.add_(upd * (-self.lr_t))
                if lp is not None:
                    lp.copy_(master.to(lp.dtype))

    def state_dict(self):
        return {
            "lr": self.lr,
            "momentum": {str(dt): st["mom"] for dt, st in self.state.items()},
            "master": {str(dt): (g.master if g.master is not None else g.param)
                       for dt, g in self.flat.groups.items()},
        }

    def load_state_dict(self, sd):
        self.set_lr(sd["lr"])
        for dt, st in self.state.items():
            st["mom"].copy_(sd["momentum"][str(dt)])
        for dt, g in self.flat.groups.items():
            src = sd["master"][str(dt)]
            if g.master is not None:
                g.master.copy_(src)
                g.param.copy_(src.to(g.param.dtype))
            else:
                g.param.copy_(src)


class FlatAdam(_FlatOptimizerBase):
    """Adam / AdamW on flat buffers (CTR-DNN uses Adam 1e-4, example/ctr/ctr/train.py:234; the NLP
    distill students use AdamW, example/distill/nlp/model.py:35-51)."""

    def __init__(self, flat, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0,
                 decoupled=False):
        super().__init__(flat, lr)
        self.betas, self.eps, self.weight_decay, self.decoupled = betas, eps, weight_decay, decoupled
        self.step_t = torch.zeros(1, dtype=torch.float32, device=flat.device)
        self.state = {dt: {"m": torch.zeros(g.numel, dtype=torch.float32, device=flat.device),
                           "v": torch.zeros(g.numel, dtype=torch.float32, device=flat.device)}
                      for dt, g in flat.groups.items()}

    @torch.no_grad()
    def step(self):
        from . import native, count_launch

        # bias correction counts APPLIED steps only: a step skipped by found_inf (loss-scaling overflow, broken
        # collective) must not advance it -- decided on the device, no host round trip
        if self.found_inf_t is not None:
            if not self.step_t.is_cuda and int(self.found_inf_t.item()) != 0:
                return
            self.step_t += (self.found_inf_t.view(-1)[:1] == 0).to(self.step_t.dtype)
        else:
            self.step_t += 1
        for dt, g in self.flat.groups.items():
            st = self.state[dt]
            master = g.master if g.master is not None else g.param
            lp = g.param if g.master is not None else None
            if g.param.is_cuda:
                native().adam_step(lp, master, st["m"], st["v"], g.grad, self.lr_t,
                                   self.grad_scale_t, self.found_inf_t, self.step_t, self.betas[0],
                                   self.betas[1], self.eps, self.weight_decay, self.decoupled)
                count_launch()
            else:
                grad = g.grad.float()
                if self.grad_scale_t is not None:
                    grad = grad * self.grad_scale_t
                if not self.decoupled:
                    grad = grad + self.weight_decay * master
                b1, b2 = self.betas
                st["m"].mul_(b1).add_(grad, alpha=1 - b1)
                st["v"].mul_(b2).addcmul_(grad, grad, value=1 - b2)
                t = float(self.step_t.item())
                mhat = st["m"] / (1 - b1 ** t)
                vhat = st["v"] / (1 - b2 ** t)
                if self.decoupled:
                    master.mul_(1 - self.lr * self.weight_decay)
                master.add_(-self.lr * mhat / (vhat.sqrt() + self.eps))
                if lp is not None:
                    lp.copy_(master.to(lp.dtype))

    def state_dict(self):
        return {"lr": self.lr, "step": self.step_t,
                "m": {str(dt): st["m"] for dt, st in self.state.items()},
                "v": {str(dt): st["v"] for dt, st in self.state.items()},
                "master": {str(dt): (g.master if g.master is not None else g.param)
                           for dt, g in self.flat.groups.items()}}

    def load_state_dict(self, sd):
        self.set_lr(sd["lr"])
        self.step_t.copy_(sd["step"])
        for dt, st in self.state.items():
            st["m"].copy_(sd["m"][str(dt)])
            st["v"].copy_(sd["v"][str(dt)])
        for dt, g in self.flat.groups.items():
            src = sd["master"][str(dt)]
            if g.master is not None:
                g.master.copy_(src)
                g.param.copy_(src.to(g.param.dtype))
            else:
                g.param.copy_(src)


class SparseAdam:
    """Lazy Adam for fp32 tables with row-sparse gradients (``ops.embedding_bag_mean_sparse``; Paddle's ``adam`` with
    ``lazy_mode=True``).  Only the rows present in a gradient are updated, with FlatAdam's formula
    ``w -= lr * mhat / (sqrt(vhat) + eps)``; other rows and their ``m`` / ``v`` are not touched.  The bias correction
    counts ``step()`` calls on a device scalar, so steps never synchronise with the host.  On a GPU the gradients of
    all tables of one width are keyed by (table, row) and stably sorted, and one kernel (csrc/embedding.cu) sums every
    run of equal keys in a fixed order and updates that row: the result is deterministic, and every rank that applies
    the same gathered gradient gets the same tables."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
        self.params = list(params)
        for p in self.params:
            if p.dtype != torch.float32 or p.dim() != 2:
                raise TypeError("SparseAdam: fp32 [V, D] tables only, got %s %s" % (p.dtype, tuple(p.shape)))
        dev = self.params[0].device if self.params else torch.device("cpu")
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        self.lr = float(lr)
        self.lr_t = torch.full((1,), self.lr, dtype=torch.float32, device=dev)
        self.step_t = torch.zeros(1, dtype=torch.float32, device=dev)
        self.state = [{"m": torch.zeros_like(p, dtype=torch.float32), "v": torch.zeros_like(p, dtype=torch.float32)}
                      for p in self.params]

    def set_lr(self, lr: float):
        self.lr = float(lr)
        self.lr_t.fill_(self.lr)

    def zero_grad(self):
        for p in self.params:
            p.grad = None

    @torch.no_grad()
    def step(self):
        self.step_t += 1
        todo = []
        for i, p in enumerate(self.params):
            if p.grad is None:
                continue
            if not p.grad.is_sparse:
                raise TypeError("SparseAdam: the gradient of a %s table is dense; build the model with "
                                "sparse_grad=True" % (tuple(p.shape),))
            todo.append(i)
        if todo and self.params[0].is_cuda:
            self._step_cuda(todo)
        else:
            for i in todo:
                self._step_cpu(self.params[i], self.state[i])

    def _step_cuda(self, todo):
        """One key / sort / update sequence per group of up to 64 tables of one width (csrc/embedding.cu)."""
        from . import native, count_launch

        groups = {}
        for i in todo:
            groups.setdefault(self.params[i].shape[1], []).append(i)
        for ids in groups.values():
            for k in range(0, len(ids), 64):
                chunk = ids[k:k + 64]
                grads = [self.params[i].grad for i in chunk]
                native().sparse_adam([g._indices()[0] for g in grads], [g._values() for g in grads],
                                     [self.params[i].data for i in chunk], [self.state[i]["m"] for i in chunk],
                                     [self.state[i]["v"] for i in chunk], self.lr_t, self.step_t, self.betas[0],
                                     self.betas[1], self.eps)
                count_launch(2)

    def _step_cpu(self, p, st):
        b1, b2 = self.betas
        gc = p.grad.double().coalesce()           # repeated rows summed in fp64, like the kernel
        rows, grad = gc.indices()[0], gc.values().float()
        m = st["m"][rows].mul_(b1).add_(grad, alpha=1 - b1)
        v = st["v"][rows].mul_(b2).addcmul_(grad, grad, value=1 - b2)
        t = float(self.step_t.item())
        mhat = m / (1 - b1 ** t)
        vhat = v / (1 - b2 ** t)
        p.data[rows] = p.data[rows] - self.lr * mhat / (vhat.sqrt() + self.eps)
        st["m"][rows] = m
        st["v"][rows] = v

    def state_dict(self):
        return {"lr": self.lr, "step": self.step_t,
                "m": [st["m"] for st in self.state], "v": [st["v"] for st in self.state]}

    def load_state_dict(self, sd):
        self.set_lr(sd["lr"])
        self.step_t.copy_(sd["step"])
        for st, m, v in zip(self.state, sd["m"], sd["v"]):
            st["m"].copy_(m)
            st["v"].copy_(v)


# ---------------------------------------------------------------------------------------------
# LR schedules (host side; the result is written into the optimizer's device scalar)

def cosine_decay_with_warmup(step: int, base_lr: float, steps_per_epoch: int, epochs: int,
                             warmup_epochs: int = 5) -> float:
    """Linear warm-up then per-epoch cosine decay (reference utils/learning_rate.py:39-60)."""
    warm = warmup_epochs * steps_per_epoch
    if step < warm:
        return base_lr * step / max(warm, 1)
    epoch = step // max(steps_per_epoch, 1)
    return base_lr * 0.5 * (math.cos((epoch - warmup_epochs) * math.pi / max(epochs - warmup_epochs, 1)) + 1)


def piecewise_decay_with_warmup(step: int, base_lr: float, steps_per_epoch: int, boundaries_epochs,
                                gamma: float = 0.1, warmup_epochs: int = 5) -> float:
    """Step decay at epoch boundaries with linear warm-up (reference utils/learning_rate.py:62-95)."""
    warm = warmup_epochs * steps_per_epoch
    if step < warm:
        return base_lr * step / max(warm, 1)
    epoch = step // max(steps_per_epoch, 1)
    k = sum(1 for b in boundaries_epochs if epoch >= b)
    return base_lr * (gamma ** k)


def scaled_lr(lr: float, batch_per_trainer: int, num_trainers: int, ref_batch: int = 256) -> float:
    """``base_lr = lr * (batch * num_trainers) / 256`` -- the reference's world-size LR rescale
    (example/collective/resnet50/train_with_fleet.py:129-141)."""
    return lr * (batch_per_trainer * num_trainers) / ref_batch
