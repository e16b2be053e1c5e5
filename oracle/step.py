"""ORACLE (test infrastructure only): one reference training iteration on CPU, W ranks over gloo.

Restates the inner loop of the reference (train.py:284-310) with plain torch CPU ops:

    preds = model(x)                                   train.py:293
    loss, strs = get_total_loss(preds, m, [BCE, CEL])  train.py:295  (utils/pipeline_ops.py:37-42)
    optimizer.zero_grad(); loss.backward()             train.py:297-302
    [apex DDP: flat SUM all-reduce, ×1/W]              train.py:185   (parity unpinned: apex)
    optimizer.step()                                   train.py:303   (torch.optim.SGD, f3_trick groups)
    reduced = allreduce_tensor(loss)                   train.py:306   (utils/tensor_ops.py:60-64)

and the apex wrappers by their published semantics: SyncBN = batch statistics over all ranks
(`OracleSyncBN`, arithmetic of torch/nn/modules/_functions.py:7-209 with CPU ops + gloo all_reduce —
the stock torch module refuses CPU tensors, torch/nn/modules/batchnorm.py:798-811).

`model_factory` is injected: tools/make_golden.py passes the UNMODIFIED reference `network.res50`
(imported from a checkout of the reference); tests and bench.py pass this repo's plugin of the
same architecture (bit-identical init and outputs: tests/test_host_cpu.py::test_model_plugin_is_bit_identical_to_reference).
"""
from __future__ import annotations

import time

import torch
import torch.distributed as dist
import torch.nn as nn


# ----------------------------------------------------------------------------------------------
# losses, written the way the reference writes them (so autograd produces the reference gradient)
# ----------------------------------------------------------------------------------------------
class OracleCEL(nn.Module):
    eps = 1e-6

    def forward(self, pred, target):  # loss/CEL.py:15-20
        p = pred.sigmoid()
        inter = p * target
        return ((p - inter).sum() + (target - inter).sum()) / (p.sum() + target.sum() + self.eps)


def total_loss(preds, masks, loss_funcs):  # utils/pipeline_ops.py:37-42
    outs = [f(preds, masks) for f in loss_funcs]
    return sum(outs), [f"{o.item():.5f}" for o in outs]


# ----------------------------------------------------------------------------------------------
# SyncBN on CPU/gloo
# ----------------------------------------------------------------------------------------------
class _SyncBNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, eps, momentum, group):
        C = x.shape[1]
        xf = x.float()
        stats = torch.cat([xf.sum(dim=(0, 2, 3)), (xf * xf).sum(dim=(0, 2, 3)),
                           torch.tensor([float(x.numel() // C)])])
        if group is not None:
            dist.all_reduce(stats, group=group)
        n = stats[-1]
        mean = stats[:C] / n
        var = (stats[C:2 * C] / n - mean * mean).clamp_min(0)
        invstd = torch.rsqrt(var + eps)
        if running_mean is not None:
            running_mean.mul_(1 - momentum).add_(mean, alpha=momentum)
            running_var.mul_(1 - momentum).add_(var * (n / (n - 1)), alpha=momentum)
        y = (xf - mean[None, :, None, None]) * (invstd * weight)[None, :, None, None] + bias[None, :, None, None]
        ctx.save_for_backward(xf, weight, mean, invstd, n)
        ctx.group = group
        return y.to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        xf, weight, mean, invstd, n = ctx.saved_tensors
        C = xf.shape[1]
        dyf = dy.float()
        xmu = xf - mean[None, :, None, None]
        sum_dy = dyf.sum(dim=(0, 2, 3))
        sum_dy_xmu = (dyf * xmu).sum(dim=(0, 2, 3))
        dgamma, dbeta = sum_dy_xmu * invstd, sum_dy.clone()
        red = torch.cat([sum_dy, sum_dy_xmu])
        if ctx.group is not None:
            dist.all_reduce(red, group=ctx.group)
        mean_dy, mean_dy_xmu = red[:C] / n, red[C:] / n
        dx = (dyf - mean_dy[None, :, None, None] - xmu * (invstd * invstd * mean_dy_xmu)[None, :, None, None]) \
            * (invstd * weight)[None, :, None, None]
        return dx.to(dy.dtype), dgamma, dbeta, None, None, None, None, None


class OracleSyncBN(nn.BatchNorm2d):
    group = None

    def forward(self, x):
        if not self.training:
            return super().forward(x)
        if self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        return _SyncBNFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var,
                               self.eps, self.momentum, self.group)


def convert_syncbn_oracle(module: nn.Module, group) -> nn.Module:
    """Swap every BatchNorm2d for OracleSyncBN, SHARING the affine Parameters (SURVEY Q2 decision:
    γ/β stay in the optimizer that was built before the conversion, train.py:157 vs :180)."""
    for name, child in list(module.named_children()):
        if isinstance(child, nn.BatchNorm2d) and not isinstance(child, OracleSyncBN):
            new = OracleSyncBN(child.num_features, child.eps, child.momentum)
            new.weight, new.bias = child.weight, child.bias
            new.running_mean, new.running_var = child.running_mean, child.running_var
            new.num_batches_tracked = child.num_batches_tracked
            new.group = group
            new.train(child.training)
            if isinstance(module, nn.Sequential):
                module[int(name)] = new
            else:
                setattr(module, name, new)
        else:
            convert_syncbn_oracle(child, group)
    return module


# ----------------------------------------------------------------------------------------------
# optimizer / DDP restatement
# ----------------------------------------------------------------------------------------------
def f3_trick_groups(model: nn.Module, lr: float):
    """utils/pipeline_ops.py:295-307."""
    backbone, head = [], []
    for name, p in model.named_parameters():
        if name.startswith("div_2"):
            continue
        (backbone if name.startswith("div") else head).append(p)
    return [{"params": backbone, "lr": 0.1 * lr}, {"params": head, "lr": lr}]


def flat_allreduce_mean(params, world: int, group=None):
    """apex DDP(delay_allreduce=True): flatten all grads → one SUM all-reduce → ×1/W → copy back."""
    grads = [p.grad for p in params if p.grad is not None]
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, group=group)
    flat.mul_(1.0 / world)
    off = 0
    for g in grads:
        g.copy_(flat[off:off + g.numel()].view_as(g))
        off += g.numel()


class OracleTrainer:
    """Holds model/optimizer for repeated `step(x, m)` calls (fp32, CPU)."""

    def __init__(self, model_factory, lr=0.05, momentum=0.9, weight_decay=5e-4, reduction="mean",
                 use_aux_loss=True, world_size=1, seed=0):
        import random
        import numpy as np
        random.seed(seed); np.random.seed(seed); torch.manual_seed(seed)   # utils/misc.py:38-43
        self.world = world_size
        self.model = model_factory()
        self.optimizer = torch.optim.SGD(f3_trick_groups(self.model, lr), momentum=momentum,
                                         weight_decay=weight_decay, nesterov=False)
        self.base_lrs = [g["lr"] for g in self.optimizer.param_groups]
        if world_size > 1:
            convert_syncbn_oracle(self.model, dist.group.WORLD)
            for p in self.model.parameters():           # DDP ctor: broadcast from rank 0
                dist.broadcast(p.data, 0)
            for b in self.model.buffers():
                dist.broadcast(b.data, 0)
        self.loss_funcs = [nn.BCEWithLogitsLoss(reduction=reduction)]
        if use_aux_loss:
            self.loss_funcs.append(OracleCEL())
        self.model.train()

    def set_lr_coefficient(self, coef: float):
        for g, base in zip(self.optimizer.param_groups, self.base_lrs):
            g["lr"] = base * coef

    def step(self, x, m):
        preds = self.model(x)
        loss, strs = total_loss(preds, m, self.loss_funcs)
        self.optimizer.zero_grad()
        loss.backward()
        if self.world > 1:
            flat_allreduce_mean(list(self.model.parameters()), self.world)
        self.optimizer.step()
        red = loss.detach().clone()
        if self.world > 1:
            dist.all_reduce(red)
            red /= self.world
        return dict(loss=float(red.item()), items=strs, preds=preds.detach())


def time_steps(trainer: OracleTrainer, x, m, steps: int, warmup: int = 1) -> float:
    """seconds per step (wall clock, CPU)."""
    for _ in range(warmup):
        trainer.step(x, m)
    t0 = time.perf_counter()
    for _ in range(steps):
        trainer.step(x, m)
    return (time.perf_counter() - t0) / steps
