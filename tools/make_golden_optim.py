#!/usr/bin/env python
"""Generate tests/golden/optim_ext_kat.npz by running the UNMODIFIED reference's `make_optimizer` and `CustomScheduler`
on CPU, for the two optimizer settings `tools/make_golden.py` does not record: optim "adam", and Nesterov momentum
(`nesterov: True`) for sgd_trick and f3_trick.  Same recipe as `make_golden.py:sgd_kats` (the `_Tiny` module, seed 3,
poly schedule over 4 steps, gradients from a generator seeded 11):

    SOD_REFERENCE=/path/to/Distributed-SOD-Project python tools/make_golden_optim.py

Recorded per case: parameter names, the group of every parameter (-1: none), the groups' lr / weight_decay (and
betas / eps for Adam), the flat parameters before the first step and after every step, the gradients and the groups'
lr of every step.  For Adam also the state_dict after step 4: per parameter (in `named_parameters()` order) `step`,
`exp_avg`, `exp_avg_sq` flattened and concatenated.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, _Tiny, install_reference  # noqa: E402

CASES = (("adam", "adam", False), ("sgd_trick_nesterov", "sgd_trick", True), ("f3_trick_nesterov", "f3_trick", True))


def optim_ext_kats():
    from utils.pipeline_ops import CustomScheduler, make_optimizer
    out = {}
    for tag, kind, nesterov in CASES:
        torch.manual_seed(3)
        net = _Tiny()
        opt = make_optimizer(net, kind, dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=nesterov))
        named = list(net.named_parameters())
        out[f"{tag}/names"] = np.array([n for n, _ in named])
        out[f"{tag}/group_of"] = np.array([next((gi for gi, g in enumerate(opt.param_groups) if any(p is q for q in g["params"])), -1)
                                           for _, p in named])
        out[f"{tag}/group_lr"] = np.array([g["lr"] for g in opt.param_groups])
        out[f"{tag}/group_wd"] = np.array([g["weight_decay"] for g in opt.param_groups])
        if kind == "adam":
            out[f"{tag}/group_betas"] = np.array([g["betas"] for g in opt.param_groups])
            out[f"{tag}/group_eps"] = np.array([g["eps"] for g in opt.param_groups])
        else:
            out[f"{tag}/group_nesterov"] = np.array([g["nesterov"] for g in opt.param_groups])
        out[f"{tag}/p0"] = np.concatenate([p.detach().numpy().ravel() for p in net.parameters()])
        sched = CustomScheduler(opt, total_num=4, scheduler_type="poly", scheduler_info=dict(lr_decay=0.9, warmup_epoch=1))
        g = torch.Generator().manual_seed(11)
        for it in range(4):
            sched.step(opt, curr_epoch=it)
            out[f"{tag}/lr{it}"] = np.array([gr["lr"] for gr in opt.param_groups])
            grads = []
            for p in net.parameters():
                p.grad = torch.randn(p.shape, generator=g)
                grads.append(p.grad.numpy().ravel().copy())
            out[f"{tag}/g{it}"] = np.concatenate(grads)
            opt.step()
            out[f"{tag}/p{it + 1}"] = np.concatenate([p.detach().numpy().ravel() for p in net.parameters()])
        if kind == "adam":
            sd = opt.state_dict()
            state = [sd["state"][i] for i in range(len(named))]
            out[f"{tag}/state_step"] = np.array([float(s["step"]) for s in state])
            out[f"{tag}/state_exp_avg"] = np.concatenate([s["exp_avg"].numpy().ravel() for s in state])
            out[f"{tag}/state_exp_avg_sq"] = np.concatenate([s["exp_avg_sq"].numpy().ravel() for s in state])
    np.savez_compressed(os.path.join(OUT, "optim_ext_kat.npz"), **out)
    print("optim_ext_kat:", len(out), "arrays")


if __name__ == "__main__":
    install_reference()
    optim_ext_kats()
