"""Checkpoint seam: `save_checkpoint` / `resume_checkpoint` with the reference's signatures and file layout
(reference utils/pipeline_ops.py:46-143; called at train.py:188-201 and :259-270).

Layout kept byte-for-byte compatible at the key level:
    full  : {"arch": exp_name, "epoch": int, "net_state": module.state_dict(), "opti_state": optimizer.state_dict(),
             "amp_state": amp.state_dict() | None}
    state : module.state_dict()
`net_state` keys are the un-prefixed module names (the wrapper's `.module` is unwrapped, utils/pipeline_ops.py:68),
`opti_state` is `torch.optim.SGD`'s state_dict layout (per-parameter `momentum_buffer`) — `FusedSGD.state_dict()`
materialises it from the flat momentum buffer and `load_state_dict` scatters it back, so checkpoints written by
the reference load here and vice versa.  With optim "adam" it is `torch.optim.Adam`'s layout (per-parameter `step`,
`exp_avg`, `exp_avg_sq`), which `FusedAdam` writes and reads the same way.

One deliberate difference (SURVEY Q5): the reference resumes on rank 0 only, leaving the other ranks at their
initial weights; here every rank calls `resume_checkpoint` and loads the same file.
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn
from torch.optim import Optimizer

from .utils import construct_print


def _unwrap(model: nn.Module) -> nn.Module:
    return model.module if hasattr(model, "module") else model


def _compact(obj):
    """detached copies with storage of their own: the live tensors are views into the flat (possibly symmetric-memory)
    buffers, and torch.save serialises the whole underlying storage of a view"""
    if isinstance(obj, torch.Tensor):
        return obj.detach().clone()
    if isinstance(obj, dict):
        return type(obj)((k, _compact(v)) for k, v in obj.items())
    if isinstance(obj, (list, tuple)):
        return type(obj)(_compact(v) for v in obj)
    return obj


def save_checkpoint(model: nn.Module = None, optimizer: Optimizer = None, amp=None, exp_name: str = "", current_epoch: int = 1,
                    full_net_path: str = "", state_net_path: str = "", write: bool | None = None):
    """Full checkpoint (model + optimizer + amp) and the weights-only file, as the reference writes them.

    Distributed: EVERY rank must call this (the momentum of `FusedSGD`, and Adam's two moments, are sharded over the
    ranks and `state_dict()` gathers them with collectives); only the rank with `write=True` (default: rank 0) touches the files, and all ranks
    leave through a barrier so that nobody runs ahead into the next iteration's device-side barriers while rank 0 is
    still writing."""
    import torch.distributed as dist
    distributed = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
    if write is None:
        write = (not distributed) or dist.get_rank() == 0
    opti_state = optimizer.state_dict()                       # collective when the momentum is sharded
    if write:
        net_state = _compact(_unwrap(model).state_dict())
        torch.save({"arch": exp_name, "epoch": current_epoch, "net_state": net_state, "opti_state": _compact(opti_state),
                    "amp_state": amp.state_dict() if amp else None}, full_net_path)
        torch.save(net_state, state_net_path)
    if distributed:
        dist.barrier()


def resume_checkpoint(model: nn.Module = None, optimizer: Optimizer = None, amp=None, exp_name: str = "", load_path: str = "",
                      mode: str = "all", local_rank: int = 0):
    """mode 'all': restore model, optimizer (and amp) and return the epoch to continue from; 'onlynet': weights only.
    Accepts both the full dict and a bare state_dict file for 'onlynet'."""
    if not (os.path.exists(load_path) and os.path.isfile(load_path)):
        raise Exception(f"{load_path}路径不正常，请检查")
    construct_print(f"Loading checkpoint '{load_path}'")
    device = f"cuda:{local_rank}" if torch.cuda.is_available() else "cpu"
    checkpoint = torch.load(load_path, map_location=device, weights_only=False)
    target = _unwrap(model)
    if mode == "all":
        if exp_name != checkpoint["arch"]:
            raise Exception(f"{load_path} does not match.")
        target.load_state_dict(checkpoint["net_state"])
        optimizer.load_state_dict(checkpoint["opti_state"])
        if checkpoint.get("amp_state"):
            if amp:
                amp.load_state_dict(checkpoint["amp_state"])
            else:
                construct_print("You are not using amp.")
        else:
            construct_print("The state_dict of amp is None.")
        construct_print(f"Loaded '{load_path}' (will train at epoch {checkpoint['epoch']})")
        return checkpoint["epoch"]
    if mode == "onlynet":
        state = checkpoint["net_state"] if isinstance(checkpoint, dict) and "net_state" in checkpoint else checkpoint
        target.load_state_dict(state)
        construct_print(f"Loaded checkpoint '{load_path}' (only has the model's weight params)")
        return None
    raise NotImplementedError(mode)
