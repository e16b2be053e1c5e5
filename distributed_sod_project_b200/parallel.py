"""DDP seam: `DistributedDataParallel(model, delay_allreduce=True)` of the reference (apex; train.py:16,185).

Kept: the wrapper is callable like the model, exposes `.module` (relied on by the reference's checkpoint code,
utils/pipeline_ops.py:68,114,133), forwards `.train()/.eval()/.state_dict()`, and at construction makes every
rank start from rank 0's parameters and buffers.

Changed by design: apex flattens all gradients at the end of backward, calls NCCL all-reduce, divides by the
world size and unflattens (four full passes over 99.6 MB plus the collective).  Here the gradients are *born*
in one flat symmetric-memory buffer (each `.grad` is a view), and the averaging is folded into the optimizer
step kernel (`sod_allreduce_sgd` / `sod_allreduce_adam`, csrc/sgd.cu): reduce-scatter over NVSwitch → SGD or Adam
on the owned shard → all-gather of the updated parameters.  `delay_allreduce=True` semantics hold trivially: nothing is
exchanged before backward has finished.  With an optimizer other than FusedSGD / FusedAdam the wrapper falls back to an explicit
in-place peer-memory all-reduce of the flat gradient buffer at the end of backward (`sod_allreduce_f32`).
"""
from __future__ import annotations

import torch.distributed as dist
import torch.nn as nn
from torch.autograd import Variable

from . import comm
from .optim import FlatParams, FusedOptimizer, flat_registry as _flat_registry


class DistributedDataParallel(nn.Module):
    def __init__(self, module: nn.Module, delay_allreduce: bool = True, optimizer: FusedOptimizer | None = None,
                 process_group=None, **_ignored):
        super().__init__()
        self.module = module
        self.world = comm.world_size()
        self.delay_allreduce = delay_allreduce
        self.flat: FlatParams | None = None
        self.arena = None
        self._explicit_allreduce = False
        self._cb_queued = False
        params = [p for p in module.parameters() if p.requires_grad]
        if optimizer is not None:
            self.flat = optimizer.flat
        elif params:
            self.flat = _flat_registry.get(id(params[0]))
        if self.world == 1:
            return
        if self.flat is None:
            # no fused optimizer: own the flat layout (module order) and average explicitly after backward
            self.flat = FlatParams([params], [])
            self._explicit_allreduce = True
        n = self.flat.numel
        self.arena = comm.Arena(payload_bytes=2 * (4 * n + 256) + (2 * n + 256) + 1024, group=process_group)   # p, g fp32 + g bf16
        p_off = self.arena.alloc(4 * n)
        g_off = self.arena.alloc(4 * n)
        self.flat.relocate(self.arena, p_off, g_off)
        # every rank starts from rank 0's weights / buffers (apex DDP ctor)
        dist.broadcast(self.flat.param, 0, group=process_group)
        self.flat.refresh_shadow()
        for b in module.buffers():
            dist.broadcast(b, 0, group=process_group)
        if self._explicit_allreduce:
            for p in params:
                p.register_hook(self._make_hook())

    def _make_hook(self):
        def hook(grad):
            if not self._cb_queued:
                self._cb_queued = True
                Variable._execution_engine.queue_callback(self._allreduce_grads_cb)
            return grad
        return hook

    def _allreduce_grads_cb(self):
        self._cb_queued = False
        self.allreduce_grads()

    def allreduce_grads(self):
        """Materialise the averaged gradients in place (what apex leaves in `.grad` after backward)."""
        if self.world == 1:
            return
        # an optimizer that is not a fused one may have dropped the bound views (torch's zero_grad(set_to_none=True) is the
        # default): autograd then produced fresh .grad tensors OUTSIDE the symmetric buffer.  Fold them in and rebind,
        # so that what is averaged is what backward computed.
        import torch
        from .optim import FlatParams
        with torch.no_grad():
            for p, off in self.flat.slots:
                view = FlatParams._view(self.flat.grad, off, p.data)
                if p.grad is None:
                    view.zero_()                      # no local gradient this time: contribute zeros, not last step's values
                elif p.grad.data_ptr() != view.data_ptr():
                    view.copy_(p.grad)
                    p.grad = view
        self.arena.allreduce_(self.flat.grad_off, self.flat.numel, scale=1.0 / self.world, algo=2)

    def forward(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def state_dict(self, *args, **kwargs):
        return self.module.state_dict(*args, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        return self.module.load_state_dict(*args, **kwargs)
