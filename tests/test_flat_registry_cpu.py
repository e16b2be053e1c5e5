"""The registry that lets DistributedDataParallel find a fused optimizer's flat layout must not keep the flat buffers
alive: every Trainer built in a process (tests, sweeps, a notebook) would otherwise keep its parameter, gradient,
momentum and shadow buffers on the device until exit."""
from __future__ import annotations

import gc
import weakref


def test_flat_buffers_are_freed_with_their_optimizer():
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.optim import flat_registry, make_optimizer
    from distributed_sod_project_b200.parallel import DistributedDataParallel
    model = network.res50()
    opt = make_optimizer(model, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    first = next(p for p in model.parameters() if p.requires_grad)
    assert flat_registry.get(id(first)) is opt.flat
    assert DistributedDataParallel(model).flat is opt.flat
    ref = weakref.ref(opt.flat)
    n = sum(1 for _ in opt.flat.slots)
    before = len(flat_registry)
    del opt
    gc.collect()
    assert ref() is None
    assert len(flat_registry) == before - n
    assert DistributedDataParallel(model).flat is None
