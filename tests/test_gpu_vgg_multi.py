"""`vgg16` at world 2 against the reference's two-rank fp32 trajectory (step_vgg16_w2_s64, the concatenated-batch
construction of tools/make_golden.py): per-rank losses of two iterations, and identical parameters on both ranks.
Needs two GPUs; skipped otherwise."""
from __future__ import annotations

import os
import socket
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _entry(rank, world, port):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        _w_step(rank)
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _w_step(rank):
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.loss import get_total_loss
    from distributed_sod_project_b200.synthetic import synth_batch
    g = np.load(os.path.join(ROOT, "tests", "golden", "step_vgg16_w2_s64.npz"))
    g64 = np.load(os.path.join(ROOT, "tests", "golden", "step_vgg16_w2_s64_fp64.npz"))
    _, bs, size, _ = (int(v) for v in g["meta"])
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    tr = Trainer(model_name="vgg16", dtype=torch.float32, channels_last=True)
    for it in range(2):
        x, m = synth_batch(1234 + rank + 1000 * it, bs, size)
        preds = tr.model(x.cuda().contiguous(memory_format=torch.channels_last))
        loss, _ = get_total_loss(preds, m.cuda(), tr.loss_funcs, unit_upstream=True)
        tr.optimizer.zero_grad(); loss.backward(); tr.optimizer.step()
        want = float(g[f"loss{it}"][rank])
        tol = 1e-3 * abs(want) if it == 0 else max(1e-3 * abs(want), 2 * abs(want - float(g64[f"loss{it}"][rank])))
        assert abs(float(loss) - want) <= tol, (rank, it, float(loss), want)
        flat = tr.optimizer.flat.param
        other = flat.clone(); torch.distributed.broadcast(other, 0)
        assert torch.equal(flat, other)
    tr.model.arena.check_error()


@pytest.mark.skipif(NGPU < 2, reason="needs 2 GPUs")
def test_training_step_world2_vs_reference():
    import torch.multiprocessing as mp
    mp.spawn(_entry, args=(2, _free_port()), nprocs=2, join=True)
