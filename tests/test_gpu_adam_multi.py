"""World-size-2 checks of the fused Adam step (`sod_allreduce_adam`, and `FusedAdam` inside the Trainer): needs ≥2 GPUs
on one NVSwitch domain and is skipped otherwise.  `SOD_TEST_WORLD` picks a larger world when more GPUs are present."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
needs2 = pytest.mark.skipif(NGPU < 2, reason="needs 2 GPUs")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _entry(rank, world, port, fn_name, args):
    import sys
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        globals()[fn_name](rank, world, *args)
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _spawn(fn_name, world=None, args=()):
    import torch.multiprocessing as mp
    world = world or max(2, min(NGPU, int(os.environ.get("SOD_TEST_WORLD", "2"))))
    mp.spawn(_entry, args=(world, _free_port(), fn_name, args), nprocs=world, join=True)


# ---------------------------------------------------------------------------------------------------------
def _w_allreduce_adam(rank, world):
    """against dist.all_reduce / W followed by torch.optim.Adam(foreach=False), fp32 gradients and bf16 gradients on the
    wire; parameters and shadow bit-identical on every rank; the moments of the owned shard match"""
    import torch.distributed as dist
    from distributed_sod_project_b200 import _lib, comm
    n = 1_000_000 + 64
    a = (n // 2) // 4 * 4
    arena = comm.Arena(payload_bytes=2 * 4 * n + 2 * n + 4096)
    p_off, g_off, h_off = arena.alloc(4 * n), arena.alloc(4 * n), arena.alloc(2 * n)
    rng = np.random.default_rng(5)
    p0 = torch.tensor(rng.standard_normal(n).astype(np.float32), device="cuda")
    g32 = torch.tensor(np.random.default_rng(50 + rank).standard_normal(n).astype(np.float32), device="cuda")
    g16 = torch.tensor(np.random.default_rng(90 + rank).standard_normal(n).astype(np.float32)).to(torch.bfloat16).cuda()
    shard = (n // 4 + world - 1) // world * 4
    lo, hi = rank * shard, min(n, (rank + 1) * shard)
    for wire16 in (False, True):
        for flags in (_lib.SOD_SGD_ZERO_GRAD, _lib.SOD_SGD_ZERO_GRAD | _lib.SOD_ALGO_NO_MULTIMEM):
            p = arena.view(p_off, n, torch.float32); g = arena.view(g_off, n, torch.float32); h = arena.view(h_off, n, torch.bfloat16)
            m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
            step_dev = torch.zeros(_lib.SOD_ADAM_STEP_WORDS, dtype=torch.int32, device="cuda")
            shadow = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
            ref_p = p0.clone().requires_grad_(True)
            ref = torch.optim.Adam([ref_p], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=5e-4, foreach=False)
            fl = _lib.SOD_SEG_GRAD16 if wire16 else 0
            segs = (_lib.sod_adam_segment * 1)(_lib.sod_adam_segment(0, n, 1e-3, 5e-4, 0.9, 0.999, 1e-8, fl))
            p.copy_(p0)
            for it in range(3):
                mine = (g16.float() if wire16 else g32) * (1.0 + it)
                g.copy_(mine); h.copy_(g16 * (1.0 + it))
                torch.cuda.synchronize(); dist.barrier()
                rc = _lib.lib().sod_allreduce_adam(arena.ref, g_off, h_off if wire16 else 0, p_off, m.data_ptr(), v.data_ptr(),
                                                   shadow.data_ptr(), n, segs, 1, None, step_dev.data_ptr(), 1.0, None, flags,
                                                   torch.cuda.current_stream().cuda_stream)
                assert rc == 0
                want_g = mine.clone(); dist.all_reduce(want_g); want_g /= world
                ref_p.grad = want_g
                ref.step()
                torch.cuda.synchronize(); dist.barrier()
                torch.testing.assert_close(p, ref_p.detach(), rtol=3e-6, atol=1e-6)
                st = ref.state[ref_p]
                torch.testing.assert_close(m[lo:hi], st["exp_avg"][lo:hi], rtol=3e-6, atol=1e-6)
                torch.testing.assert_close(v[lo:hi], st["exp_avg_sq"][lo:hi], rtol=3e-6, atol=1e-9)
                assert step_dev.tolist()[:2] == [it + 1, 0]
                assert float(h.float().abs().max()) == 0.0
                if not wire16:
                    assert float(g.abs().max()) == 0.0
                assert torch.equal(shadow, p.to(torch.bfloat16))
                for t in (p.clone(), shadow.clone()):
                    other = t.clone(); dist.broadcast(other, 0)
                    assert torch.equal(t, other)
                dist.barrier()
    arena.check_error()


@needs2
def test_allreduce_adam_vs_torch_adam():
    _spawn("_w_allreduce_adam")


def _w_trainer_adam(rank, world, tmpdir):
    """FusedAdam in the Trainer at world 2: the gathered state_dict equals a full reference state, save after 3 steps →
    step 4 equals resume → step 4 bit for bit, and graph replay equals the eager run"""
    import torch.distributed as dist
    from distributed_sod_project_b200.checkpoint import resume_checkpoint, save_checkpoint
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    full, state = os.path.join(tmpdir, "full.pth.tar"), os.path.join(tmpdir, "state.pth")

    def batch(it):
        x, m = synth_batch(1234 + rank + 1000 * it, 2, 64)
        return x.cuda(), m.cuda()

    def trainer(**kw):
        return Trainer(model_name="res50", lr=1e-4, optim="adam", dtype=torch.float32, channels_last=True,
                       report_items=False, **kw)

    tr = trainer()
    for it in range(3):
        tr.forward_backward_update(*batch(it))
    opt = tr.optimizer
    sd = opt.state_dict()                                   # collective: gathers both moments
    # every rank holds the same full state, equal to the owners' shards
    for key, buf in (("exp_avg", opt.flat.mom), ("exp_avg_sq", opt.exp_avg_sq)):
        other = buf.clone(); dist.broadcast(other, 0)
        assert torch.equal(buf, other), key
    assert all(float(s["step"]) == 3.0 for s in sd["state"].values())
    assert len(sd["state"]) == sum(len(g["params"]) for g in sd["param_groups"])
    big = [s["exp_avg_sq"] for s in sd["state"].values() if s["exp_avg_sq"].numel() > 10000]
    assert all(float(b.abs().max()) > 0 for b in big)       # no stale all-zero shard
    save_checkpoint(model=tr.model, optimizer=opt, amp=None, exp_name="adam_ckpt", current_epoch=1,
                    full_net_path=full, state_net_path=state)
    loss4, _, _ = tr.forward_backward_update(*batch(3))
    want_p, want_loss = opt.flat.param.clone(), float(loss4)
    lo, hi = opt.shard_bounds(rank, world)
    want_m, want_v = opt.flat.mom[lo:hi].clone(), opt.exp_avg_sq[lo:hi].clone()

    tr2 = trainer(seed=123)
    resume_checkpoint(model=tr2.model, optimizer=tr2.optimizer, amp=None, exp_name="adam_ckpt", load_path=full, mode="all",
                      local_rank=rank)
    assert tr2.optimizer.group_steps() == [3]
    loss4b, _, _ = tr2.forward_backward_update(*batch(3))
    assert float(loss4b) == want_loss
    assert torch.equal(tr2.optimizer.flat.param, want_p)
    assert torch.equal(tr2.optimizer.flat.mom[lo:hi], want_m) and torch.equal(tr2.optimizer.exp_avg_sq[lo:hi], want_v)
    tr.check_errors(); tr2.check_errors()

    runs = {}
    for use_graph in (False, True):
        t = Trainer(model_name="res50", lr=1e-4, optim="adam", dtype=torch.bfloat16, channels_last=True, report_items=False,
                    use_graph=use_graph)
        runs[use_graph] = [float(t.forward_backward_update(*batch(10 + it))[0]) for it in range(3)]
        assert t.optimizer.group_steps() == [3]
        if use_graph:
            assert len(t._graphs) == 1
        t.check_errors()
    assert runs[True][:2] == pytest.approx(runs[False][:2], rel=2e-3)
    assert runs[True] == pytest.approx(runs[False], rel=5e-2)


@needs2
def test_trainer_adam_checkpoint_and_graph_at_world_2(tmp_path):
    _spawn("_w_trainer_adam", args=(str(tmp_path),))
