"""World-size-2 parity of the peer-memory collectives (needs ≥2 GPUs on one NVSwitch domain; skipped otherwise).
Run on a machine with at least two GPUs: `python -m pytest tests/test_gpu_multi.py -m gpu`."""
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
def _w_allreduce(rank, world):
    from distributed_sod_project_b200 import comm
    arena = comm.Arena(payload_bytes=(64 << 20) + 4096)
    off = arena.alloc(64 << 20)
    for n in (4, 1024, 65536 + 4, 1 << 20, (16 << 20) // 4 + 8):
        for algo, nomc in ((2, False), (2, True), (1, False), (0, False)):
            if algo == 1 and n * 4 > (1 << 20):
                continue
            buf = arena.view(off, n, torch.float32)
            g = torch.Generator().manual_seed(100 + rank)
            mine = torch.randn(n, generator=g)
            buf.copy_(mine)
            torch.cuda.synchronize(); torch.distributed.barrier()
            arena.allreduce_(off, n, scale=0.5, algo=algo, no_multimem=nomc)
            torch.cuda.synchronize()
            want = sum(torch.randn(n, generator=torch.Generator().manual_seed(100 + r)) for r in range(world)) * 0.5
            got = buf.cpu()
            assert torch.allclose(got, want, rtol=1e-6, atol=1e-6), (n, algo, nomc, (got - want).abs().max())
            torch.distributed.barrier()
    arena.check_error()
    # scalar mean used for logging (reference utils/tensor_ops.py:60-64)
    t = torch.tensor([float(rank + 1)], device="cuda")
    assert float(comm.allreduce_tensor(t)) == pytest.approx((1 + world) / 2)


@needs2
def test_allreduce_variants():
    _spawn("_w_allreduce")


def _w_allreduce_sgd(rank, world):
    from oracle import sgd as osgd
    from distributed_sod_project_b200 import _lib, comm
    n = 1_000_000 + 64
    arena = comm.Arena(payload_bytes=2 * 4 * n + 4096)
    p_off, g_off = arena.alloc(4 * n), arena.alloc(4 * n)
    rng = np.random.default_rng(5)
    p0 = rng.standard_normal(n).astype(np.float32); v0 = rng.standard_normal(n).astype(np.float32)
    grads = [np.random.default_rng(50 + r).standard_normal(n).astype(np.float32) for r in range(world)]
    a, b = (n // 3) // 4 * 4, (2 * n // 3) // 4 * 4
    segs_o = [osgd.Segment(0, a, 0.005, 5e-4, 0.9), osgd.Segment(a, b, 0.05, 5e-4, 0.9), osgd.Segment(b, n, 0, 0, frozen=True)]
    segs = (_lib.sod_sgd_segment * 3)(_lib.sod_sgd_segment(0, a, 0.005, 5e-4, 0.9, 0), _lib.sod_sgd_segment(a, b, 0.05, 5e-4, 0.9, 0),
                                      _lib.sod_sgd_segment(b, n, 0, 0, 0, 1))
    pe, ve = p0.copy(), v0.copy()
    for flags in (_lib.SOD_SGD_ZERO_GRAD, _lib.SOD_SGD_ZERO_GRAD | _lib.SOD_ALGO_NO_MULTIMEM):
        p = arena.view(p_off, n, torch.float32); g = arena.view(g_off, n, torch.float32)
        mom = torch.tensor(ve, device="cuda")
        p.copy_(torch.tensor(pe)); g.copy_(torch.tensor(grads[rank]))
        torch.cuda.synchronize(); torch.distributed.barrier()
        rc = _lib.lib().sod_allreduce_sgd(arena.ref, g_off, 0, p_off, mom.data_ptr(), None, n, segs, 3, None, 0.5, None, flags,
                                          torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize(); torch.distributed.barrier()
        gm = osgd.allreduce_mean(grads)
        assert osgd.sgd_step(pe, ve, gm, segs_o, inv_scale=0.5)
        np.testing.assert_allclose(p.cpu().numpy(), pe, rtol=3e-6, atol=1e-6)
        shard = (n // 4 + world - 1) // world * 4
        lo, hi = rank * shard, min(n, (rank + 1) * shard)
        np.testing.assert_allclose(mom.cpu().numpy()[lo:hi], ve[lo:hi], rtol=3e-6, atol=1e-6)   # momentum: owned shard only
        assert float(g.abs().max()) == 0.0
        # bit-identical parameters on every rank (owner computes, then broadcast)
        mine = p.clone(); other = p.clone()
        torch.distributed.broadcast(other, 0)
        assert torch.equal(mine, other)
        ve = v0.copy() if False else ve
        # next round starts from the same full momentum on both ranks (test convenience)
        full = torch.tensor(ve, device="cuda")
        ve = full.cpu().numpy()
    arena.check_error()


@needs2
def test_allreduce_sgd_vs_oracle():
    _spawn("_w_allreduce_sgd")


def _w_syncbn(rank, world):
    from oracle import syncbn as obn
    from distributed_sod_project_b200.syncbn import SyncBatchNorm
    for (shape, dtype, variant) in [((4, 64, 20, 20), torch.float32, "all"), ((2, 2048, 2, 2), torch.float32, "relu"),
                                    ((16, 256, 20, 20), torch.bfloat16, "res_relu"), ((3, 32, 9, 7), torch.float32, "plain"),
                                    ((8, 512, 10, 10), torch.bfloat16, "pre_relu")]:
        n, c, h, w = shape
        def mk(seed, r, scale=1.0, shift=0.0):
            g = torch.Generator().manual_seed(seed * 10 + r)
            return (torch.randn(shape, generator=g) * scale + shift).to(dtype)
        xs = [mk(1, r, 1.5, 0.2 * r) for r in range(world)]
        pres = [mk(2, r) for r in range(world)] if variant in ("pre_relu", "all") else None
        ress = [mk(3, r) for r in range(world)] if variant in ("res_relu", "all") else None
        dys = [mk(4, r) for r in range(world)]
        relu = variant != "plain"
        bn = SyncBatchNorm(c).cuda()
        with torch.no_grad():
            bn.weight.copy_(torch.linspace(0.5, 1.5, c)); bn.bias.copy_(torch.linspace(-0.3, 0.3, c))
        cl = lambda t: t.cuda().contiguous(memory_format=torch.channels_last)  # noqa: E731
        x = cl(xs[rank]).requires_grad_(True)
        pre = cl(pres[rank]).requires_grad_(True) if pres else None
        res = cl(ress[rank]).requires_grad_(True) if ress else None
        y = bn.fused_forward(x, pre_add=pre, residual=res, relu=relu)
        y.backward(cl(dys[rank]))
        torch.cuda.synchronize()
        f64 = lambda t: t.detach().float().cpu().numpy().astype(np.float64)  # noqa: E731
        ref = obn.syncbn_forward([f64(t) for t in xs], f64(bn.weight), f64(bn.bias), np.zeros(c), np.ones(c),
                                 pre_adds=[f64(t) for t in pres] if pres else None,
                                 residuals=[f64(t) for t in ress] if ress else None, relu=relu)
        tol = dict(rtol=2e-2, atol=2e-2) if dtype != torch.float32 else dict(rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(f64(y), ref["ys"][rank], **tol)
        np.testing.assert_allclose(f64(bn.running_mean), ref["running_mean"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(f64(bn.running_var), ref["running_var"], rtol=1e-3, atol=1e-5)
        ys_for_mask = [ref["ys"][r] for r in range(world)]
        ys_for_mask[rank] = f64(y)
        rb = obn.syncbn_backward([f64(t) for t in dys], ref["zs"], ys_for_mask, ref["mean"], ref["invstd"], f64(bn.weight), relu=relu)
        gs = max(np.abs(rb["dzs"][rank]).max(), 1e-6)
        assert np.abs(f64(x.grad) - rb["dzs"][rank]).max() / gs < (3e-2 if dtype != torch.float32 else 3e-4), (shape, variant)
        np.testing.assert_allclose(f64(bn.weight.grad), rb["dgammas"][rank], rtol=3e-2 if dtype != torch.float32 else 1e-3,
                                   atol=(3e-1 if dtype != torch.float32 else 1e-3))
        torch.distributed.barrier()
    # folded conv bias across ranks: the bias gradient is the LOCAL Σ dz (non-zero per rank, zero in the rank sum)
    shape, c = (4, 64, 12, 12), 64
    g = torch.Generator().manual_seed(77)
    b_cpu = torch.randn(c, generator=g)
    xs = [(torch.randn(shape, generator=torch.Generator().manual_seed(500 + r)) * (1 + r) + 0.3 * r) for r in range(world)]
    dys = [torch.randn(shape, generator=torch.Generator().manual_seed(600 + r)) for r in range(world)]
    bn = SyncBatchNorm(c).cuda()
    b = b_cpu.cuda().requires_grad_(True)
    x = xs[rank].cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = bn.fused_forward(x, relu=True, conv_bias=(b, None))
    y.backward(dys[rank].cuda().contiguous(memory_format=torch.channels_last))
    torch.cuda.synchronize()
    f64 = lambda t: t.detach().float().cpu().numpy().astype(np.float64)  # noqa: E731
    bb = f64(b_cpu)[None, :, None, None]
    ref = obn.syncbn_forward([f64(t) + bb for t in xs], f64(bn.weight), f64(bn.bias), np.zeros(c), np.ones(c), relu=True)
    np.testing.assert_allclose(f64(y), ref["ys"][rank], rtol=1e-4, atol=1e-4)
    ys_mask = [ref["ys"][r] for r in range(world)]; ys_mask[rank] = f64(y)
    rb = obn.syncbn_backward([f64(t) for t in dys], ref["zs"], ys_mask, ref["mean"], ref["invstd"], f64(bn.weight), relu=True)
    np.testing.assert_allclose(f64(x.grad), rb["dzs"][rank], rtol=2e-3, atol=2e-4)
    want_db = rb["dzs"][rank].sum(axis=(0, 2, 3))
    assert np.abs(want_db).max() > 1e-2                      # genuinely non-zero per rank
    np.testing.assert_allclose(f64(b.grad), want_db, rtol=2e-3, atol=2e-3)
    from distributed_sod_project_b200 import comm
    comm.small_arena().check_error()


@needs2
def test_syncbn_world2_vs_oracle():
    _spawn("_w_syncbn")


def _w_step(rank, world):
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    g = np.load(os.path.join(ROOT, "tests", "golden", "step_res50_w2_s128.npz"))
    _, bs, size, iters = (int(v) for v in g["meta"])
    golden_ok = world == 2          # the reference trajectory was generated for two ranks
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    tr = Trainer(model_name="res50", dtype=torch.float32, channels_last=True)
    for it in range(3):
        x, m = synth_batch(1234 + rank + 1000 * it, bs, size)
        preds = tr.model(x.cuda().contiguous(memory_format=torch.channels_last))
        from distributed_sod_project_b200.loss import get_total_loss
        loss, items = get_total_loss(preds, m.cuda(), tr.loss_funcs, unit_upstream=True)
        tr.optimizer.zero_grad(); loss.backward(); tr.optimizer.step()
        assert np.isfinite(float(loss))
        if golden_ok:
            want = float(g[f"loss{it}"][rank])
            # iterations 0 and 1: north_star's 1e-3.  Iteration 2: the reference's own float32 run is 3.9e-3 from its float64
            # run at this configuration (profiles/r02_reference_fp32_vs_fp64.txt, "bs 8 size 128 iter 2"): 5e-3
            assert float(loss) == pytest.approx(want, rel=1e-3 if it < 2 else 5e-3), (rank, it, float(loss), want)
        if it == 0 and golden_ok:
            ref_l = g["logits0"][rank * bs:(rank + 1) * bs]
            got = preds.detach().float().cpu().numpy()
            assert np.abs(got - ref_l).max() / np.abs(ref_l).max() < 1e-3
        # all ranks hold bit-identical parameters after the fused step
        flat = tr.optimizer.flat.param
        other = flat.clone(); torch.distributed.broadcast(other, 0)
        assert torch.equal(flat, other)
    tr.model.arena.check_error()


@needs2
def test_training_step_world2_vs_reference():
    _spawn("_w_step")


def _w_stress(rank, world):
    """many back-to-back collectives with deliberately skewed ranks: no deadlock, no stale packet is ever consumed"""
    import time
    from distributed_sod_project_b200 import comm
    from distributed_sod_project_b200.syncbn import SyncBatchNorm
    bn = SyncBatchNorm(64).cuda()
    x = torch.full((2, 64, 8, 8), float(rank + 1), device="cuda").contiguous(memory_format=torch.channels_last)
    for i in range(300):
        if i % 37 == rank * 11:
            time.sleep(0.01)                      # skew
        xi = x * (i + 1)
        y = bn.fused_forward(xi)
        # rank r holds the constant (r+1)(i+1) ⇒ mean = (i+1)(W+1)/2, biased var = (i+1)²(W²-1)/12 (γ=1, β=0)
        want = (rank + 1 - (world + 1) / 2) / ((world * world - 1) / 12) ** 0.5
        assert torch.allclose(y, torch.full_like(y, want), atol=2e-3), (i, float(y.mean()), want)
    comm.small_arena().check_error()


@needs2
def test_skewed_ranks_stress():
    _spawn("_w_stress")


def _w_checkpoint(rank, world, tmpdir):
    """train 3 steps → save (collective: the momentum is sharded over the ranks) → step 4; a fresh process state resumed
    from the file must produce the SAME step 4 bit for bit (reference utils/pipeline_ops.py:46-143; SURVEY §8e
    'gather-on-save')."""
    from distributed_sod_project_b200 import comm
    from distributed_sod_project_b200.checkpoint import resume_checkpoint, save_checkpoint
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    full, state = os.path.join(tmpdir, "full.pth.tar"), os.path.join(tmpdir, "state.pth")

    def batch(it):
        x, m = synth_batch(1234 + rank + 1000 * it, 2, 64)
        return x.cuda(), m.cuda()

    tr = Trainer(model_name="res50", dtype=torch.float32, channels_last=True, report_items=False)
    for it in range(3):
        tr.forward_backward_update(*batch(it))
    save_checkpoint(model=tr.model, optimizer=tr.optimizer, amp=None, exp_name="ckpt_test", current_epoch=1,
                    full_net_path=full, state_net_path=state)
    # what was written: full-length momentum with EVERY shard populated, compact storages
    if rank == 0:
        ck = torch.load(full, map_location="cpu", weights_only=False)
        sd = ck["opti_state"]
        bufs = [s["momentum_buffer"] for s in sd["state"].values()]
        assert len(bufs) == sum(len(g["params"]) for g in sd["param_groups"])
        big = [b for b in bufs if b.numel() > 10000]
        assert all(float(b.abs().max()) > 0 for b in big)                  # no stale all-zero shard
        assert all(b.untyped_storage().nbytes() == b.numel() * 4 for b in bufs)
        assert os.path.getsize(full) < 2.3 * 4 * tr.optimizer.flat.numel     # ≈ params + momentum, not the whole arena
    loss4, _, _ = tr.forward_backward_update(*batch(3))
    want_p, want_loss = tr.optimizer.flat.param.clone(), float(loss4)
    lo, hi = tr.optimizer.shard_bounds(rank, world)
    want_v = tr.optimizer.flat.mom[lo:hi].clone()

    tr2 = Trainer(model_name="res50", dtype=torch.float32, channels_last=True, report_items=False, seed=123)   # different init
    epoch = resume_checkpoint(model=tr2.model, optimizer=tr2.optimizer, amp=None, exp_name="ckpt_test", load_path=full,
                              mode="all", local_rank=rank)
    assert epoch == 1
    loss4b, _, _ = tr2.forward_backward_update(*batch(3))
    assert float(loss4b) == want_loss
    assert torch.equal(tr2.optimizer.flat.param, want_p)
    assert torch.equal(tr2.optimizer.flat.mom[lo:hi], want_v)
    tr.check_errors(); tr2.check_errors()


@needs2
def test_checkpoint_roundtrip_with_sharded_momentum(tmp_path):
    _spawn("_w_checkpoint", args=(str(tmp_path),))


def _w_adam(rank, world):
    """an optimizer other than FusedSGD (make_optimizer('adam') → torch Adam, whose zero_grad drops the bound .grad
    views): the wrapper must still average what backward computed."""
    from distributed_sod_project_b200.parallel import DistributedDataParallel
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4)).cuda()
    ddp = DistributedDataParallel(net, delay_allreduce=True)
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    for it in range(3):
        g = torch.Generator().manual_seed(100 * it + rank)
        x = torch.randn(8, 16, generator=g).cuda()
        opt.zero_grad()                                   # set_to_none=True: autograd will allocate fresh gradients
        twin = {k: v.detach().clone().requires_grad_(True) for k, v in net.named_parameters()}     # no hooks on these
        local = torch.autograd.grad(torch.func.functional_call(net, twin, (x,)).pow(2).mean(), list(twin.values()))
        want = []
        for t in local:
            t = t.clone(); torch.distributed.all_reduce(t); want.append(t / world)
        ddp(x).pow(2).mean().backward()
        torch.cuda.synchronize()
        for p, w in zip(net.parameters(), want):
            assert torch.allclose(p.grad, w, rtol=1e-5, atol=1e-7), it
        opt.step()
        ref = [p.detach().clone() for p in net.parameters()]
        for r in ref:
            torch.distributed.broadcast(r, 0)
        assert all(torch.equal(a, b) for a, b in zip(ref, net.parameters()))
    ddp.arena.check_error()


@needs2
def test_non_fused_optimizer_gets_averaged_gradients():
    _spawn("_w_adam")


def _w_graph_step(rank, world):
    """the configuration the scaling bench runs: bf16, shadow weights, stolen weight gradients gathered by one launch,
    whole iteration replayed as a CUDA graph with the learning rate moving underneath — against the eager run of the
    same thing, and bit-identical parameters on all ranks throughout."""
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    runs = {}
    for use_graph in (False, True):
        tr = Trainer(model_name="res50", dtype=torch.bfloat16, channels_last=True, report_items=False, use_graph=use_graph)
        sched = tr.scheduler(total_num=5, lr_type="poly")
        losses = []
        for it in range(5):
            sched.step(tr.optimizer, curr_epoch=it)
            x, m = synth_batch(1234 + rank + 1000 * it, 4, 64 if it % 2 else 96)
            red, _, _ = tr.forward_backward_update(x.cuda(), m.cuda())
            losses.append(float(red))
            flat = tr.optimizer.flat.param
            other = flat.clone(); torch.distributed.broadcast(other, 0)
            assert torch.equal(flat, other), (use_graph, it)
        runs[use_graph] = (losses, tr.optimizer.flat.param.clone())
        tr.check_errors()
    # iterations 0-1 tight; later ones only as close as two bf16 runs stay (see test_gpu_step.py, same test at world 1)
    assert runs[True][0][:2] == pytest.approx(runs[False][0][:2], rel=3e-3)
    assert runs[True][0] == pytest.approx(runs[False][0], rel=5e-2)


@needs2
def test_graph_replay_world2_matches_eager():
    _spawn("_w_graph_step")


def _w_allreduce_sgd_bf16_wire(rank, world):
    """ABI v7: ranges flagged SOD_SEG_GRAD16 are reduced from the symmetric bf16 gradient buffer (the bf16 values cross
    NVLink, fp32 sum in rank order), the rest from the fp32 buffer — against the oracle on the same (bf16-rounded) inputs"""
    from oracle import sgd as osgd
    from distributed_sod_project_b200 import _lib, comm
    n = 1_000_000 + 64
    arena = comm.Arena(payload_bytes=2 * 4 * n + 2 * n + 4096)
    p_off, g_off, h_off = arena.alloc(4 * n), arena.alloc(4 * n), arena.alloc(2 * n)
    rng = np.random.default_rng(5)
    p0 = rng.standard_normal(n).astype(np.float32); v0 = rng.standard_normal(n).astype(np.float32)
    a, b = (n // 3) // 4 * 4, (2 * n // 3) // 4 * 4
    g32 = [np.random.default_rng(50 + r).standard_normal(n).astype(np.float32) for r in range(world)]
    g16 = [torch.tensor(np.random.default_rng(90 + r).standard_normal(n).astype(np.float32)).to(torch.bfloat16) for r in range(world)]
    # effective gradient per rank: bf16 buffer in [0, a), fp32 buffer in [a, b); [b, n) frozen
    eff = [np.concatenate([g16[r][:a].float().numpy(), g32[r][a:]]) for r in range(world)]
    segs_o = [osgd.Segment(0, a, 0.005, 5e-4, 0.9), osgd.Segment(a, b, 0.05, 5e-4, 0.9), osgd.Segment(b, n, 0, 0, frozen=True)]
    segs = (_lib.sod_sgd_segment * 3)(_lib.sod_sgd_segment(0, a, 0.005, 5e-4, 0.9, _lib.SOD_SEG_GRAD16), _lib.sod_sgd_segment(a, b, 0.05, 5e-4, 0.9, 0),
                                      _lib.sod_sgd_segment(b, n, 0, 0, 0, _lib.SOD_SEG_FROZEN))
    for flags in (_lib.SOD_SGD_ZERO_GRAD, _lib.SOD_SGD_ZERO_GRAD | _lib.SOD_ALGO_NO_MULTIMEM):
        p = arena.view(p_off, n, torch.float32); g = arena.view(g_off, n, torch.float32); h = arena.view(h_off, n, torch.bfloat16)
        mom = torch.tensor(v0, device="cuda"); shadow = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
        p.copy_(torch.tensor(p0)); g.copy_(torch.tensor(g32[rank])); h.copy_(g16[rank])
        g[:a].fill_(123.0)                                   # garbage in the fp32 buffer where the bf16 one rules
        torch.cuda.synchronize(); torch.distributed.barrier()
        rc = _lib.lib().sod_allreduce_sgd(arena.ref, g_off, h_off, p_off, mom.data_ptr(), shadow.data_ptr(), n, segs, 3, None, 1.0, None, flags,
                                          torch.cuda.current_stream().cuda_stream)
        assert rc == 0
        torch.cuda.synchronize(); torch.distributed.barrier()
        pe, ve = p0.copy(), v0.copy()
        assert osgd.sgd_step(pe, ve, osgd.allreduce_mean(eff), segs_o, inv_scale=1.0)
        np.testing.assert_allclose(p.cpu().numpy(), pe, rtol=3e-6, atol=1e-6)
        shard = (n // 4 + world - 1) // world * 4
        lo, hi = rank * shard, min(n, (rank + 1) * shard)
        np.testing.assert_allclose(mom.cpu().numpy()[lo:hi], ve[lo:hi], rtol=3e-6, atol=1e-6)
        assert float(g[a:].abs().max()) == 0.0 and float(g[:a].min()) == 123.0       # fp32 buffer: cleared only where it is in use
        assert float(h.float().abs().max()) == 0.0
        assert torch.equal(shadow, p.to(torch.bfloat16))
        other = p.clone(); torch.distributed.broadcast(other, 0)
        assert torch.equal(p, other)
        torch.distributed.barrier()
    arena.check_error()


@needs2
def test_allreduce_sgd_bf16_wire_vs_oracle():
    _spawn("_w_allreduce_sgd_bf16_wire")
