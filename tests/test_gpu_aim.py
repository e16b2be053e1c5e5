"""`aim_res50` / `cp_aim_res50` (ResNet-50, MINet's LightAIM neck, the TestModel decoder) on the engine: the reference's
fp32 trajectories, graph replay and activation checkpointing bit for bit, every parameter gradient against float64, the
backward nodes of a whole forward, the fp16 loss scaler on a neck overflow, the command line, and two ranks.  Each neck
block alone, run through the real Trainer's seams against float64, is a row of tests/test_gpu_block_seams.py."""
from __future__ import annotations

import socket
import sys

import numpy as np
import pytest
import torch

from distributed_sod_project_b200.network import blocks
from _backbones import ROOT, Backbone, _exact, _grads, _run, _train_resume_and_test, _trainer, _world2_steps, amp_reset  # noqa: F401

pytestmark = pytest.mark.gpu
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
DTYPES = [torch.float32, torch.bfloat16, torch.float16]

# the reference's own 64² fp32 logits are already 6.7e-4 (relative) from its float64 ones before any step
ROW = Backbone("aim_res50", frozenset({"div_2.0.weight", "div_2.1.weight", "div_2.1.bias"}),
               plugins=((lambda m: isinstance(m, blocks.LightAIM), 1),), noise_from=0, cli=_train_resume_and_test)


def _node_names(t):
    """names of every autograd node reachable from t"""
    seen, stack, names = set(), [t.grad_fn], []
    while stack:
        fn = stack.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        names.append(type(fn).__name__)
        stack.extend(f for f, _ in fn.next_functions)
    return names


@pytest.mark.parametrize("config,iters", [("w1_s64", 1), ("w1_s128", 2)])
def test_fp32_trajectory_vs_reference(golden, config, iters, amp_reset):  # noqa: F811
    """loss and logits within 1e-3 relative of the reference's fp32 run, or twice the reference's own fp32 distance
    from its float64 run where that is larger (the rule of tests/test_gpu_backbones.py, from iteration 0).  64² at bs 2
    is checked at iteration 0 only, as res50's is kept for first-iteration checks: conv4's BatchNorms there see 8 values
    per channel (a 2×2 map), and one step over the neck's 91 M parameters moves the loss 3.2e-3 (relative) from the
    reference's on an H100, where the 128² run stays within 1e-3"""
    from distributed_sod_project_b200.synthetic import synth_batch
    g = golden(f"step_aim_res50_{config}.npz")
    g64 = golden(f"step_aim_res50_{config}_fp64.npz")
    _, bs, size, _ = (int(v) for v in g["meta"])
    with _exact():
        tr = _trainer(ROW.name, dtype=torch.float32)
        assert [sum(map(pred, tr.model.modules())) for pred, _ in ROW.plugins] == [n for _, n in ROW.plugins]
        for it in range(iters):
            x, m = synth_batch(1234 + 1000 * it, bs, size)
            out = tr.step(x.cuda(), m.cuda())
            ref = float(g[f"loss{it}"][0])
            noise = 0.0 if it < ROW.noise_from else 2 * abs(ref - float(g64[f"loss{it}"][0]))
            assert abs(out["loss"] - ref) <= max(1e-3 * abs(ref), noise), (it, out["loss"], ref)
            if f"logits{it}" in g:
                ref = g[f"logits{it}"]
                got = out["preds"].float().cpu().numpy()
                assert got.shape == ref.shape
                noise = 0.0 if it < ROW.noise_from else 2 * np.abs(ref - g64[f"logits{it}"]).max()
                assert np.abs(got - ref).max() <= max(1e-3 * np.abs(ref).max(), noise), it


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_graph_replay_and_checkpointing_are_bit_identical(dtype, amp_reset):  # noqa: F811
    """eager ≡ CUDA-graph replay and cp_aim_res50 ≡ aim_res50, three iterations, every parameter bit for bit"""
    with _exact():
        ref = _run(ROW.name, dtype, False)
        for name, graph in ((ROW.name, True), (ROW.cp, False), (ROW.cp, True)):
            got = _run(name, dtype, graph)
            assert got[0] == ref[0], (name, graph)
            assert torch.equal(got[1], ref[1]), (name, graph)
    assert all(np.isfinite(ref[0]))


@pytest.mark.parametrize("dtype,A", [(torch.float32, 3.0), (torch.bfloat16, 2.5), (torch.float16, 2.5)], ids=str)
def test_iteration_gradients_match_fp64(dtype, A):
    """the A-rule of tests/test_gpu_model_grads.py: for every parameter P,
    e(engine, P) ≤ A · (e(stock, P) + median_Q e(stock, Q)), e = ‖g − g64‖₂ / ‖g64‖₂, "stock" the torch model in the
    same precision on the same GPU"""
    with _exact():
        ref = _grads(ROW.name, torch.float64, False, 1.0)
        scale = 1024.0 if dtype == torch.float16 else 1.0
        stock = _grads(ROW.name, dtype, False, scale)
        eng = _grads(ROW.name, dtype, True, scale)
    assert ref.keys() == eng.keys() and ROW.frozen <= ref.keys()
    assert sum(n.startswith("trans.") for n in ref) == 2 * 65 + 2 * 36
    e = lambda g, n: float((g[n] - ref[n]).norm() / ref[n].norm().clamp_min(1e-300))  # noqa: E731
    es = {n: e(stock, n) for n in ref}
    med = float(np.median(list(es.values())))
    worst = max((e(eng, n) / (es[n] + med), n) for n in ref)
    assert worst[0] <= A, f"{worst[1]}: engine error {worst[0]:.2f}x (stock + median)"


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_whole_model_backward_nodes(dtype, amp_reset):  # noqa: F811
    """one trainer forward: 12 nearest up-samples and 12 neck average pools (22 with the five SIMs' ten), one SyncBN
    node per BatchNorm, and under amp the five biased `identity` convolutions on `_ConvBias` (bias gradient by
    sod_colsum)"""
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(ROW.name, dtype=dtype)
    x, _ = synth_batch(3, 2, 64)
    preds = tr.model(x.cuda().contiguous(memory_format=torch.channels_last))
    names = _node_names(preds)
    assert names.count("_UpNearest2xBackward") == 12
    assert names.count("_AvgPool2x2Backward") == 12 + 10
    assert names.count("_SyncBNFnBackward") == sum(isinstance(m, torch.nn.BatchNorm2d) for m in tr.module.modules())
    assert names.count("_ConvBiasBackward") == (5 if dtype != torch.float32 else 0)


def test_fp16_scaler_skips_and_recovers_on_a_neck_overflow(amp_reset, monkeypatch):  # noqa: F811
    """once the scale has settled (clean steps until one is not skipped), infs written into one channel of the gradient
    conv4's nearest up-sample hands back (1024 channels at S/32) reach conv4's stage-0 weights: the fused step skips and halves the
    scale, and the next clean step trains"""
    from distributed_sod_project_b200 import amp, resample
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(ROW.name, dtype=torch.float16)
    conv = tr.module.trans.conv4.l2l_0
    orig = resample._UpNearest2x.backward
    armed = {"on": False}

    def backward(ctx, dy):
        dx = orig(ctx, dy)
        if armed["on"] and ctx.shape[1] == 1024:
            dx[0, 5].fill_(float("inf"))          # one channel of one sample: past the ReLU mask wherever y > 0
        return dx

    monkeypatch.setattr(resample._UpNearest2x, "backward", staticmethod(backward))
    x, m = synth_batch(5, 2, 64)
    for _ in range(24):
        tr.step(x.cuda(), m.cuda())
        if amp.read_scaler()["found_inf"] == 0:
            break
    assert amp.read_scaler()["found_inf"] == 0
    s0 = amp.read_scaler()["scale"]
    before = conv.weight.detach().clone()
    armed["on"] = True
    tr.step(x.cuda(), m.cuda())
    armed["on"] = False
    st = amp.read_scaler()
    assert st["found_inf"] == 1 and st["scale"] == s0 / 2
    assert torch.equal(conv.weight.detach(), before)
    tr.step(x.cuda(), m.cuda())
    st = amp.read_scaler()
    assert st["found_inf"] == 0 and not torch.equal(conv.weight.detach(), before)
    assert bool(torch.isfinite(conv.weight).all())


def test_train_and_test_cli():
    """train.py (CUDA graph, a checkpoint per epoch, resume) and test.py with "model": "aim_res50" at input 96"""
    ROW.cli(ROW.name)


def _aim_world2_entry(rank, world, port):
    """`torch.multiprocessing.spawn` target: one rank of the two-rank check"""
    import os
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        _world2_steps(rank, ROW)
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(NGPU < 2, reason="needs 2 GPUs")
def test_training_step_world2_vs_reference():
    """two ranks against the reference's two-rank fp32 trajectory (`_backbones._world2_steps`)"""
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_aim_world2_entry, args=(2, port), nprocs=2, join=True)
