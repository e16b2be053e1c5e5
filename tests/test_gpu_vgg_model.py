"""`vgg16` / `cp_vgg16` on the engine: the reference's fp32 trajectories, every parameter gradient against float64, graph
replay and activation checkpointing bit for bit, the 2×2 max-pool kernels against torch's op inside a whole iteration,
no torch max-pool kernel in a profiled iteration, `res50`'s iteration unchanged, and the command line."""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_wsgn_model import _exact, _loss, _trainer, amp_reset  # noqa: F401  (amp_reset is a fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# res50 at bs 2, 64², measured on an H100 80GB HBM3 at the parent commit of the VGG16-BN plugins (which change nothing on
# res50's path): library launches of the second iteration, the number of convolutions with a 16-bit shadow, and the
# fused optimizer's segment table as (begin, end, param group index or None for the frozen stem, 16-bit gradients)
_RES50_PLAN16 = [(0, 23445504, 0, True), (23445504, 23498496, 0, False), (23498496, 24894144, 1, True),
                 (24894144, 24898112, 1, False), (24898112, 24907520, None, True), (24907520, 24907648, None, False)]
RES50 = {
    "torch.float32": {"launches": 222, "shadows": 0,
                      "plan": [(0, 23498496, 0, False), (23498496, 24898112, 1, False), (24898112, 24907648, None, False)]},
    "torch.bfloat16": {"launches": 228, "shadows": 105, "plan": _RES50_PLAN16},
    "torch.float16": {"launches": 229, "shadows": 105, "plan": _RES50_PLAN16},
}


def _res50_probe(dtype):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer("res50", dtype=dtype)
    x, m = synth_batch(9, 2, 64)
    tr.step(x.cuda(), m.cuda())
    n0 = _lib.launches
    tr.step(x.cuda(), m.cuda())
    groups = [id(g) for g in tr.optimizer.param_groups]
    plan = [(b, e, None if g is None else groups.index(id(g)), bool(f)) for b, e, g, f in tr.optimizer._segment_plan()]
    return {"launches": _lib.launches - n0, "shadows": sum(hasattr(mm, "_sod_w16") for mm in tr.module.modules()),
            "plan": plan}


@pytest.mark.parametrize("tag", ["vgg16_w1_s64", "vgg16_w1_s128"])
def test_fp32_trajectory_vs_reference(golden, tag, amp_reset):  # noqa: F811
    """iteration 0: loss and logits within 1e-3 relative of the reference's fp32 run (tools/make_golden_vgg.py).
    Iteration 1: within 1e-3, or within twice the reference's own fp32 distance from its float64 run where that is
    larger (one SGD step amplifies fp32 rounding to 1.8e-2 on the reference's own 128² logits)"""
    from distributed_sod_project_b200.network.blocks import _VGGPool
    from distributed_sod_project_b200.synthetic import synth_batch
    g = golden(f"step_{tag}.npz")
    g64 = golden(f"step_{tag}_fp64.npz")
    _, bs, size, _ = (int(v) for v in g["meta"])
    with _exact():
        tr = _trainer("vgg16", dtype=torch.float32)
        assert sum(isinstance(m, _VGGPool) for m in tr.model.modules()) == 4
        for it in range(2):
            x, m = synth_batch(1234 + 1000 * it, bs, size)
            out = tr.step(x.cuda(), m.cuda())
            ref = float(g[f"loss{it}"][0])
            noise = 0.0 if it == 0 else 2 * abs(ref - float(g64[f"loss{it}"][0]))
            assert abs(out["loss"] - ref) <= max(1e-3 * abs(ref), noise), (it, out["loss"], ref)
            if f"logits{it}" in g:
                ref = g[f"logits{it}"]
                got = out["preds"].float().cpu().numpy()
                assert got.shape == ref.shape
                noise = 0.0 if it == 0 else 2 * np.abs(ref - g64[f"logits{it}"]).max()
                assert np.abs(got - ref).max() <= max(1e-3 * np.abs(ref).max(), noise), it


def _run(model_name, dtype, use_graph, steps=3):
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(model_name, dtype=dtype, use_graph=use_graph)
    losses = []
    for it in range(steps):
        x, m = synth_batch(77 + it, 2, 64)
        losses.append(tr.step(x.cuda(), m.cuda())["loss"])
    params = torch.cat([p.detach().reshape(-1).float() for p in tr.module.parameters()]).cpu()
    return losses, params


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_graph_replay_and_checkpointing_are_bit_identical(dtype, amp_reset):  # noqa: F811
    """eager ≡ CUDA-graph replay and cp_vgg16 ≡ vgg16, three iterations, every parameter bit for bit"""
    with _exact():
        ref = _run("vgg16", dtype, False)
        for name, graph in (("vgg16", True), ("cp_vgg16", False), ("cp_vgg16", True)):
            got = _run(name, dtype, graph)
            assert got[0] == ref[0], (name, graph)
            assert torch.equal(got[1], ref[1]), (name, graph)
    assert all(np.isfinite(ref[0]))


def test_maxpool_kernels_off_equals_on(amp_reset, monkeypatch):  # noqa: F811
    """one fp32 iteration under deterministic cuDNN with the 2×2 kernels (the default) and with torch's op
    (`MAXPOOL_ENABLED = False`, what SOD_MAXPOOL=0 sets): loss, logits and every parameter bit for bit"""
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.synthetic import synth_batch
    calls = []
    orig = resample._MaxPool2x2s2.forward

    def fwd(ctx, x):
        calls.append(tuple(x.shape))
        return orig(ctx, x)

    monkeypatch.setattr(resample._MaxPool2x2s2, "forward", staticmethod(fwd))

    def one(enabled):
        monkeypatch.setattr(resample, "MAXPOOL_ENABLED", enabled)
        tr = _trainer("vgg16", dtype=torch.float32)
        x, m = synth_batch(31, 4, 96)
        out = tr.step(x.cuda(), m.cuda())
        params = torch.cat([p.detach().reshape(-1) for p in tr.module.parameters()]).cpu()
        return out["loss"], out["preds"].cpu(), params

    with _exact():
        on = one(True)
        assert calls == [(4, 64, 96, 96), (4, 128, 48, 48), (4, 256, 24, 24), (4, 512, 12, 12)]
        off = one(False)
        assert len(calls) == 4
    assert on[0] == off[0]
    assert torch.equal(on[1].view(torch.int32), off[1].view(torch.int32))
    assert torch.equal(on[2].view(torch.int32), off[2].view(torch.int32))


def test_profiled_iteration_has_no_torch_max_pool(amp_reset):  # noqa: F811
    """a bf16 iteration under torch.profiler: the four pools and their backward run as csrc/maxpool.cu kernels, and no
    `max_pool2d_with_indices` op or torch max-pool kernel appears"""
    from torch.profiler import ProfilerActivity, profile
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer("vgg16", dtype=torch.bfloat16)
    x, m = synth_batch(3, 2, 64)
    tr.step(x.cuda(), m.cuda())
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        tr.step(x.cuda(), m.cuda())
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    assert not [n for n in names if "max_pool" in n], sorted({n for n in names if "max_pool" in n})
    assert sum("maxpool2x2s2_fwd_kernel" in n for n in names) == 4
    assert sum("maxpool2x2s2_bwd_kernel" in n for n in names) == 4


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_res50_iteration_is_unchanged(dtype, amp_reset, monkeypatch):  # noqa: F811
    """res50 never reaches the 2×2 kernels; its launches per iteration, shadow set and segment table are the parent's"""
    from distributed_sod_project_b200 import resample
    monkeypatch.setattr(resample, "maxpool2x2s2", lambda x: pytest.fail("res50 reached the 2x2 max-pool"))
    assert _res50_probe(dtype) == RES50[str(dtype)]


# -- every parameter gradient of one iteration against float64 -------------------------------------------------------
def _grads(dtype, engine_side: bool, scale: float):
    from distributed_sod_project_b200 import network, resample
    from distributed_sod_project_b200.network import blocks
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    from distributed_sod_project_b200.synthetic import synth_batch
    from distributed_sod_project_b200.utils import init_seed
    x, m = synth_batch(1234, 4, 128)
    init_seed(0)
    model = network.vgg16()
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    resample.ENABLED = blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = engine_side
    try:
        if dtype == torch.float64:
            model, x, m = model.double().cuda(), x.double().cuda(), m.double().cuda()
        else:
            model = model.cuda().to(memory_format=torch.channels_last)
            x, m = x.cuda().contiguous(memory_format=torch.channels_last), m.cuda()
            if engine_side:
                model = convert_syncbn_model(model)
        model.train()
        with torch.autocast("cuda", dtype=dtype, enabled=dtype in (torch.bfloat16, torch.float16)):
            preds = model(x)
        (_loss(preds.to(m.dtype), m) * scale).backward()
    finally:
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old
    return {n: p.grad.double() / scale for n, p in model.named_parameters()}


@pytest.mark.parametrize("dtype,A", [(torch.float32, 3.0), (torch.bfloat16, 2.5), (torch.float16, 2.5)], ids=str)
def test_iteration_gradients_match_fp64(dtype, A):
    """the A-rule of tests/test_gpu_model_grads.py (DESIGN §2): for every parameter P,
    e(engine, P) ≤ A · (e(stock, P) + median_Q e(stock, Q)), e = ‖g − g64‖₂ / ‖g64‖₂, "stock" the torch model
    (nn.BatchNorm2d, nn.MaxPool2d) in the same precision on the same GPU.  div_2's gradients are included: they are
    computed, as in the reference, though f3_trick leaves div_2 out of the optimizer"""
    with _exact():
        ref = _grads(torch.float64, False, 1.0)
        scale = 1024.0 if dtype == torch.float16 else 1.0
        stock = _grads(dtype, False, scale)
        eng = _grads(dtype, True, scale)
    assert "div_2.0.bias" in ref and len(ref) == len(eng)
    e = lambda g, n: float((g[n] - ref[n]).norm() / ref[n].norm().clamp_min(1e-300))  # noqa: E731
    es = {n: e(stock, n) for n in ref}
    med = float(np.median(list(es.values())))
    worst = max((e(eng, n) / (es[n] + med), n) for n in ref)
    assert worst[0] <= A, f"{worst[1]}: engine error {worst[0]:.2f}x (stock + median)"


def test_train_resume_and_test_cli():
    """train.py with "model": "vgg16" on CUDA graphs: 2 epochs with validation and a checkpoint each; the checkpoint,
    marked as written after epoch 1 (a run stopped there), resumed with resume_mode "train", which trains epoch 2 only;
    then test.py on the saved weights"""
    import glob
    common = {"epoch_num": 2, "synthetic_iters_per_epoch": 2, "batch_size": 4, "print_freq": 1, "save_freq": 1,
              "is_distributed": False, "input_size": 96, "model": "vgg16", "synthetic_eval_images": 5, "val_freq": 1,
              "final_test": False, "cuda_graph": True}

    def run(script, cfg, *args):
        env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
        out = subprocess.run([sys.executable, os.path.join(ROOT, script), *args], cwd=ROOT, env=env, capture_output=True,
                             text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-3000:]
        return out.stdout

    out = run("train.py", common, "-ng", "1", "-p", "29713")
    assert "End Training" in out and out.count("[I:") == 4 and out.count("'MAE':") == 2
    saved = glob.glob(os.path.join(ROOT, "output*", "vgg16_SIZE96_BS4_*_E2_*", "pth", "checkpoint_final.pth.tar"))
    assert len(saved) == 1, saved
    ck = torch.load(saved[0], map_location="cpu", weights_only=False)
    assert ck["epoch"] == 2
    ck["epoch"] = 1
    torch.save(ck, saved[0])
    out = run("train.py", dict(common, resume_mode="train"), "-ng", "1", "-p", "29714")
    assert "End Training" in out and out.count("[I:") == 2 and "[E:1:2]" in out and "[E:0:" not in out
    out = run("test.py", dict(common, resume_mode="test"))
    assert out.count("'MAE':") == 6
