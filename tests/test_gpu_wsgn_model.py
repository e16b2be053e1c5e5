"""`wsgn_res50` / `cp_wsgn_res50` on the engine: the reference's fp32 trajectory, every parameter gradient against float64,
graph replay and activation checkpointing bit for bit, the fp16 loss scaler on a WS gradient, and `res50` untouched."""
from __future__ import annotations

import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _exact():
    """TF32 off and deterministic cuDNN: what bit-for-bit comparisons and the fp32 trajectory need"""
    b = torch.backends
    old = b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic, b.cudnn.benchmark
    b.cudnn.allow_tf32 = b.cuda.matmul.allow_tf32 = False
    b.cudnn.deterministic, b.cudnn.benchmark = True, False
    try:
        yield
    finally:
        b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic, b.cudnn.benchmark = old


@pytest.fixture
def amp_reset():
    from distributed_sod_project_b200 import amp
    saved = dict(amp._cfg)
    yield
    amp._cfg.clear()
    amp._cfg.update(saved)


def _trainer(model_name="wsgn_res50", **kw):
    from distributed_sod_project_b200.engine import Trainer
    return Trainer(model_name=model_name, lr=0.05, momentum=0.9, weight_decay=5e-4, **kw)


@pytest.mark.parametrize("tag", ["wsgn_res50_w1_s64", "wsgn_res50_w1_s128"])
def test_fp32_trajectory_vs_reference(golden, tag, amp_reset):
    """north_star rule: iteration 0 loss and logits within 1e-3 relative of the reference's fp32 run on the WS-GN
    backbone (tools/make_golden_wsgn.py).  Iteration 1: within 1e-3, or within twice the reference's own fp32 distance
    from its float64 run where that is larger — one SGD step of this model amplifies fp32 rounding to ~1e-2 on the 64²
    loss and ~4e-2 on the 128² logits in the reference itself (the `_fp64` vectors), which no fp32 run can beat"""
    from distributed_sod_project_b200.synthetic import synth_batch
    g = golden(f"step_{tag}.npz")
    g64 = golden(f"step_{tag}_fp64.npz")
    world, bs, size, _ = (int(v) for v in g["meta"])
    with _exact():
        tr = _trainer(dtype=torch.float32)
        assert sum(type(m).__name__ == "GroupNorm32" for m in tr.model.modules()) == 53
        assert sum(type(m).__name__ == "FusedWSConv2d" for m in tr.model.modules()) == 53
        for it in range(2):
            x, m = synth_batch(1234 + 1000 * it, bs, size)
            out = tr.step(x.cuda(), m.cuda())
            ref = float(g[f"loss{it}"][0])
            noise = 0.0 if it == 0 else 2 * abs(ref - float(g64[f"loss{it}"][0]))
            assert abs(out["loss"] - ref) <= max(1e-3 * abs(ref), noise), (it, out["loss"], ref)
            if f"logits{it}" in g:
                ref = g[f"logits{it}"]
                got = out["preds"].float().cpu().numpy()
                noise = 0.0 if it == 0 else 2 * np.abs(ref - g64[f"logits{it}"]).max()
                assert np.abs(got - ref).max() <= max(1e-3 * np.abs(ref).max(), noise), it


def _run(model_name, dtype, use_graph, steps=3, inject=None):
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(model_name, dtype=dtype, use_graph=use_graph)
    losses = []
    for it in range(steps):
        x, m = synth_batch(77 + it, 2, 64)
        losses.append(tr.step(x.cuda(), m.cuda())["loss"])
    params = torch.cat([p.detach().reshape(-1).float() for p in tr.module.parameters()]).cpu()
    return losses, params


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_graph_replay_and_checkpointing_are_bit_identical(dtype, amp_reset):
    """eager ≡ CUDA-graph replay and cp_wsgn_res50 ≡ wsgn_res50, three iterations, every parameter bit for bit"""
    with _exact():
        ref = _run("wsgn_res50", dtype, False)
        for name, graph in (("wsgn_res50", True), ("cp_wsgn_res50", False), ("cp_wsgn_res50", True)):
            got = _run(name, dtype, graph)
            assert got[0] == ref[0], (name, graph)
            assert torch.equal(got[1], ref[1]), (name, graph)
    assert all(np.isfinite(ref[0]))


def test_fp16_scaler_skips_and_recovers_on_a_ws_gradient_overflow(amp_reset, monkeypatch):
    """an inf written into one WS convolution's fp32 gradient (where the standardisation's backward puts it) makes the
    fused step skip and halve the scale; the next clean step trains"""
    from distributed_sod_project_b200 import amp, wsgn
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(dtype=torch.float16)
    conv = tr.module.div_16[2].conv2
    assert isinstance(conv, wsgn.FusedWSConv2d) and not hasattr(conv, "_sod_w16")
    orig = wsgn._WSFn.backward
    armed = {"on": False}

    def backward(ctx, g):
        out = orig(ctx, g)
        if armed["on"] and ctx.weight_ref is conv.weight:
            conv.weight.grad[3, 1, 0, 0] = float("inf")
        return out

    monkeypatch.setattr(wsgn._WSFn, "backward", staticmethod(backward))
    x, m = synth_batch(5, 2, 64)
    tr.step(x.cuda(), m.cuda())
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


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=str)
def test_wsgn_segments_and_shadow_set(dtype, amp_reset):
    """WS convolutions get no 16-bit shadow and no 16-bit gradient range; their weights sit in fp32 ranges"""
    from distributed_sod_project_b200.network.blocks import WSConv2d
    tr = _trainer(dtype=dtype)
    f = tr.optimizer.flat
    shadowed = {id(m.weight) for m in tr.module.modules() if hasattr(m, "_sod_w16")}
    ws = {id(m.weight) for m in tr.module.modules() if isinstance(m, WSConv2d)}
    assert len(ws) == 53 and not (ws & shadowed) and shadowed
    for p, off in f.slots:
        if id(p) in ws:
            bucket = next(i for i, (b, e) in enumerate(f.ranges) if b <= off < e)
            assert off >= f.splits[bucket]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16], ids=str)
def test_res50_iteration_is_unchanged(dtype, amp_reset, monkeypatch):
    """res50 through the WS-GN-aware Trainer: the same segment table, shadow set and launches per iteration as with the
    conversion switched off and every Conv2d counted as a 16-bit-gradient convolution"""
    import torch.nn as nn
    from distributed_sod_project_b200 import _lib, engine
    from distributed_sod_project_b200.synthetic import synth_batch

    def probe():
        tr = _trainer("res50", dtype=dtype)
        f = tr.optimizer.flat
        x, m = synth_batch(9, 2, 64)
        tr.step(x.cuda(), m.cuda())
        n0 = _lib.launches
        tr.step(x.cuda(), m.cuda())
        shadow = sorted(f.offset_of(mm.weight) for mm in tr.module.modules() if hasattr(mm, "_sod_w16"))
        conv = sorted(f.offset_of(mm.weight) for mm in tr.module.modules() if isinstance(mm, nn.Conv2d))
        return tr.optimizer._segment_plan(), shadow, conv, _lib.launches - n0, list(f.ranges), list(f.splits)

    plan, shadow, conv, launches, ranges, splits = probe()
    monkeypatch.setattr(engine, "convert_wsgn_model", lambda mdl: mdl)
    plan2, shadow2, _, launches2, ranges2, splits2 = probe()
    strip = lambda pl: [(b, e, part) for b, e, _, part in pl]  # noqa: E731
    assert strip(plan) == strip(plan2) and ranges == ranges2 and splits == splits2
    assert shadow == shadow2 and launches == launches2
    if dtype != torch.float32:
        assert shadow == conv          # every convolution of res50 keeps its shadow


# -- every parameter gradient of one iteration against float64 -------------------------------------------------------
def _loss(logits, mask, eps=1e-6):
    bce = F.binary_cross_entropy_with_logits(logits, mask)
    p = torch.sigmoid(logits)
    inter = p * mask
    return bce + ((p - inter).sum() + (mask - inter).sum()) / (p.sum() + mask.sum() + eps)


def _grads(dtype, engine_side: bool, scale: float):
    from distributed_sod_project_b200 import network, resample
    from distributed_sod_project_b200.network import blocks
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    from distributed_sod_project_b200.synthetic import synth_batch
    from distributed_sod_project_b200.utils import init_seed
    from distributed_sod_project_b200.wsgn import convert_wsgn_model
    x, m = synth_batch(1234, 4, 128)
    init_seed(0)
    model = network.wsgn_res50()
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    resample.ENABLED = blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = engine_side
    try:
        if dtype == torch.float64:
            model, x, m = model.double().cuda(), x.double().cuda(), m.double().cuda()
        else:
            model = model.cuda().to(memory_format=torch.channels_last)
            x, m = x.cuda().contiguous(memory_format=torch.channels_last), m.cuda()
            if engine_side:
                model = convert_wsgn_model(convert_syncbn_model(model))
        model.train()
        with torch.autocast("cuda", dtype=dtype, enabled=dtype in (torch.bfloat16, torch.float16)):
            preds = model(x)
        (_loss(preds.to(m.dtype), m) * scale).backward()
    finally:
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old
    return {n: p.grad.double() / scale for n, p in model.named_parameters()}


@pytest.mark.parametrize("dtype,A", [(torch.float32, 3.0), (torch.bfloat16, 2.5), (torch.float16, 2.5)], ids=str)
def test_iteration_gradients_match_fp64(dtype, A):
    """the A-rule of tests/test_gpu_model_grads.py on the e2 metric: for every parameter P,
    e(engine, P) ≤ A · (e(stock, P) + median_Q e(stock, Q)), e = ‖g − g64‖₂ / ‖g64‖₂, "stock" the torch WS-GN model
    (reference WS expression, nn.GroupNorm, nn.BatchNorm2d) in the same precision on the same GPU"""
    with _exact():
        ref = _grads(torch.float64, False, 1.0)
        scale = 1024.0 if dtype == torch.float16 else 1.0
        stock = _grads(dtype, False, scale)
        eng = _grads(dtype, True, scale)
    e = lambda g, n: float((g[n] - ref[n]).norm() / ref[n].norm().clamp_min(1e-300))  # noqa: E731
    es = {n: e(stock, n) for n in ref}
    med = float(np.median(list(es.values())))
    worst = max((e(eng, n) / (es[n] + med), n) for n in ref)
    assert worst[0] <= A, f"{worst[1]}: engine error {worst[0]:.2f}x (stock + median)"
