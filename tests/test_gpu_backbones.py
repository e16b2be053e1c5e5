"""The TestModel backbones of tests/_backbones.py on the engine: the reference's fp32 trajectories (one and two ranks),
every parameter gradient against float64, graph replay and activation checkpointing bit for bit, the command line, the
fp16 loss scaler and the flat buffer's fp32 ranges on the WS convolutions, and what is particular to one backbone:
VGG's 2×2 max-pool kernels, the grouped-convolution path of ResNeXt, and `res50`'s iteration left as it was."""
from __future__ import annotations

import socket

import numpy as np
import pytest
import torch
import torch.nn as nn

from distributed_sod_project_b200.network.blocks import WSConv2d
from _backbones import PLUGINS, _exact, _grads, _run, _trainer, _world2_entry, amp_reset  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu
NGPU = torch.cuda.device_count() if torch.cuda.is_available() else 0
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
ROW = pytest.mark.parametrize("row", PLUGINS, ids=lambda r: r.name)

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


@pytest.mark.parametrize("config", ["w1_s64", "w1_s128"])
@ROW
def test_fp32_trajectory_vs_reference(golden, row, config, amp_reset):  # noqa: F811
    """iteration 0: loss and logits within 1e-3 relative of the reference's fp32 run.  From the row's `noise_from`
    iteration on: within 1e-3, or within twice the reference's own fp32 distance from its float64 run where that is
    larger — one SGD step amplifies fp32 rounding in the reference itself (the `_fp64` vectors; 1.8e-2 on VGG's 128²
    logits, ~1e-2 on WS-GN ResNet-50's 64² loss and ~4e-2 on its 128² logits), which no fp32 run can beat"""
    from distributed_sod_project_b200.synthetic import synth_batch
    g = golden(f"step_{row.name}_{config}.npz")
    g64 = golden(f"step_{row.name}_{config}_fp64.npz")
    _, bs, size, _ = (int(v) for v in g["meta"])
    with _exact():
        tr = _trainer(row.name, dtype=torch.float32)
        assert [sum(map(pred, tr.model.modules())) for pred, _ in row.plugins] == [n for _, n in row.plugins]
        for it in range(2):
            x, m = synth_batch(1234 + 1000 * it, bs, size)
            out = tr.step(x.cuda(), m.cuda())
            ref = float(g[f"loss{it}"][0])
            noise = 0.0 if it < row.noise_from else 2 * abs(ref - float(g64[f"loss{it}"][0]))
            assert abs(out["loss"] - ref) <= max(1e-3 * abs(ref), noise), (it, out["loss"], ref)
            if f"logits{it}" in g:
                ref = g[f"logits{it}"]
                got = out["preds"].float().cpu().numpy()
                assert got.shape == ref.shape
                noise = 0.0 if it < row.noise_from else 2 * np.abs(ref - g64[f"logits{it}"]).max()
                assert np.abs(got - ref).max() <= max(1e-3 * np.abs(ref).max(), noise), it


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@ROW
def test_graph_replay_and_checkpointing_are_bit_identical(row, dtype, amp_reset):  # noqa: F811
    """eager ≡ CUDA-graph replay and cp_X ≡ X, three iterations, every parameter bit for bit"""
    with _exact():
        ref = _run(row.name, dtype, False)
        for name, graph in ((row.name, True), (row.cp, False), (row.cp, True)):
            got = _run(name, dtype, graph)
            assert got[0] == ref[0], (name, graph)
            assert torch.equal(got[1], ref[1]), (name, graph)
    assert all(np.isfinite(ref[0]))


@pytest.mark.parametrize("dtype,A", [(torch.float32, 3.0), (torch.bfloat16, 2.5), (torch.float16, 2.5)], ids=str)
@ROW
def test_iteration_gradients_match_fp64(row, dtype, A):
    """the A-rule of tests/test_gpu_model_grads.py (DESIGN §2): for every parameter P,
    e(engine, P) ≤ A · (e(stock, P) + median_Q e(stock, Q)), e = ‖g − g64‖₂ / ‖g64‖₂, "stock" the torch model
    (nn.BatchNorm2d, nn.MaxPool2d, the reference WS expression, nn.GroupNorm, cuDNN's grouped convolutions) in the same
    precision on the same GPU.  div_2's gradients are included: they are computed, as in the reference, though f3_trick
    leaves div_2 out of the optimizer"""
    with _exact():
        ref = _grads(row.name, torch.float64, False, 1.0)
        scale = 1024.0 if dtype == torch.float16 else 1.0
        stock = _grads(row.name, dtype, False, scale)
        eng = _grads(row.name, dtype, True, scale)
    assert ref.keys() == eng.keys() and row.frozen <= ref.keys()
    e = lambda g, n: float((g[n] - ref[n]).norm() / ref[n].norm().clamp_min(1e-300))  # noqa: E731
    es = {n: e(stock, n) for n in ref}
    med = float(np.median(list(es.values())))
    worst = max((e(eng, n) / (es[n] + med), n) for n in ref)
    assert worst[0] <= A, f"{worst[1]}: engine error {worst[0]:.2f}x (stock + median)"


@pytest.mark.skipif(NGPU < 2, reason="needs 2 GPUs")
@ROW
def test_training_step_world2_vs_reference(row):
    """the row at world 2 against the reference's two-rank fp32 trajectory (`_backbones._world2_steps`)"""
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_world2_entry, args=(2, port, row.name), nprocs=2, join=True)


@pytest.mark.parametrize("row", [r for r in PLUGINS if r.cli], ids=lambda r: r.name)
def test_train_and_test_cli(row):
    """train.py and test.py with "model" set to the row, in the row's scenario"""
    row.cli(row.name)


# -- the convolutions the optimizer keeps out of the 16-bit shadow ----------------------------------------------------
@pytest.mark.parametrize("model,path,fn,groups", [("wsgn_res50", "div_16.2.conv2", "_WSFn", 1),
                                                  ("wsgn_resnext50", "div_8.0.conv2", "_WSGroupConvFn", 32)],
                         ids=["ws", "grouped"])
def test_fp16_scaler_skips_and_recovers_on_a_ws_conv_overflow(model, path, fn, groups, amp_reset,  # noqa: F811
                                                              monkeypatch):
    """an inf written into one WS convolution's fp32 gradient — where the standardisation's backward puts it, or the
    grouped convolution's wgrad kernel on csrc/gconv.cu — makes the fused step skip and halve the scale; the next clean
    step trains"""
    from distributed_sod_project_b200 import amp, wsgn
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(model, dtype=torch.float16)
    conv = tr.module.get_submodule(path)
    assert isinstance(conv, wsgn.FusedWSConv2d) and conv.groups == groups and not hasattr(conv, "_sod_w16")
    assert wsgn.grouped_conv_on_kernels(conv) == (groups > 1)
    autograd_fn = getattr(wsgn, fn)
    orig = autograd_fn.backward
    armed = {"on": False}

    def backward(ctx, g):
        out = orig(ctx, g)
        if armed["on"] and ctx.weight_ref is conv.weight:
            conv.weight.grad[3, 1, 0, 0] = float("inf")
        return out

    monkeypatch.setattr(autograd_fn, "backward", staticmethod(backward))
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


@pytest.mark.parametrize("model,grouped,count", [("wsgn_res50", False, 53), ("wsgn_resnext50", True, 16)],
                         ids=["ws", "grouped"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=str)
def test_ws_convs_get_no_shadow_and_fp32_gradient_ranges(model, grouped, count, dtype, amp_reset):  # noqa: F811
    """WS convolutions (all of them, or the grouped ones) get no 16-bit shadow and no 16-bit gradient range; their
    weights sit in fp32 ranges"""
    tr = _trainer(model, dtype=dtype)
    f = tr.optimizer.flat
    shadowed = {id(m.weight) for m in tr.module.modules() if hasattr(m, "_sod_w16")}
    ws = {id(m.weight) for m in tr.module.modules() if isinstance(m, WSConv2d) and (m.groups > 1 or not grouped)}
    assert len(ws) == count and not (ws & shadowed) and shadowed
    for p, off in f.slots:
        if id(p) in ws:
            bucket = next(i for i, (b, e) in enumerate(f.ranges) if b <= off < e)
            assert off >= f.splits[bucket]


# -- res50 -------------------------------------------------------------------------------------------------------------
def _res50_probe(dtype):
    """res50's second iteration at bs 2, 64²: the pinned quantities of RES50, then the shadowed and all convolutions'
    flat offsets, the flat buffer's ranges and splits"""
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer("res50", dtype=dtype)
    f = tr.optimizer.flat
    x, m = synth_batch(9, 2, 64)
    tr.step(x.cuda(), m.cuda())
    n0 = _lib.launches
    tr.step(x.cuda(), m.cuda())
    groups = [id(g) for g in tr.optimizer.param_groups]
    plan = [(b, e, None if g is None else groups.index(id(g)), bool(f)) for b, e, g, f in tr.optimizer._segment_plan()]
    shadow = sorted(f.offset_of(mm.weight) for mm in tr.module.modules() if hasattr(mm, "_sod_w16"))
    conv = sorted(f.offset_of(mm.weight) for mm in tr.module.modules() if isinstance(mm, nn.Conv2d))
    pinned = {"launches": _lib.launches - n0, "shadows": len(shadow), "plan": plan}
    return pinned, shadow, conv, list(f.ranges), list(f.splits)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_res50_iteration_is_unchanged(dtype, amp_reset, monkeypatch):  # noqa: F811
    """res50 never reaches the 2×2 max-pool kernels; its launches per iteration, shadow count and segment table are the
    pinned ones; with the WS-GN conversion switched off it has the same segment table, flat ranges and splits, shadow
    offsets and launches; in 16 bit every convolution keeps its shadow"""
    from distributed_sod_project_b200 import engine, resample
    monkeypatch.setattr(resample, "maxpool2x2s2", lambda x: pytest.fail("res50 reached the 2x2 max-pool"))
    pinned, shadow, conv, ranges, splits = _res50_probe(dtype)
    assert pinned == RES50[str(dtype)]
    monkeypatch.setattr(engine, "convert_wsgn_model", lambda mdl: mdl)
    pinned2, shadow2, _, ranges2, splits2 = _res50_probe(dtype)
    assert pinned2 == pinned and shadow2 == shadow and ranges2 == ranges and splits2 == splits
    if dtype != torch.float32:
        assert shadow == conv


# -- vgg16: the 2×2 max-pool kernels -----------------------------------------------------------------------------------
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


# -- wsgn_resnext50: the grouped-convolution path ----------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=str)
def test_wsgn_res50_never_takes_the_grouped_path(dtype, amp_reset, monkeypatch):  # noqa: F811
    """wsgn_res50 never calls the grouped-convolution path; wsgn_resnext50 calls it once per forward (layer2.0)"""
    from distributed_sod_project_b200 import _lib, wsgn
    from distributed_sod_project_b200.synthetic import synth_batch
    calls = []
    orig = wsgn._WSGroupConvFn.forward

    def fwd(ctx, *a):
        calls.append(1)
        return orig(ctx, *a)

    def probe():
        tr = _trainer("wsgn_res50", dtype=dtype)
        x, m = synth_batch(9, 2, 64)
        tr.step(x.cuda(), m.cuda())
        n0 = _lib.launches
        tr.step(x.cuda(), m.cuda())
        return _lib.launches - n0

    monkeypatch.setattr(wsgn._WSGroupConvFn, "forward", staticmethod(fwd))
    launches = probe()
    assert not calls
    tr = _trainer("wsgn_resnext50", dtype=dtype)
    x, m = synth_batch(9, 2, 64)
    tr.step(x.cuda(), m.cuda())
    assert len(calls) == 1
    assert launches > 0
