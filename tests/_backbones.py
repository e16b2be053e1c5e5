"""The reference's TestModel backbones as one table, and the helpers the backbone tests share
(tests/test_backbones_cpu.py, tests/test_gpu_backbones.py).  Not a test module: pytest does not collect it.

A row carries only what differs between backbones.  Each row's golden vectors are `model_<name>_init.npz` and
`step_<name>_{w1_s64,w1_s128,w2_s64}[_fp64].npz`, written by `tools/make_golden_backbones.py <name>`."""
from __future__ import annotations

import contextlib
import json
import os
import subprocess
import sys
from dataclasses import dataclass
from typing import Callable

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from distributed_sod_project_b200 import wsgn
from distributed_sod_project_b200.network import blocks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


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


def _trainer(model_name, **kw):
    from distributed_sod_project_b200.engine import Trainer
    return Trainer(model_name=model_name, lr=0.05, momentum=0.9, weight_decay=5e-4, **kw)


def _loss(logits, mask, eps=1e-6):
    """the reference's BCE + CEL in plain torch"""
    bce = F.binary_cross_entropy_with_logits(logits, mask)
    p = torch.sigmoid(logits)
    inter = p * mask
    return bce + ((p - inter).sum() + (mask - inter).sum()) / (p.sum() + mask.sum() + eps)


def _run(model_name, dtype, use_graph, steps=3):
    """`steps` iterations of the engine at bs 2, 64²: the losses and every parameter after the last step"""
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(model_name, dtype=dtype, use_graph=use_graph)
    losses = []
    for it in range(steps):
        x, m = synth_batch(77 + it, 2, 64)
        losses.append(tr.step(x.cuda(), m.cuda())["loss"])
    params = torch.cat([p.detach().reshape(-1).float() for p in tr.module.parameters()]).cpu()
    return losses, params


def _grads(model_name, dtype, engine_side: bool, scale: float):
    """every parameter gradient of one training-mode iteration (bs 4, 128²) of the plugin: on the engine's seams
    (`Trainer`'s SyncBN and WS-GN conversions, identities where the backbone has nothing to convert) or as the stock
    torch model, in `dtype` (float64: the stock model in double)"""
    from distributed_sod_project_b200 import network, resample
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    from distributed_sod_project_b200.synthetic import synth_batch
    from distributed_sod_project_b200.utils import init_seed
    x, m = synth_batch(1234, 4, 128)
    init_seed(0)
    model = getattr(network, model_name)()
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    resample.ENABLED = blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = engine_side
    try:
        if dtype == torch.float64:
            model, x, m = model.double().cuda(), x.double().cuda(), m.double().cuda()
        else:
            model = model.cuda().to(memory_format=torch.channels_last)
            x, m = x.cuda().contiguous(memory_format=torch.channels_last), m.cuda()
            if engine_side:
                model = wsgn.convert_wsgn_model(convert_syncbn_model(model))
        model.train()
        with torch.autocast("cuda", dtype=dtype, enabled=dtype in (torch.bfloat16, torch.float16)):
            preds = model(x)
        (_loss(preds.to(m.dtype), m) * scale).backward()
    finally:
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old
    return {n: p.grad.double() / scale for n, p in model.named_parameters()}


# -- two ranks ---------------------------------------------------------------------------------------------------------
def _world2_entry(rank, world, port, name):
    """`torch.multiprocessing.spawn` target: one rank of the two-rank check of row `name`"""
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        _world2_steps(rank, ROWS[name])
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _world2_steps(rank, row):
    """two fp32 iterations against the reference's two-rank trajectory (the concatenated-batch construction of
    tools/make_golden.py): iteration 0 within 1e-3; iteration 1 within 1e-3, or twice the reference's own fp32
    distance from its float64 run where that is larger.  Every rank holds the same parameters after each fused step"""
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.loss import get_total_loss
    from distributed_sod_project_b200.synthetic import synth_batch
    g = np.load(os.path.join(GOLDEN, f"step_{row.name}_w2_s64.npz"))
    g64 = np.load(os.path.join(GOLDEN, f"step_{row.name}_w2_s64_fp64.npz"))
    _, bs, size, _ = (int(v) for v in g["meta"])
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    tr = Trainer(model_name=row.name, dtype=torch.float32, channels_last=True)
    for it in range(2):
        x, m = synth_batch(1234 + rank + 1000 * it, bs, size)
        preds = tr.model(x.cuda().contiguous(memory_format=torch.channels_last))
        loss, _ = get_total_loss(preds, m.cuda(), tr.loss_funcs, unit_upstream=True)
        tr.optimizer.zero_grad(); loss.backward(); tr.optimizer.step()
        want = float(g[f"loss{it}"][rank])
        tol = 1e-3 * abs(want) if it == 0 else max(1e-3 * abs(want), 2 * abs(want - float(g64[f"loss{it}"][rank])))
        assert abs(float(loss) - want) <= tol, (rank, it, float(loss), want)
        if it == 0 and row.world2_logits0:
            ref_l = g["logits0"][rank * bs:(rank + 1) * bs]
            got = preds.detach().float().cpu().numpy()
            assert np.abs(got - ref_l).max() / np.abs(ref_l).max() < 1e-3
        flat = tr.optimizer.flat.param
        other = flat.clone(); torch.distributed.broadcast(other, 0)
        assert torch.equal(flat, other)
    tr.model.arena.check_error()


# -- command line ------------------------------------------------------------------------------------------------------
def _script(script, cfg, *args, timeout):
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
    out = subprocess.run([sys.executable, os.path.join(ROOT, script), *args], cwd=ROOT, env=env, capture_output=True,
                         text=True, timeout=timeout)
    assert out.returncode == 0, out.stderr[-3000:]
    return out.stdout


def _train_resume_and_test(name):
    """train.py on CUDA graphs: 2 epochs with validation and a checkpoint each; the checkpoint, marked as written
    after epoch 1 (a run stopped there), resumed with resume_mode "train", which trains epoch 2 only; then test.py on
    the saved weights"""
    import glob
    common = {"epoch_num": 2, "synthetic_iters_per_epoch": 2, "batch_size": 4, "print_freq": 1, "save_freq": 1,
              "is_distributed": False, "input_size": 96, "model": name, "synthetic_eval_images": 5, "val_freq": 1,
              "final_test": False, "cuda_graph": True}
    out = _script("train.py", common, "-ng", "1", "-p", "29713", timeout=600)
    assert "End Training" in out and out.count("[I:") == 4 and out.count("'MAE':") == 2
    saved = glob.glob(os.path.join(ROOT, "output*", f"{name}_SIZE96_BS4_*_E2_*", "pth", "checkpoint_final.pth.tar"))
    assert len(saved) == 1, saved
    ck = torch.load(saved[0], map_location="cpu", weights_only=False)
    assert ck["epoch"] == 2
    ck["epoch"] = 1
    torch.save(ck, saved[0])
    out = _script("train.py", dict(common, resume_mode="train"), "-ng", "1", "-p", "29714", timeout=600)
    assert "End Training" in out and out.count("[I:") == 2 and "[E:1:2]" in out and "[E:0:" not in out
    out = _script("test.py", dict(common, resume_mode="test"), timeout=600)
    assert out.count("'MAE':") == 6


def _train_and_test(name):
    """one train.py epoch and one test.py evaluation of the saved checkpoint, written under output_resnext"""
    common = {"epoch_num": 1, "synthetic_iters_per_epoch": 2, "batch_size": 4, "print_freq": 1, "save_freq": 1,
              "is_distributed": False, "input_size": 96, "model": name, "output_name": "output_resnext",
              "synthetic_eval_images": 5, "val_freq": 1, "final_test": False}
    out = _script("train.py", common, "-ng", "1", "-p", "29711", timeout=500)
    assert "End Training" in out and out.count("[I:") == 2
    out = _script("test.py", dict(common, resume_mode="test"), timeout=500)
    assert out.count("'MAE':") == 6


# -- the table ---------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Backbone:
    name: str                    # the model plugin; its golden vectors carry the same name
    frozen: frozenset            # the div_2 parameters f3_trick leaves out of the optimizer
    plugins: tuple               # (predicate, count): the engine's modules the trainer's model must hold
    noise_from: int = 1          # first iteration whose trajectory allowance includes the reference's fp32 noise
    world2_logits0: bool = False  # the two-rank check also compares iteration 0's logits
    cli: Callable | None = None  # the train.py / test.py scenario run on this backbone

    @property
    def cp(self):
        return f"cp_{self.name}"


_WSGN_FROZEN = frozenset({"div_2.0.weight", "div_2.1.weight", "div_2.1.bias"})

PLUGINS = [
    Backbone("vgg16", frozenset(f"div_2.{i}.{k}" for i in (0, 1, 3, 4) for k in ("weight", "bias")),
             plugins=((lambda m: isinstance(m, blocks._VGGPool), 4),), cli=_train_resume_and_test),
    Backbone("wsgn_res50", _WSGN_FROZEN,
             plugins=((lambda m: isinstance(m, wsgn.GroupNorm32), 53),
                      (lambda m: isinstance(m, wsgn.FusedWSConv2d), 53)),
             world2_logits0=True),
    # the reference's own 64² fp32 logits are already 1.1e-3 (relative) from its float64 ones before any step
    Backbone("wsgn_resnext50", _WSGN_FROZEN,
             plugins=((lambda m: isinstance(m, wsgn.FusedWSConv2d) and m.groups > 1, 16),), noise_from=0,
             cli=_train_and_test),
]
ROWS = {r.name: r for r in PLUGINS}
