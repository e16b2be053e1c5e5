#!/usr/bin/env python
"""Cost of the fused Adam step, and what optim "adam" does to training throughput.  Prints one JSON line.

    python tools/bench_optim.py [--steps 200] [--train-steps 30] [--warmup 5]

In one run, on the current GPU:
* `fused_adam_step`: the optimizer step of the res50 model (24.9 M parameters, bf16 amp with shadow weights) — the bf16
  weight-gradient gather plus `sod_adam` — captured in a CUDA graph and replayed; µs per step and GB/s of algorithmic
  bytes (each buffer the step must read or write counted once, see `_adam_bytes`);
* `torch_fused_adam_step`: `torch.optim.Adam(fused=True)` over the same number of parameters as one flat fp32 tensor;
* `train_img_s`: img/s of the captured training iteration at 320², batch 16, bf16 for optim "adam", optim "f3_trick",
  and optim "adam" with `make_optimizer` swapped back to `torch.optim.Adam` (what "adam" built before `FusedAdam`: no
  graph, no shadow weights).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import gpu_info  # noqa: E402


def _time_ms(fn, steps: int) -> float:
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def _adam_bytes(opt) -> int:
    """GRAD16 ranges: read g16, p, m, v; write p, m, v, shadow; clear g16 → 2+12+12+2+2 = 30 B/elem.  Other ranges
    also read and clear the fp32 gradient: 38 B/elem.  Plus the gather: 2 B read + 2 B written per gathered element."""
    total = 0
    for b, e, g, bf16_part in opt._segment_plan():
        if g is not None:
            total += (e - b) * (30 if bf16_part else 38)
    gathered = sum(leaf.numel() for leaf, _, steal in opt.flat.shadow_leaves if steal)
    return total + 4 * gathered


def fused_adam_step(steps: int) -> dict:
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = Trainer(model_name="res50", lr=1e-4, optim="adam", dtype=torch.bfloat16, channels_last=True, report_items=False)
    opt = tr.optimizer
    x, m = synth_batch(1, 2, 64)
    tr.forward_backward_update(x.cuda(), m.cuda())
    # leave the stolen bf16 weight gradients of one more backward in place: every replay gathers them and steps
    tr.optimizer.zero_grad()
    tr.model(x.cuda().contiguous(memory_format=torch.channels_last)).float().mean().backward()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        opt.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    for _ in range(10):
        graph.replay()
    ms = _time_ms(graph.replay, steps)
    nbytes = _adam_bytes(opt)
    return {"us": round(ms * 1e3, 1), "algorithmic_bytes": nbytes, "gbs": round(nbytes / (ms * 1e-3) / 1e9, 1),
            "numel": opt.flat.numel}


def torch_fused_adam_step(numel: int, steps: int) -> dict:
    p = torch.nn.Parameter(torch.randn(numel, device="cuda"))
    p.grad = torch.randn(numel, device="cuda")
    opt = torch.optim.Adam([p], lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=5e-4, fused=True)
    for _ in range(10):
        opt.step()
    ms = _time_ms(opt.step, steps)
    nbytes = numel * 4 * 7                                   # read g, p, m, v; write p, m, v
    return {"us": round(ms * 1e3, 1), "algorithmic_bytes": nbytes, "gbs": round(nbytes / (ms * 1e-3) / 1e9, 1)}


def train_img_s(optim: str, steps: int, warmup: int, torch_adam: bool = False) -> float:
    from distributed_sod_project_b200 import engine, optim as optim_mod
    from distributed_sod_project_b200.synthetic import synth_batch
    saved = engine.make_optimizer
    if torch_adam:
        def make(model, kind, info):
            if kind != "adam":
                return saved(model, kind, info)
            return torch.optim.Adam(model.parameters(), lr=info["lr"], betas=(0.9, 0.999), eps=1e-8,
                                    weight_decay=info["weight_decay"])
        engine.make_optimizer = make
    try:
        lr = 1e-4 if optim == "adam" else 0.05
        tr = engine.Trainer(model_name="res50", lr=lr, optim=optim, dtype=torch.bfloat16, channels_last=True,
                            report_items=False, use_graph=True)
    finally:
        engine.make_optimizer = saved
    bs = 16
    batches = [tuple(t.cuda() for t in synth_batch(1234 + i, bs, 320)) for i in range(4)]
    for i in range(warmup):
        tr.forward_backward_update(*batches[i % 4])
    torch.cuda.synchronize()
    it = iter(range(10 ** 9))
    ms = _time_ms(lambda: tr.forward_backward_update(*batches[next(it) % 4]), steps)
    assert isinstance(tr.optimizer, optim_mod.FusedOptimizer) != torch_adam
    return round(bs / (ms * 1e-3), 1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=200, help="replays of the optimizer step")
    ap.add_argument("--train-steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    out = {"gpu": gpu_info(torch.cuda.current_device())}
    out["fused_adam_step"] = fused_adam_step(args.steps)
    out["torch_fused_adam_step"] = torch_fused_adam_step(out["fused_adam_step"]["numel"], args.steps)
    out["train_img_s"] = {"bs": 16, "size": 320, "dtype": "bf16",
                          "adam": train_img_s("adam", args.train_steps, args.warmup),
                          "f3_trick": train_img_s("f3_trick", args.train_steps, args.warmup),
                          "adam_torch_optim_before": train_img_s("adam", args.train_steps, args.warmup, torch_adam=True)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
