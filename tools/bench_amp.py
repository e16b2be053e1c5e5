#!/usr/bin/env python
"""What fp16 amp (apex O1 with the device-resident loss scaler) costs next to bf16.  Prints one JSON line.

    python tools/bench_amp.py [--steps 200] [--train-steps 30] [--warmup 5] [--repeats 2]

In one run, on the current GPU (its name and power limit are part of the output):
* `train_img_s`: img/s of the training iteration at 320², batch 16, res50, optim f3_trick — fp16 on CUDA graphs with the
  fp16 shadow weights; fp16 eager without shadow weights (the path fp16 took before the device scaler: no graph, no
  shadow, one host sync per step); bf16 on CUDA graphs.  The configurations run interleaved, `--repeats` times each.
* `step_tail_us`: the optimizer tail of one fp16 iteration — clear the flag, checked gather of the stolen fp16 weight
  gradients, the range check, `sod_sgd_momentum_scaler` — captured in a CUDA graph and replayed, for the res50 model
  (24.9 M parameters); next to it the same tail in bf16 (gather + `sod_sgd_momentum`), the step `bench.py` runs.
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


def _reset_amp():
    from distributed_sod_project_b200 import amp
    amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None, dev=None)


def step_tail_us(dtype: torch.dtype, steps: int) -> dict:
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    _reset_amp()
    tr = Trainer(model_name="res50", dtype=dtype, channels_last=True, report_items=False)
    opt = tr.optimizer
    x, m = synth_batch(1, 2, 64)
    tr.forward_backward_update(x.cuda(), m.cuda())
    # leave the stolen 16-bit weight gradients of one more backward in place: every replay gathers them and steps
    opt.zero_grad()
    tr.model(x.cuda().contiguous(memory_format=torch.channels_last)).float().mean().backward()
    opt._scaler_readback = None                       # the tail alone: no host read-back while warming up
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
    _reset_amp()
    return {"us": round(ms * 1e3, 1), "numel": opt.flat.numel}


def train_img_s(dtype: torch.dtype, graph: bool, shadow: bool, steps: int, warmup: int) -> float:
    from distributed_sod_project_b200 import engine
    from distributed_sod_project_b200.synthetic import synth_batch
    _reset_amp()
    tr = engine.Trainer(model_name="res50", lr=0.05, dtype=dtype, channels_last=True, report_items=False, use_graph=graph,
                        shadow_weights=shadow)
    assert tr.use_graph == graph
    bs = 16
    batches = [tuple(t.cuda() for t in synth_batch(1234 + i, bs, 320)) for i in range(4)]
    for i in range(warmup):
        tr.forward_backward_update(*batches[i % 4])
    torch.cuda.synchronize()
    it = iter(range(10 ** 9))
    ms = _time_ms(lambda: tr.forward_backward_update(*batches[next(it) % 4]), steps)
    _reset_amp()
    return round(bs / (ms * 1e-3), 1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=200, help="replays of the step tail")
    ap.add_argument("--train-steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    out = {"gpu": gpu_info(torch.cuda.current_device())}
    out["step_tail_us"] = {"fp16_scaler": step_tail_us(torch.float16, args.steps),
                           "bf16": step_tail_us(torch.bfloat16, args.steps)}
    configs = {"fp16_graph": (torch.float16, True, True), "fp16_eager_no_shadow": (torch.float16, False, False),
               "bf16_graph": (torch.bfloat16, True, True)}
    runs = {k: [] for k in configs}
    for _ in range(args.repeats):
        for k, (dt, graph, shadow) in configs.items():
            runs[k].append(train_img_s(dt, graph, shadow, args.train_steps, args.warmup))
    out["train_img_s"] = {"bs": 16, "size": 320, "model": "res50", **runs}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
