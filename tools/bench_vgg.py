#!/usr/bin/env python
"""Measure `vgg16` (VGG16-BN backbone) on the GPU; one JSON line on stdout.

    python tools/bench_vgg.py [--steps K --warmup W]

On the bench workload (320×320, bs 16, bf16):
* `engine_img_s`: the engine's iteration (2×2 max-pool kernels, SyncBN kernels with the 13 backbone conv biases folded
  in, fused loss and SGD), replayed from a CUDA graph, batch resident in HBM; `engine_peak_gib` its peak allocation;
* `stock_img_s`: the same model in stock PyTorch — nn.MaxPool2d (torch's kernel, with its int64 indices),
  nn.BatchNorm2d, F.interpolate, nn.AvgPool2d, channels-last, bf16 autocast, torch.optim.SGD — run eagerly, before the
  engine leg and with the engine's resampling seams off; `stock_peak_gib` its peak allocation;
* `pools`: per pool of the backbone, forward and backward µs of the csrc/maxpool.cu entries and of torch's operators
  (`aten.max_pool2d_with_indices` and its backward, what nn.MaxPool2d runs) on the same channels-last bf16 tensors,
  each device time from a CUDA graph of back-to-back calls, with the bytes the algorithm has to move and the achieved
  GB/s.  The kernels read x and write y and one byte of window position per output forward, and read dy and that byte
  and write dx backward; torch does the same with an int64 index per output.
The card's name and power limit are part of the line.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_wsgn import BS, SIZE, card, engine_img_s, graph_us, stock_img_s  # noqa: E402

import torch  # noqa: E402

# (channels, input side) of the four 2×2 pools of VGG16-BN at a 320×320 input
POOL_SHAPES = ((64, SIZE), (128, SIZE // 2), (256, SIZE // 4), (512, SIZE // 8))


def _peak(fn, *a):
    gc.collect()                         # a previous leg's graphs, arena and workspaces must not count toward this peak
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    r = fn(*a)
    torch.cuda.synchronize()
    return r, torch.cuda.max_memory_allocated() / 2 ** 30


def stock_vgg_img_s(steps: int, warmup: int) -> float:
    """the stock leg with the engine's resampling seams switched off: a `Trainer` built earlier in this process sets
    `resample.ENABLED` and `blocks.INTERPOLATE_IN_ACTIVATION_DTYPE`, and the model's pools, up-samples and average
    pools would then take this repo's kernels"""
    from distributed_sod_project_b200 import _lib, resample
    from distributed_sod_project_b200.network import blocks
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    resample.ENABLED = blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = False
    try:
        n0 = _lib.launches
        r = stock_img_s(steps, warmup, "vgg16")
        if _lib.launches != n0:
            raise RuntimeError(f"the stock leg launched {_lib.launches - n0} of this repo's kernels")
        return r
    finally:
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old


def pool_layers() -> list[dict]:
    from distributed_sod_project_b200 import _lib
    lib, code, es = _lib.lib(), _lib.dtype_code(torch.bfloat16), 2
    rows = []
    for c, s in POOL_SHAPES:
        x = torch.randn(BS, c, s, s, device="cuda").clamp_min(0).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.empty(BS, c, s // 2, s // 2, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        arg = torch.empty(y.numel(), dtype=torch.uint8, device="cuda")
        dy = torch.randn_like(y)
        dx = torch.empty_like(x)

        def k_fwd():
            _lib.check(lib.sod_maxpool2x2s2_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), BS, s, s, c, code,
                                                _lib.stream_ptr()), "sod_maxpool2x2s2_fwd")

        def k_bwd():
            _lib.check(lib.sod_maxpool2x2s2_bwd(dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), BS, s, s, c, code,
                                                _lib.stream_ptr()), "sod_maxpool2x2s2_bwd")

        ty, idx = torch.ops.aten.max_pool2d_with_indices(x, [2, 2], [2, 2], [0, 0], [1, 1], False)
        t_fwd = lambda: torch.ops.aten.max_pool2d_with_indices(x, [2, 2], [2, 2], [0, 0], [1, 1], False)  # noqa: E731
        t_bwd = lambda: torch.ops.aten.max_pool2d_with_indices_backward(dy, x, [2, 2], [2, 2], [0, 0], [1, 1], False, idx)  # noqa: E731
        nx, ny = x.numel(), y.numel()
        bytes_ = {"kernel_fwd": (nx + ny) * es + ny, "kernel_bwd": (ny + nx) * es + ny,
                  "torch_fwd": (nx + ny) * es + 8 * ny, "torch_bwd": (ny + nx) * es + 8 * ny}
        row = {"shape": [BS, c, s, s]}
        for name, fn in (("kernel_fwd", k_fwd), ("kernel_bwd", k_bwd), ("torch_fwd", t_fwd), ("torch_bwd", t_bwd)):
            us = graph_us(fn)
            row[f"{name}_us"] = round(us, 2)
            row[f"{name}_MB"] = round(bytes_[name] / 1e6, 2)
            row[f"{name}_GBps"] = round(bytes_[name] / (us * 1e-6) / 1e9, 1)
        rows.append(row)
        del x, y, arg, dy, dx, ty, idx
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vgg.py measures on a GPU; none is visible")
    stock, stock_peak = _peak(stock_vgg_img_s, a.steps, a.warmup)
    eng, eng_peak = _peak(engine_img_s, a.steps, a.warmup, "vgg16")
    out = {"card": card(), "model": "vgg16", "size": SIZE, "bs": BS, "dtype": "bf16",
           "engine_img_s": round(eng, 1), "engine_peak_gib": round(eng_peak, 2),
           "stock_img_s": round(stock, 1), "stock_peak_gib": round(stock_peak, 2), "pools": pool_layers()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
