#!/usr/bin/env python
"""Measure `aim_res50` (ResNet-50 + MINet's LightAIM neck + the TestModel decoder) on the GPU; one JSON line on stdout.

    python tools/bench_aim.py [--steps K --warmup W]

On the bench workload (320×320, bs 16, bf16):
* `engine_img_s`: the engine's iteration (nearest ×2 and 2×2 average-pool kernels, SyncBN kernels with the neck's conv
  biases folded in, fused loss and SGD), replayed from a CUDA graph, batch resident in HBM; `engine_peak_gib` its peak
  allocation;
* `stock_img_s`: the same model in stock PyTorch (nn.BatchNorm2d, F.interpolate, nn.AvgPool2d, channels-last, bf16
  autocast, torch.optim.SGD) run eagerly, before the engine leg and with the engine's resampling seams off;
  `stock_peak_gib` its peak allocation;
* `autocast_nearest_dtype`: the dtype `F.interpolate(mode="nearest")` returns for a bf16 input under CUDA bf16 autocast
  (an fp32 result means autocast runs nearest in fp32, as it does bilinear);
* `nearest`: per distinct up-sample shape of the neck (with how many of the twelve per forward have it), forward and
  backward µs of the csrc/nearest.cu entries and of torch's `upsample_nearest2d` under bf16 autocast, each device time
  from a CUDA graph of back-to-back calls, with the bytes the kernels have to move and their GB/s.  The torch legs
  include whatever casts autocast inserts.
The card's name and power limit are part of the line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_vgg import _peak  # noqa: E402
from bench_wsgn import BS, SIZE, card, engine_img_s, graph_us, stock_img_s  # noqa: E402

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

# (channels, input side, count) of the neck's nearest ×2 up-samples at a 320×320 input
NEAREST_SHAPES = ((64, SIZE // 4, 3), (64, SIZE // 8, 3), (64, SIZE // 16, 3), (64, SIZE // 32, 2), (1024, SIZE // 32, 1))


def stock_aim_img_s(steps: int, warmup: int) -> float:
    """the stock leg with the engine's resampling seams off (a `Trainer` built earlier in this process turns them on)"""
    from distributed_sod_project_b200 import _lib, resample
    from distributed_sod_project_b200.network import blocks
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    resample.ENABLED = blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = False
    try:
        n0 = _lib.launches
        r = stock_img_s(steps, warmup, "aim_res50")
        if _lib.launches != n0:
            raise RuntimeError(f"the stock leg launched {_lib.launches - n0} of this repo's kernels")
        return r
    finally:
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old


def autocast_nearest_dtype() -> str:
    x = torch.zeros(1, 8, 2, 2, device="cuda", dtype=torch.bfloat16)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        return str(F.interpolate(x, scale_factor=2, mode="nearest").dtype)


def nearest_layers() -> list[dict]:
    from distributed_sod_project_b200 import _lib
    lib, code, es = _lib.lib(), _lib.dtype_code(torch.bfloat16), 2
    rows = []
    for c, s, count in NEAREST_SHAPES:
        x = torch.randn(BS, c, s, s, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        y = torch.empty(BS, c, 2 * s, 2 * s, device="cuda", dtype=torch.bfloat16, memory_format=torch.channels_last)
        dy = torch.randn_like(y)
        dx = torch.empty_like(x)

        def k_fwd():
            _lib.check(lib.sod_upsample2x_nearest_fwd(x.data_ptr(), y.data_ptr(), BS, s, s, c, code, _lib.stream_ptr()),
                       "sod_upsample2x_nearest_fwd")

        def k_bwd():
            _lib.check(lib.sod_upsample2x_nearest_bwd(dy.data_ptr(), dx.data_ptr(), BS, s, s, c, code, _lib.stream_ptr()),
                       "sod_upsample2x_nearest_bwd")

        with torch.autocast("cuda", dtype=torch.bfloat16):
            ydt = F.interpolate(x, scale_factor=2, mode="nearest").dtype

        def t_fwd():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                F.interpolate(x, scale_factor=2, mode="nearest")

        def t_bwd():
            # what autograd runs for the op above: the incoming bf16 gradient in the output's dtype, the backward, and
            # the result back in the input's dtype (both casts are no-ops when autocast keeps nearest in bf16)
            g = torch.ops.aten.upsample_nearest2d_backward(dy.to(ydt), [2 * s, 2 * s], [BS, c, s, s], None, None)
            g.to(torch.bfloat16)

        nbytes = 5 * x.numel() * es                      # read x / write 4x (forward), read 4x / write x (backward)
        row = {"shape": [BS, c, s, s], "count": count, "MB": round(nbytes / 1e6, 2)}
        for name, fn in (("kernel_fwd", k_fwd), ("kernel_bwd", k_bwd), ("torch_fwd", t_fwd), ("torch_bwd", t_bwd)):
            us = graph_us(fn)
            row[f"{name}_us"] = round(us, 2)
            if name.startswith("kernel"):
                row[f"{name}_GBps"] = round(nbytes / (us * 1e-6) / 1e9, 1)
        rows.append(row)
        del x, y, dy, dx
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_aim.py measures on a GPU; none is visible")
    stock, stock_peak = _peak(stock_aim_img_s, a.steps, a.warmup)
    eng, eng_peak = _peak(engine_img_s, a.steps, a.warmup, "aim_res50")
    out = {"card": card(), "model": "aim_res50", "size": SIZE, "bs": BS, "dtype": "bf16",
           "engine_img_s": round(eng, 1), "engine_peak_gib": round(eng_peak, 2),
           "stock_img_s": round(stock, 1), "stock_peak_gib": round(stock_peak, 2),
           "autocast_nearest_dtype": autocast_nearest_dtype(), "nearest": nearest_layers()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
