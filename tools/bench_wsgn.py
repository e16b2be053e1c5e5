#!/usr/bin/env python
"""Measure the WS-GN backbone on the GPU; one JSON line on stdout.

    python tools/bench_wsgn.py [--model wsgn_res50 | wsgn_resnext50] [--steps K --warmup W]

On the bench workload (320×320, bs 16, bf16), `--model wsgn_res50` (the default):
* `wsgn_res50`: images/s of the engine's iteration (GroupNorm / WS kernels, SyncBN decoder, fused loss and SGD),
  replayed from a CUDA graph, batch resident in HBM;
* `stock`: the same model in stock PyTorch — the reference's WS expression, nn.GroupNorm, nn.BatchNorm2d, channels-last,
  bf16 autocast, torch.optim.SGD — run eagerly;
* `groupnorm`: per layer shape of the backbone, forward (with ReLU) and backward µs of the kernels (their C entries)
  and of torch's GroupNorm operators (`aten.native_group_norm` and its backward, what torch.nn.functional.group_norm
  runs, with the NCHW copies of x and dy those need) on the same channels-last bf16 tensors, each timed as device time from a CUDA graph of back-to-back calls, with
  algorithmic GB/s (bytes the algorithm has to move: the kernels read x and write y forward, read dy, x, y and write dx
  backward; torch reads x, writes y forward and reads dy, x and writes dx backward);
* `ws_us`: weight standardisation forward + backward of all 53 convolutions of the model, device µs from a CUDA graph.
`--model wsgn_resnext50`:
* images/s of the engine's iteration and of the stock eager model, as above, on the ResNeXt-50 32×4d backbone;
* `gconv`: per distinct shape of its sixteen 32-group 3×3 convolutions, fwd, dgrad and wgrad µs of the csrc/gconv.cu
  entries and of cuDNN (`F.conv2d(groups=32)` and `aten.convolution_backward`, cudnn.benchmark on) on the same
  channels-last bf16 tensors, each device time from a CUDA graph of back-to-back calls, with achieved TFLOP/s
  (2·Ho·Wo·N·C·9·cpg per direction) and algorithmic GB/s (fwd reads x, Ŵ and writes y; dgrad reads dy, Ŵ and writes
  dx; wgrad reads x, dy and writes dŴ — fp32 for the kernels, bf16 for cuDNN).
The card's name and power limit are part of the line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

SIZE, BS = 320, 16
# (C, channels per group, stride, input side) of the ResNeXt backbone's grouped 3×3 convolutions at a 320×320 input
GCONV_SHAPES = ((128, 4, 1, 80), (256, 8, 2, 80), (256, 8, 1, 40), (512, 16, 2, 40), (512, 16, 1, 20),
                (1024, 32, 2, 20), (1024, 32, 1, 10))
# (channels, side) of the backbone's GroupNorm layers at a 320×320 input
GN_SHAPES = ((64, 160), (64, 80), (128, 80), (256, 80), (128, 40), (256, 40), (512, 40), (256, 20), (512, 20),
             (1024, 20), (512, 10), (2048, 10))


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit_w": float(out[1])}


def timed_ms(fn, iters: int) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def engine_img_s(steps: int, warmup: int, model_name: str = "wsgn_res50") -> float:
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = Trainer(model_name=model_name, dtype=torch.bfloat16, use_graph=True, report_items=False)
    x, m = (t.cuda() for t in synth_batch(0, BS, SIZE))
    for _ in range(warmup):
        tr.forward_backward_update(x, m, report=False)
    torch.cuda.synchronize()
    return BS / (timed_ms(lambda: tr.forward_backward_update(x, m, report=False), steps) * 1e-3)


def stock_img_s(steps: int, warmup: int, model_name: str = "wsgn_res50") -> float:
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.synthetic import synth_batch
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    model = getattr(network, model_name)().cuda().to(memory_format=torch.channels_last).train()
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9, weight_decay=5e-4)
    x, m = (t.cuda() for t in synth_batch(0, BS, SIZE))
    x = x.contiguous(memory_format=torch.channels_last)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            p = model(x)
        p = p.float()
        s = torch.sigmoid(p)
        inter = s * m
        loss = F.binary_cross_entropy_with_logits(p, m) + ((s - inter).sum() + (m - inter).sum()) / (s.sum() + m.sum() + 1e-6)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    return BS / (timed_ms(step, steps) * 1e-3)


def graph_us(calls, reps: int = 20, replays: int = 20) -> float:
    """µs per call of `calls()` (a sequence of launches), from a CUDA graph holding `reps` copies of it replayed
    `replays` times: device time without the Python / ctypes cost of issuing each launch"""
    calls()                                                # eager once: workspaces, cuBLAS/cuDNN handles
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            calls()
    g.replay()
    torch.cuda.synchronize()
    return timed_ms(g.replay, replays) * 1e3 / reps


def groupnorm_layers() -> list[dict]:
    from distributed_sod_project_b200 import _lib, wsgn
    lib, G = _lib.lib(), _lib.SOD_GN_GROUPS
    rows = []
    for c, side in GN_SHAPES:
        g = torch.Generator(device="cuda").manual_seed(c + side)
        cl = torch.channels_last
        x = torch.randn(BS, c, side, side, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        dy = torch.randn(BS, c, side, side, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        gamma, beta = torch.rand(c, device="cuda") + 0.5, torch.randn(c, device="cuda")
        dgamma, dbeta = torch.empty_like(gamma), torch.empty_like(beta)
        stats = torch.empty(BS * G * 2, device="cuda")
        hw = side * side
        ws = wsgn._workspace(x.device, int(lib.sod_groupnorm_workspace_bytes(BS, hw, c, G)))
        bf16 = _lib.dtype_code(x.dtype)

        def ours_fwd():
            _lib.check(lib.sod_groupnorm_fwd(x.data_ptr(), None, y.data_ptr(), bf16, gamma.data_ptr(), beta.data_ptr(),
                                             stats.data_ptr(), BS, hw, c, G, 1e-5, 1, ws.data_ptr(), ws.numel(),
                                             _lib.stream_ptr()))

        def ours_bwd():
            _lib.check(lib.sod_groupnorm_bwd(dy.data_ptr(), x.data_ptr(), y.data_ptr(), dx.data_ptr(), None, bf16,
                                             gamma.data_ptr(), stats.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), BS, hw,
                                             c, G, 1, ws.data_ptr(), ws.numel(), 0, _lib.stream_ptr()))

        # torch's GroupNorm kernels take NCHW-contiguous input only: F.group_norm makes a channels-last tensor contiguous
        # first (and autograd hands the kernel a contiguous dy), so those copies are part of its time here too
        g16, b16 = gamma.to(x.dtype), beta.to(x.dtype)
        xc = x.contiguous()
        _, mean, rstd = torch.ops.aten.native_group_norm(xc, g16, b16, BS, c, hw, G, 1e-5)
        torch_fwd = lambda: torch.ops.aten.native_group_norm(x.contiguous(), g16, b16, BS, c, hw, G, 1e-5)  # noqa: E731
        torch_bwd = lambda: torch.ops.aten.native_group_norm_backward(dy.contiguous(), xc, mean, rstd, g16, BS, c, hw,  # noqa: E731
                                                                      G, [True, True, True])
        ours_fwd()
        out = {"c": c, "hw": side, "n": BS}
        es, numel = x.element_size(), x.numel()
        for name, fwd, bwd, fb, bb in (("sod", ours_fwd, ours_bwd, 2, 4), ("torch", torch_fwd, torch_bwd, 2, 3)):
            tf, tb = graph_us(fwd), graph_us(bwd)
            out[f"{name}_fwd_us"], out[f"{name}_bwd_us"] = round(tf, 2), round(tb, 2)
            out[f"{name}_fwd_gbs"] = round(fb * numel * es / (tf * 1e-6) / 1e9, 1)
            out[f"{name}_bwd_gbs"] = round(bb * numel * es / (tb * 1e-6) / 1e9, 1)
        rows.append(out)
    return rows


def ws_model_us() -> float:
    """weight standardisation forward + backward of all 53 convolutions (bf16 Ŵ), device µs from a CUDA graph"""
    from distributed_sod_project_b200 import _lib, network
    lib = _lib.lib()
    model = network.wsgn_res50().cuda().to(memory_format=torch.channels_last)
    ws = [m.weight.detach() for m in model.modules() if isinstance(m, network.blocks.WSConv2d)]
    hats = [torch.empty_like(w, dtype=torch.bfloat16) for w in ws]
    ups = [torch.randn_like(w).to(torch.bfloat16) for w in ws]
    grads = [torch.empty_like(w) for w in ws]
    bf16 = _lib.dtype_code(torch.bfloat16)

    def both():
        for w, h, u, d in zip(ws, hats, ups, grads):
            _lib.check(lib.sod_ws_fwd(w.data_ptr(), h.data_ptr(), bf16, w.shape[0], w[0].numel(), 1e-5, _lib.stream_ptr()))
            _lib.check(lib.sod_ws_bwd(w.data_ptr(), u.data_ptr(), bf16, d.data_ptr(), w.shape[0], w[0].numel(), 1e-5, 0,
                                      _lib.stream_ptr()))

    return round(graph_us(both, reps=2, replays=20), 1)


def gconv_flops_bytes(c: int, cpg: int, stride: int, side: int, es: int = 2) -> dict:
    """operations of one direction, and the bytes each direction has to move, from the shape"""
    so = (side - 1) // stride + 1
    x, y, w = BS * side * side * c * es, BS * so * so * c * es, c * 9 * cpg
    return {"flop": 2 * BS * so * so * c * 9 * cpg, "fwd": x + w * es + y, "dgrad": y + w * es + x,
            "wgrad_sod": x + y + 4 * w, "wgrad_cudnn": x + y + w * es}


def gconv_layers() -> list[dict]:
    from distributed_sod_project_b200 import _lib
    lib, G, st = _lib.lib(), _lib.SOD_GCONV_GROUPS, _lib.stream_ptr
    torch.backends.cudnn.benchmark = True
    rows = []
    for c, cpg, stride, side in GCONV_SHAPES:
        g = torch.Generator(device="cuda").manual_seed(c + side)
        cl, so = torch.channels_last, (side - 1) // stride + 1
        x = torch.randn(BS, c, side, side, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        dy = torch.randn(BS, c, so, so, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=cl)
        w = (torch.randn(c, cpg, 3, 3, device="cuda", generator=g) * 0.1).to(torch.bfloat16).contiguous(memory_format=cl)
        y, dx = torch.empty_like(dy), torch.empty_like(x)
        dw = torch.empty(w.shape, dtype=torch.float32, device="cuda", memory_format=cl)
        ws = torch.empty(int(lib.sod_gconv3x3_wgrad_workspace_bytes(BS, side, side, c, G, stride)), dtype=torch.uint8,
                         device="cuda")
        bf16 = _lib.dtype_code(x.dtype)
        sod = {
            "fwd": lambda: _lib.check(lib.sod_gconv3x3_fwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), bf16, BS, side,
                                                           side, c, G, stride, st())),
            "dgrad": lambda: _lib.check(lib.sod_gconv3x3_dgrad(dy.data_ptr(), w.data_ptr(), dx.data_ptr(), bf16, BS,
                                                               side, side, c, G, stride, st())),
            "wgrad": lambda: _lib.check(lib.sod_gconv3x3_wgrad(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), bf16, BS,
                                                               side, side, c, G, stride, ws.data_ptr(), ws.numel(),
                                                               st())),
        }
        cb = torch.ops.aten.convolution_backward
        cudnn = {
            "fwd": lambda: F.conv2d(x, w, None, stride, 1, 1, G),
            "dgrad": lambda: cb(dy, x, w, None, [stride] * 2, [1, 1], [1, 1], False, [0, 0], G, [True, False, False]),
            "wgrad": lambda: cb(dy, x, w, None, [stride] * 2, [1, 1], [1, 1], False, [0, 0], G, [False, True, False]),
        }
        fb = gconv_flops_bytes(c, cpg, stride, side)
        out = {"c": c, "cpg": cpg, "stride": stride, "hw": side, "n": BS}
        for name, fns in (("sod", sod), ("cudnn", cudnn)):
            for d, fn in fns.items():
                t = graph_us(fn)
                nbytes = fb[d] if d != "wgrad" else fb[f"wgrad_{name}"]
                out[f"{name}_{d}_us"] = round(t, 2)
                out[f"{name}_{d}_tflops"] = round(fb["flop"] / (t * 1e-6) / 1e12, 2)
                out[f"{name}_{d}_gbs"] = round(nbytes / (t * 1e-6) / 1e9, 1)
        rows.append(out)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=("wsgn_res50", "wsgn_resnext50"), default="wsgn_res50")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    line = {"gpu": card(), "workload": f"{SIZE}x{SIZE}, bs {BS}, bf16"}
    line[f"{args.model}_img_s"] = round(engine_img_s(args.steps, args.warmup, args.model), 1)
    line["stock_img_s"] = round(stock_img_s(args.steps, args.warmup, args.model), 1)
    if args.model == "wsgn_res50":
        line["groupnorm"] = groupnorm_layers()
        line["ws_us"] = ws_model_us()
    else:
        line["gconv"] = gconv_layers()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
