#!/usr/bin/env python
"""What evaluating an on-disk test set costs.  Prints one JSON line.

    python tools/bench_eval.py [--images 512] [--batch 24] [--size 320] [--workers 4] [--iters 200]

In one run, on the current GPU (its name and power limit are part of the output):
* writes a seeded test set under a temporary directory: `--images` JPEG images of 300–500 px in both orientations,
  PNG masks with soft edges;
* `end_to_end_img_s`: images/s of `evaluate.test_process` over that set at the reference's test batch size (24,
  reference test.py:30) — decode on `--workers` DataLoader workers, upload, Pillow-exact resize to S², network (res50,
  fp32, as the reference's test.py), quantize, resize back, ragged metric kernels — without the weighted F-measure
  (`no_wfm`), with it on the GPU (`wfm_gpu`, csrc/wfm.cu) and with it on the host (`wfm_host`, scipy); the last two
  report all six metrics as the reference does;
* `kernels_us`: one batch's resize and metric kernels alone (CUDA events, warmed up, `--iters` repetitions): RGB
  BILINEAR to S², "L" BICUBIC back to each ground truth's size, ragged head + hist, and the weighted F-measure's three
  launches (`wfm_ragged`, head included as it feeds them; `wfm_alone` without it);
* `host_reference_us`: the same batch through the reference's per-image host path — `ToPILImage`-equivalent 8-bit map,
  PIL `.resize(gt.size)` and the numpy metrics of `oracle.metrics.TotalMetric` (without the weighted F-measure).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import gpu_info  # noqa: E402


def write_set(root: str, n: int, seed: int = 0) -> None:
    from PIL import Image
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "Image"))
    os.makedirs(os.path.join(root, "Mask"))
    for i in range(n):
        a, b = int(rng.integers(300, 501)), int(rng.integers(300, 501))
        h, w = (max(a, b), min(a, b)) if i % 2 else (min(a, b), max(a, b))
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        img = np.stack([xx * 255 / w, yy * 255 / h, rng.integers(0, 256, (h, w)).astype(np.float32)], -1)
        img = np.clip(img + rng.normal(0, 20, img.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(root, "Image", f"{i:05d}.jpg"), quality=90)
        cy, cx, r = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w, rng.uniform(0.15, 0.35) * min(h, w)
        m = np.clip((r - np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)) / 4.0 + 0.5, 0, 1)
        Image.fromarray((m * 255).round().astype(np.uint8), "L").save(os.path.join(root, "Mask", f"{i:05d}.png"))


def _events_us(fn, iters: int) -> float:
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--batch", type=int, default=24)
    ap.add_argument("--size", type=int, default=320)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a GPU")
    from PIL import Image

    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.data import make_eval_loader
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.evaluate import prepare_inputs, test_process
    from distributed_sod_project_b200.metrics import SaliencyMetrics, wfm_sums_ragged
    from distributed_sod_project_b200.pipeline import Ragged, resize_u8
    from oracle import metrics as om

    torch.cuda.set_device(0)
    result = {"gpu": gpu_info(0), "images": args.images, "batch": args.batch, "size": args.size, "workers": args.workers}
    model = Trainer(model_name="res50", dtype=torch.float32, channels_last=True, report_items=False).model
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "SET")
        write_set(root, args.images)
        loader, n = make_eval_loader(root, args.batch, num_workers=args.workers)
        warm, _ = make_eval_loader(root, args.batch, indices=range(2 * args.batch), num_workers=0)
        test_process(model, warm, length=2 * args.batch, input_size=args.size)             # cuDNN picks its algorithms
        e2e = {}
        for wfm in (None, "gpu", "host"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            test_process(model, loader, length=n, wfm=wfm, input_size=args.size)
            torch.cuda.synchronize()
            e2e[f"wfm_{wfm}" if wfm else "no_wfm"] = round(n / (time.perf_counter() - t0), 1)
        result["end_to_end_img_s"] = e2e

        # one batch, kernels alone
        batch = next(iter(warm))
        model.eval()
        with torch.no_grad():
            x, gt = prepare_inputs(batch, args.size)
            pred_s = SaliencyMetrics.quantize(model(x).float(), apply_sigmoid=True)[:, 0].contiguous()
        dev = torch.device("cuda", 0)
        img = Ragged(batch.img.to(dev), batch.img_hw, 3)
        pred_r = Ragged.stack(pred_s)
        pred = resize_u8(pred_r, gt.hw, _lib.SOD_RESIZE_BICUBIC)
        cal = SaliencyMetrics()
        head = torch.empty((len(gt), 8), dtype=torch.int64, device=dev)
        lib = _lib.lib()

        def head_launch():
            _lib.check(lib.sod_saliency_head_ragged(pred.data.data_ptr(), gt.data.data_ptr(), len(gt), pred.off_d.data_ptr(),
                                                    pred.hw_d.data_ptr(), head.data_ptr(), _lib.stream_ptr()))

        head_launch()
        result["kernels_us"] = {
            "resize_rgb_bilinear_to_S": round(_events_us(lambda: resize_u8(img, (args.size, args.size), _lib.SOD_RESIZE_BILINEAR), args.iters), 1),
            "resize_l_bicubic_to_gt": round(_events_us(lambda: resize_u8(pred_r, gt.hw, _lib.SOD_RESIZE_BICUBIC), args.iters), 1),
            "metric_head_hist_ragged": round(_events_us(lambda: cal.update_ragged(pred, gt), args.iters), 1),
            "wfm_ragged": round(_events_us(lambda: (head_launch(), wfm_sums_ragged(pred, gt, head)), args.iters), 1),
            "wfm_alone": round(_events_us(lambda: wfm_sums_ragged(pred, gt, head), args.iters), 1),
        }
        cal._pending.clear()

        # the reference's host path on the same batch: PIL resize + numpy metrics, per image
        p8 = pred_s.cpu().numpy()
        gts = [gt.image(i).cpu().numpy() for i in range(len(gt))]
        reps = 3
        t0 = time.perf_counter()
        for _ in range(reps):
            tot = om.TotalMetric(len(gts), with_wfm=False)
            for i, g in enumerate(gts):
                out = np.asarray(Image.fromarray(p8[i], "L").resize(g.shape[::-1]))
                tot.update(*om.normalise(out, g))
            tot.show()
        result["host_reference_us"] = round((time.perf_counter() - t0) * 1e6 / reps, 1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
