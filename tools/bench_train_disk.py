#!/usr/bin/env python
"""What training from an on-disk set costs.  Prints one JSON line.

    python tools/bench_train_disk.py [--images 512] [--batch 16] [--size 320] [--workers 4 8] [--iters 200]
                                     [--joint-transforms '[["JointResize", 320], ["RandomScaleCrop", 320, 1.5], ...]']

In one run, on the current GPU (its name and power limit are part of the output):
* writes a seeded training set under a temporary directory: `--images` JPEG images of 300–500 px in both orientations,
  PNG masks with soft edges (the set of tools/bench_eval.py);
* `gpu_us_per_batch`: one batch's device work after warm-up (CUDA events, `--iters` repetitions): Pillow-exact BICUBIC
  resize of images and masks to S², flip / rotate / ColorJitter (`augment_u8`), ToTensor + Normalize
  (`preprocess_batch`), each and all together; the upload is not included;
* `host_reference_us_per_batch`: the same batch through the reference's per-sample PIL chain on one host thread:
  JointResize, flip, rotate, ColorJitter, ToTensor, Normalize, then the stack of the default collate;
* `decode_img_s`: images/s the DataLoader workers deliver alone (decode and collate, no GPU), per worker count;
* `train_img_s`: end-to-end training images/s from disk (res50, bf16, CUDA-graph replay, the benchmark's
  configuration), per worker count, over one whole epoch after a warm-up epoch;
* `synthetic_device_img_s`: the same trainer on a device-resident batch, i.e. the iteration alone.
With `--joint-transforms` (a `joint_transforms` list as config.py takes it), also:
* `joint_gpu_us_per_batch`: the chain's stages on the same batch after warm-up: the size step, RandomScaleCrop, the
  blur (on the drawn radii: about half the samples blur, the others run the identity box), the whole chain with
  ColorJitter (`joint_chain_u8`), and the chain plus `preprocess_batch`;
* `joint_train_img_s`: end-to-end training images/s from disk with the chain, per worker count.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import gpu_info  # noqa: E402
from bench_eval import _events_us, write_set  # noqa: E402


def _epoch_img_s(trainer, pf, epoch: int) -> float:
    pf.set_epoch(epoch)
    torch.cuda.synchronize()
    t0, n = time.perf_counter(), 0
    for x, m, _ in pf:
        trainer.forward_backward_update(x, m)
        n += x.shape[0]
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=320)
    ap.add_argument("--workers", type=int, nargs="+", default=[4, 8])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--joint-transforms", type=json.loads, default=None,
                    help="a joint_transforms chain (JSON) measured besides the reference's")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_disk.py measures on a GPU")
    import torchvision.transforms as T
    import torchvision.transforms.functional as TF
    from PIL import Image

    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.data import make_train_loader
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.pipeline import (Ragged, TrainPrefetcher, augment_u8, draw_augment_params,
                                                       draw_joint_params, gaussian_blur_u8, joint_chain_u8, joint_size_step,
                                                       parse_joint_transforms, preprocess_batch, random_scale_crop,
                                                       resize_u8)

    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda", 0)
    S, bs = args.size, args.batch
    result = {"gpu": gpu_info(0), "images": args.images, "batch": bs, "size": S}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "TR")
        write_set(root, args.images)

        # one batch, device work alone
        batch = next(iter(make_train_loader(root, bs, num_workers=0)))
        img = Ragged(batch.img.to(dev), batch.img_hw, 3)
        mask = Ragged(batch.gt.to(dev), batch.gt_hw, 1)
        params = draw_augment_params(bs, S, torch.Generator().manual_seed(0))
        ri = resize_u8(img, (S, S), _lib.SOD_RESIZE_BICUBIC).as_batch()
        rm = resize_u8(mask, (S, S), _lib.SOD_RESIZE_BICUBIC).as_batch()
        ai, am = augment_u8(ri, rm, params)

        def chain():
            a, b = augment_u8(resize_u8(img, (S, S), _lib.SOD_RESIZE_BICUBIC).as_batch(),
                              resize_u8(mask, (S, S), _lib.SOD_RESIZE_BICUBIC).as_batch(), params)
            preprocess_batch(a, b)

        result["gpu_us_per_batch"] = {
            "resize_image_and_mask": round(_events_us(lambda: (resize_u8(img, (S, S), _lib.SOD_RESIZE_BICUBIC),
                                                                resize_u8(mask, (S, S), _lib.SOD_RESIZE_BICUBIC)), args.iters), 1),
            "augment": round(_events_us(lambda: augment_u8(ri, rm, params), args.iters), 1),
            "preprocess": round(_events_us(lambda: preprocess_batch(ai, am), args.iters), 1),
            "all": round(_events_us(chain, args.iters), 1),
        }

        chain = parse_joint_transforms(args.joint_transforms, S) if args.joint_transforms is not None else None
        if chain is not None:
            result["joint_transforms"] = chain
            jp = draw_joint_params(bs, chain, torch.Generator().manual_seed(0))
            us = {"size_step": round(_events_us(lambda: joint_size_step(chain[0], img, mask), args.iters), 1)}
            si, sm = joint_size_step(chain[0], img, mask)
            if jp.crop is not None:
                us["random_scale_crop"] = round(_events_us(lambda: random_scale_crop(si, sm, jp.crop), args.iters), 1)
            if jp.blur is not None:
                bi = si.as_batch().contiguous()
                us["gaussian_blur"] = round(_events_us(lambda: gaussian_blur_u8(bi, jp.blur), args.iters), 1)
            us["chain_with_jitter"] = round(_events_us(lambda: joint_chain_u8(chain, jp, img, mask), args.iters), 1)
            us["all"] = round(_events_us(lambda: preprocess_batch(*joint_chain_u8(chain, jp, img, mask)), args.iters), 1)
            result["joint_gpu_us_per_batch"] = us

        # the reference's host chain on the same batch, decoded images in hand
        norm = T.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
        ims = [Image.fromarray(img.image(i).cpu().numpy(), "RGB") for i in range(bs)]
        mks = [Image.fromarray(mask.image(i).cpu().numpy(), "L") for i in range(bs)]
        jit = [TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation]
        reps = 3
        t0 = time.perf_counter()
        for _ in range(reps):
            xs, ms = [], []
            for i in range(bs):
                a, b = ims[i].resize((S, S)), mks[i].resize((S, S))
                if params.flip[i]:
                    a, b = a.transpose(Image.FLIP_LEFT_RIGHT), b.transpose(Image.FLIP_LEFT_RIGHT)
                a, b = a.rotate(params.angle[i], Image.BILINEAR), b.rotate(params.angle[i], Image.NEAREST)
                for op in params.order[i]:
                    a = jit[op](a, params.factor[i][op])
                xs.append(norm(TF.to_tensor(a)))
                ms.append(TF.to_tensor(b))
            torch.stack(xs), torch.stack(ms)
        result["host_reference_us_per_batch"] = round((time.perf_counter() - t0) * 1e6 / reps, 1)

        # decode alone
        result["decode_img_s"] = {}
        for w in args.workers:
            loader = make_train_loader(root, bs, num_workers=w)
            t0, n = time.perf_counter(), 0
            for b in loader:
                n += len(b)
            result["decode_img_s"][str(w)] = round(n / (time.perf_counter() - t0), 1)

        # end to end, and the iteration alone
        trainer = Trainer(model_name="res50", dtype=torch.bfloat16, channels_last=True, report_items=False, use_graph=True)
        result["train_img_s"] = {}
        for w in args.workers:
            pf = TrainPrefetcher(make_train_loader(root, bs, num_workers=w), S, seed=0)
            _epoch_img_s(trainer, pf, 0)                                            # warm-up: graph capture, cuDNN
            result["train_img_s"][str(w)] = round(_epoch_img_s(trainer, pf, 1), 1)
        if chain is not None:
            result["joint_train_img_s"] = {}
            for w in args.workers:
                pf = TrainPrefetcher(make_train_loader(root, bs, num_workers=w), S, seed=0, joint_transforms=chain)
                _epoch_img_s(trainer, pf, 0)
                result["joint_train_img_s"][str(w)] = round(_epoch_img_s(trainer, pf, 1), 1)
        x, m, _ = next(iter(TrainPrefetcher(make_train_loader(root, bs, num_workers=0), S, seed=0)))
        steps = args.images // bs
        for _ in range(5):
            trainer.forward_backward_update(x, m)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            trainer.forward_backward_update(x, m)
        torch.cuda.synchronize()
        result["synthetic_device_img_s"] = round(steps * bs / (time.perf_counter() - t0), 1)
        result["host_cpus"] = os.cpu_count()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
