"""Evaluation seam: `test()` / `_test_process()` of the reference (train.py:338-417) — distributed, with the
per-pixel work on the GPU (SURVEY §8f.4).

Reference: rank 0 alone runs every test set through the model, moves each sigmoid map to the CPU, turns it into an
8-bit PIL image, resizes it to the ground truth's size and feeds `CalTotalMetric` (≈40 numpy passes per image).
Here every rank evaluates its shard (`indices[rank::world]`, the order `DistributedSampler(shuffle=False)` would
give), the sigmoid + 8-bit quantisation + normalisation + histogramming run as four small kernels per batch
(`metrics.SaliencyMetrics`), and `show()` combines the ranks with one all-reduce.  Predictions whose size differs from
the ground truth's are resized on the GPU exactly as the reference's `to_pil(out).resize(gt.size)` does (Pillow
BICUBIC, bit for bit: `pipeline.resize_u8`).

Batches are either `(image [N,3,S,S] float CUDA, gt_u8 [N,H,W] uint8 CUDA)` tuples (the synthetic sets) or
`data.EvalBatch` (on-disk sets, images and ground truths at their original sizes).  An `EvalBatch` goes through:
upload → Pillow BILINEAR to S×S (torchvision `Resize((S, S))`, utils/dataset.py:97-104) → `preprocess_batch`
(ToTensor + Normalize) → model → `quantize` → Pillow BICUBIC to each ground truth's size → ragged metric kernels.
"""
from __future__ import annotations

import os

import torch

from . import _lib, comm
from .metrics import SaliencyMetrics
from .pipeline import Ragged, preprocess_batch, resize_u8


def prepare_inputs(batch, size: int):
    """EvalBatch → (network input [N,3,S,S] fp32 channels-last, ground truths as a ragged "L" batch), on the GPU"""
    dev = torch.device("cuda", torch.cuda.current_device())
    img = Ragged(batch.img.to(dev, non_blocking=True), batch.img_hw, 3)
    gt = Ragged(batch.gt.to(dev, non_blocking=True), batch.gt_hw, 1)
    img_s = resize_u8(img, (size, size), _lib.SOD_RESIZE_BILINEAR)
    x, _ = preprocess_batch(img_s.as_batch())
    return x, gt


def _save_predictions(pred: Ragged, names, save_dir: str) -> None:
    """`<name>.png` of every 8-bit prediction at its ground truth's size (train.py:397-399)"""
    from PIL import Image
    host = pred.data.cpu()
    for i, name in enumerate(names):
        h, w = int(pred.hw[i, 0]), int(pred.hw[i, 1])
        o = int(pred.off[i])
        Image.fromarray(host[o:o + h * w].view(h, w).numpy(), "L").save(os.path.join(save_dir, name + ".png"))


@torch.no_grad()
def test_process(model, batches, length: int | None = None, wfm: str | None = None, input_size: int = 320,
                 save_dir: str | None = None) -> dict:
    """`_test_process` (train.py:372-417).  `batches`: iterable of (image, gt_u8) tuples or `data.EvalBatch`, holding
    THIS rank's shard; `length`: total number of images over all ranks (checked in show(), like the reference's `num`);
    `input_size`: the network's S for `EvalBatch` inputs; `save_dir`: if set, each 8-bit prediction resized to its ground
    truth is written there as `<name>.png` (`EvalBatch` only: tuples carry no names); `wfm`: None (no weighted
    F-measure), "gpu" (csrc/wfm.cu) or "host" (scipy), see `metrics.SaliencyMetrics`.
    Returns {"MaxF","MeanF","WFM","MAE","SM","EM"}."""
    was_training = model.training
    model.eval()
    cal = SaliencyMetrics(num=length, wfm=wfm)
    if save_dir is not None:
        os.makedirs(save_dir, exist_ok=True)
    try:
        for batch in batches:
            if isinstance(batch, (tuple, list)):
                x, gt = batch
                logits = model(x)                                              # train.py:386-390
                pred_u8 = SaliencyMetrics.quantize(logits.float(), apply_sigmoid=True)[:, 0]    # .sigmoid() → ToPILImage
                if pred_u8.shape[-2:] != gt.shape[-2:]:
                    pred_u8 = resize_u8(Ragged.stack(pred_u8), tuple(gt.shape[-2:]), _lib.SOD_RESIZE_BICUBIC).as_batch()
                cal.update_batch(pred_u8, gt)
                continue
            x, gt = prepare_inputs(batch, input_size)
            logits = model(x)
            pred_s = SaliencyMetrics.quantize(logits.float(), apply_sigmoid=True)[:, 0]
            pred = resize_u8(Ragged.stack(pred_s), gt.hw, _lib.SOD_RESIZE_BICUBIC)      # .resize(gt.size), train.py:395
            cal.update_ragged(pred, gt)
            if save_dir is not None:
                _save_predictions(pred, batch.names, save_dir)
        return cal.show()
    finally:
        model.train(was_training)


def shard(n_items: int) -> range:
    """this rank's indices of an n-item evaluation set"""
    return range(comm.rank(), n_items, comm.world_size())
