"""On-disk SOD training and test sets: what the reference's `ImageFolder` + `create_loader` read
(utils/dataset.py:22-156, consumed at train.py:121-138 and 338-417), with everything after decoding on the GPU.

Listing follows the reference's rules:
  - `root` is a folder with `Image/` and `Mask/`, or a list file whose lines start with `<dir>/<name>`, read as
    `<dir>/Image/<name><prefix[0]>` and `<dir>/Mask/<name><prefix[1]>`;
  - in the folder form the masks drive the pairs: every mask with the mask folder's extension gives one pair, the image
    being `<stem><image folder's extension>`; a folder holding several extensions uses .png, else .jpg, else .bmp.
Pairs come sorted by mask name, so every rank sees the same order (the metrics are means: order does not change them).

Workers only decode, at the original size: `Image.open(...).convert("RGB")` for images and `.convert("L")` for ground
truths.  The collate packs both into ragged uint8 batches (`EvalBatch`, for training batches too); the device side
(`evaluate.test_process`) resizes, normalises, runs the model, resizes the predictions back and histograms them, or
(`pipeline.TrainPrefetcher`) resizes, augments and normalises the training batch.
"""
from __future__ import annotations

import os
from dataclasses import dataclass

import numpy as np
import torch

_EXT_ORDER = (".png", ".jpg", ".bmp")


def _folder_ext(names) -> str:
    exts = {os.path.splitext(f)[1] for f in names}
    if len(exts) == 1:
        return exts.pop()
    for e in _EXT_ORDER:
        if e in exts:
            return e
    raise ValueError(f"no .png, .jpg or .bmp file among the extensions {sorted(exts)}")


def list_pairs(root: str, prefix=(".jpg", ".png")) -> list[tuple[str, str]]:
    """(image path, mask path) pairs of one test set, in mask-name order"""
    if os.path.isdir(root):
        img_dir, mask_dir = os.path.join(root, "Image"), os.path.join(root, "Mask")
        img_ext = _folder_ext(os.listdir(img_dir))
        masks = os.listdir(mask_dir)
        mask_ext = _folder_ext(masks)
        stems = sorted(os.path.splitext(f)[0] for f in masks if f.endswith(mask_ext))
        return [(os.path.join(img_dir, s + img_ext), os.path.join(mask_dir, s + mask_ext)) for s in stems]
    if os.path.isfile(root):
        pairs = []
        with open(root, encoding="utf-8") as f:
            for line in f:
                if not line.split():
                    continue
                p = line.split()[0]
                d, b = os.path.dirname(p), os.path.basename(p)
                pairs.append((os.path.join(d, "Image", b + prefix[0]), os.path.join(d, "Mask", b + prefix[1])))
        return pairs
    raise FileNotFoundError(f"{root} is neither a folder nor a list file")


def image_name(img_path: str) -> str:
    """the name a saved prediction takes (`<name>.png`): the file name up to its first dot, as the reference's"""
    return os.path.basename(img_path).split(".")[0]


@dataclass
class EvalBatch:
    """host side of one ragged evaluation batch (pinned by the DataLoader): images packed HWC RGB, ground truths
    packed HW, their sizes int32 [n, 2], and the image names"""
    img: torch.Tensor
    img_hw: torch.Tensor
    gt: torch.Tensor
    gt_hw: torch.Tensor
    names: list

    def pin_memory(self):
        return EvalBatch(self.img.pin_memory(), self.img_hw, self.gt.pin_memory(), self.gt_hw, self.names)

    def __len__(self):
        return len(self.names)


class EvalFolder(torch.utils.data.Dataset):
    """the `indices` of a pair list, decoded at the original size"""

    def __init__(self, pairs, indices=None):
        self.pairs = list(pairs)
        self.indices = list(range(len(self.pairs))) if indices is None else list(indices)

    def __len__(self):
        return len(self.indices)

    def __getitem__(self, i):
        from PIL import Image
        img_path, mask_path = self.pairs[self.indices[i]]
        with Image.open(img_path) as im:
            img = np.asarray(im.convert("RGB"))
        with Image.open(mask_path) as im:
            gt = np.asarray(im.convert("L"))
        return img, gt, image_name(img_path)


def collate(samples) -> EvalBatch:
    imgs, gts, names = zip(*samples)
    return EvalBatch(img=torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs])),
                     img_hw=torch.tensor([a.shape[:2] for a in imgs], dtype=torch.int32),
                     gt=torch.from_numpy(np.concatenate([a.reshape(-1) for a in gts])),
                     gt_hw=torch.tensor([a.shape[:2] for a in gts], dtype=torch.int32),
                     names=list(names))


def make_eval_loader(root: str, batch_size: int, indices=None, num_workers: int = 0, prefix=(".jpg", ".png")):
    """→ (DataLoader of EvalBatch over `indices` of the set — this rank's shard —, number of images in the whole set)"""
    pairs = list_pairs(root, prefix)
    ds = EvalFolder(pairs, indices)
    loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=False, num_workers=num_workers, collate_fn=collate,
                                         pin_memory=torch.cuda.is_available(), drop_last=False)
    return loader, len(pairs)


def make_train_loader(root: str, batch_size: int, world_size: int = 1, rank: int = 0, num_workers: int = 0,
                      prefix=(".jpg", ".png"), seed: int = 0):
    """this rank's DataLoader of ragged `EvalBatch` training batches of the reference's training set `root`
    (utils/dataset.py:72-95, train.py:121-138): the workers only decode; resizing and augmentation run on the GPU
    (`pipeline.TrainPrefetcher`).  Sampling is `DistributedSampler`'s: a shuffle from seed + epoch (`sampler.set_epoch`),
    padded to a multiple of the world size, this rank's slice, and only full batches.  A missing path is an error naming
    it: there is no fall-back to synthetic data."""
    if not root or not os.path.exists(root):
        raise FileNotFoundError(f"training set (tr_data_path): {root!r} does not exist")
    ds = EvalFolder(list_pairs(root, prefix))
    sampler = torch.utils.data.DistributedSampler(ds, num_replicas=world_size, rank=rank, shuffle=True, seed=seed)
    loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, sampler=sampler, num_workers=num_workers, collate_fn=collate,
                                         pin_memory=torch.cuda.is_available(), drop_last=True)
    if len(loader) == 0:
        raise ValueError(f"training set {root!r}: {len(ds)} images give no batch of {batch_size} on each of {world_size} rank(s)")
    return loader


def open_test_set(data_name: str, data_path: str, batch_size: int, num_workers: int = 0, prefix=(".jpg", ".png")):
    """this rank's shard of one configured test set → (loader, number of images over all ranks).  A missing path is an
    error naming the set: there is no fall-back to synthetic data."""
    from .evaluate import shard
    if not data_path or not os.path.exists(data_path):
        raise FileNotFoundError(f"test set {data_name!r}: {data_path!r} does not exist")
    n = len(list_pairs(data_path, prefix))
    loader, _ = make_eval_loader(data_path, batch_size, indices=shard(n), num_workers=num_workers, prefix=prefix)
    return loader, n
