"""Oracle (TEST INFRASTRUCTURE): the reference's tensor-side input pipeline in plain torch CPU ops —
`ToTensor` + `Normalize` per image (utils/dataset.py:86-96), `ToTensor` per mask (:110-116), the left-right flip of
utils/joint_transforms.py:19-23, and the multi-scale collate (`_collate_fn`, utils/dataset.py:125-132: stack, then
`interpolate` bilinear align_corners=False for the image and nearest for the mask).  torchvision's ToTensor/Normalize
are `u8 → float32 / 255` and `(x - mean) / std`; they are written out here so the oracle needs no PIL round trip."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def normalise_table(mean=MEAN, std=STD):
    """float32 [3, 256]: ToTensor + Normalize of every byte value, `(u / 255 − mean) / std` in IEEE fp32"""
    u = torch.arange(256, dtype=torch.float32)
    return torch.stack([(u / 255 - torch.tensor(m, dtype=torch.float32)) / torch.tensor(s, dtype=torch.float32)
                        for m, s in zip(mean, std)])


def bilinear_taps(n_in: int, n_out: int, fused: bool = True):
    """one axis of `interpolate(bilinear, align_corners=False)` in fp32: (i0, i1, λ) per output index, float64 λ.
    The source coordinate max(scale·(o + ½) − ½, 0), scale = fp32(n_in / n_out), is rounded once to fp32 (`fused`,
    what torch's CPU kernel and the pre-processing kernel compute) or after the product and after the subtraction."""
    s = np.float32(np.float32(n_in) / np.float32(n_out))
    o = np.arange(n_out, dtype=np.float64) + 0.5                        # exact
    if fused:
        f = (np.float64(s) * o - 0.5).astype(np.float32)                   # the float64 product and difference are exact
    else:
        f = (np.float64(s) * o).astype(np.float32) - np.float32(0.5)
    f = np.maximum(f, np.float32(0))
    i0 = np.floor(f).astype(np.int64)
    i1 = np.minimum(i0 + 1, n_in - 1)
    return i0, i1, f.astype(np.float64) - i0


def nearest_index(n_in: int, n_out: int):
    """one axis of legacy `interpolate(nearest)`: min(floor(fp32(o · fp32(n_in / n_out))), n_in − 1)"""
    s = np.float32(np.float32(n_in) / np.float32(n_out))
    p = (np.arange(n_out, dtype=np.float64) * np.float64(s)).astype(np.float32)
    return np.minimum(np.floor(p).astype(np.int64), n_in - 1)


def preprocess(img_u8: torch.Tensor, mask_u8: torch.Tensor | None, size=None, flip=None, mean=MEAN, std=STD):
    """img_u8 [N,H,W,3] uint8, mask_u8 [N,H,W] uint8 (CPU) → (img [N,3,S,S] f32, mask [N,1,S,S] f32)"""
    imgs, masks = [], []
    for i in range(img_u8.shape[0]):
        im = img_u8[i]
        mk = mask_u8[i] if mask_u8 is not None else None
        if flip is not None and bool(flip[i]):
            im = im.flip(1)
            mk = mk.flip(1) if mk is not None else None
        t = im.permute(2, 0, 1).to(torch.float32).div(255)                       # ToTensor
        t = (t - torch.tensor(mean).view(3, 1, 1)) / torch.tensor(std).view(3, 1, 1)   # Normalize
        imgs.append(t)
        if mk is not None:
            masks.append(mk[None].to(torch.float32).div(255))
    img = torch.stack(imgs)
    mask = torch.stack(masks) if masks else None
    if size is not None:
        hw = (size, size) if isinstance(size, int) else tuple(size)
        img = F.interpolate(img, size=hw, mode="bilinear", align_corners=False)
        if mask is not None:
            mask = F.interpolate(mask, size=hw, mode="nearest")
    return img, mask
