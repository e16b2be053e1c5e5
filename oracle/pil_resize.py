"""Oracle (TEST INFRASTRUCTURE, never imported by the product path): numpy restatement of Pillow's 8-bit two-pass
resampler, `Image.resize(size, BILINEAR | BICUBIC)` with box = the whole image and reducing_gap=None, for "L" and "RGB".

The reference resizes every 8-bit prediction to its ground truth's size with `ToPILImage()(out).resize(gt.size)`
(train.py:392-395: BICUBIC, the default of `Image.resize`) and feeds test images through torchvision
`Resize((S, S))` (utils/dataset.py:97-104: Pillow BILINEAR).  Pillow builds per-axis float64 coefficient tables, rounds
them to 22-bit fixed point, and from there on only adds integers, so the result is reproducible bit for bit.

The float64 part is written as one operation per numpy call (no fused multiply-add can happen), in Pillow's order.
"""
from __future__ import annotations

import math

import numpy as np

BILINEAR, BICUBIC = 2, 3          # PIL.Image.Resampling values
SUPPORT = {BILINEAR: 1.0, BICUBIC: 2.0}
PRECISION_BITS = 22


def _filter(kind: int, x: float) -> float:
    x = abs(x)
    if kind == BILINEAR:
        return 1.0 - x if x < 1.0 else 0.0
    # Keys' cubic with a = -0.5; (a + 2) = 1.5 and (a + 3) = 2.5 are exact
    if x < 1.0:
        return ((1.5 * x - 2.5) * x) * x + 1.0
    if x < 2.0:
        return (((x - 5.0) * x + 8.0) * x - 4.0) * -0.5
    return 0.0


def coeffs(in_size: int, out_size: int, kind: int):
    """→ (bounds int[out, 2] = (first tap, tap count), kk int32[out, ksize]) as Pillow's precompute_coeffs followed by
    normalize_coeffs_8bpc computes them"""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = SUPPORT[kind] * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds = np.zeros((out_size, 2), dtype=np.int64)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_filter(kind, (float(x + xmin) - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:                                   # sequential, in tap order
            ww += v
        for x, v in enumerate(w):
            k = v / ww if ww != 0.0 else v
            kk[xx, x] = int(k * (1 << PRECISION_BITS) + (0.5 if k >= 0 else -0.5))     # int(): towards zero
        bounds[xx] = (xmin, xmax)
    return bounds, kk


def _pass(img: np.ndarray, bounds, kk, axis: int, first: int = 0) -> np.ndarray:
    """one 8-bit pass along `axis` (1: horizontal, 0: vertical) of img [H, W, C] uint8; tap offsets shifted by -first"""
    src = img.astype(np.int64)
    out_n = bounds.shape[0]
    shape = list(img.shape)
    shape[axis] = out_n
    acc = np.full(shape, 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for o in range(out_n):
        lo, cnt = int(bounds[o, 0]) - first, int(bounds[o, 1])
        for t in range(cnt):
            if axis == 1:
                acc[:, o] += src[:, lo + t] * int(kk[o, t])
            else:
                acc[o] += src[lo + t] * int(kk[o, t])
    return np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize(img: np.ndarray, size, kind: int = BICUBIC) -> np.ndarray:
    """img uint8 [H, W] ("L") or [H, W, 3] ("RGB"); size = (width, height) as PIL takes it."""
    out_w, out_h = int(size[0]), int(size[1])
    gray = img.ndim == 2
    x = img[:, :, None] if gray else img
    in_h, in_w = x.shape[:2]
    if (out_w, out_h) == (in_w, in_h):
        return img.copy()
    bh, kh = coeffs(in_w, out_w, kind)
    bv, kv = coeffs(in_h, out_h, kind)
    if out_w != in_w:
        # the horizontal pass only produces the source rows the vertical pass reads
        first, last = int(bv[0, 0]), int(bv[-1, 0] + bv[-1, 1])
        x = _pass(x[first:last], bh, kh, axis=1)
        bv = bv.copy()
        bv[:, 0] -= first
    if out_h != in_h:
        x = _pass(x, bv, kv, axis=0)
    return x[:, :, 0] if gray else x
