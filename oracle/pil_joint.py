"""Oracle (TEST INFRASTRUCTURE, never imported by the product path): numpy restatement of the Pillow operations behind
the reference's other joint transforms (utils/joint_transforms.py:51-137), for "L" [H, W] and "RGB" [H, W, 3] uint8:

  * `resize_nearest`: `Image.resize(size, NEAREST)`.  Pillow (libImaging/Geometry.c, ImagingScaleAffine) tabulates each
    axis with a = in / out, xo = a·0.5 and then `xo += a` once per output pixel, so the rounding of the repeated float64
    addition is part of the result; `int((x + 0.5)·a)` differs from Pillow at some sizes.  Same size: a copy.
  * `window`: an (h, w) window at (dy, dx), zeros outside the source: `Image.crop` and PaddingSquare's zero padding.
  * `blur_params` / `gaussian_blur`: `filter(GaussianBlur(r))`, Pillow's extended box blur (libImaging/BoxBlur.c).  The
    box radius comes from float32 arithmetic (with the square root and floor in float64, as the C code promotes them),
    ww = (uint32)(2²⁴ / (2·rad + 1)) in float32, fw = (2²⁴ − (2⌊rad⌋ + 1)·ww) / 2; three horizontal passes, then three
    vertical, each (ww·Σ x[i+k] + fw·(x[i−R−1] + x[i+R+1]) + 2²³) >> 24 over clamped indices.
"""
from __future__ import annotations

import math

import numpy as np

BLUR_PASSES = 3


def nearest_table(in_size: int, out_size: int) -> np.ndarray:
    """source index per output pixel of one axis, −1 outside the source, accumulated as Pillow does"""
    a = float(in_size) / out_size
    xo = a * 0.5
    tab = np.empty(out_size, dtype=np.int64)
    for x in range(out_size):
        xi = -1 if xo < 0.0 else int(xo)
        tab[x] = xi if 0 <= xi < in_size else -1
        xo += a
    return tab


def resize_nearest(img: np.ndarray, size) -> np.ndarray:
    """size = (width, height) as PIL takes it"""
    out_w, out_h = int(size[0]), int(size[1])
    h, w = img.shape[:2]
    if (out_w, out_h) == (w, h):
        return img.copy()
    tx, ty = nearest_table(w, out_w), nearest_table(h, out_h)
    out = np.zeros((out_h, out_w) + img.shape[2:], dtype=np.uint8)
    ok = (ty[:, None] >= 0) & (tx[None, :] >= 0)
    out[ok] = img[np.clip(ty, 0, None)[:, None], np.clip(tx, 0, None)[None, :]][ok]
    return out


def window(img: np.ndarray, hw, dy: int, dx: int) -> np.ndarray:
    """the (h, w) window whose top-left corner is source pixel (dy, dx); 0 where it leaves the source"""
    oh, ow = int(hw[0]), int(hw[1])
    h, w = img.shape[:2]
    out = np.zeros((oh, ow) + img.shape[2:], dtype=np.uint8)
    y0, y1 = max(dy, 0), min(dy + oh, h)
    x0, x1 = max(dx, 0), min(dx + ow, w)
    if y0 < y1 and x0 < x1:
        out[y0 - dy:y1 - dy, x0 - dx:x1 - dx] = img[y0:y1, x0:x1]
    return out


def box_radius(r: float, passes: int = BLUR_PASSES) -> np.float32:
    """Pillow's `_gaussian_blur_radius`: the extended box radius of a Gaussian of radius r over `passes` box passes"""
    f = np.float32
    radius = f(r)                                              # the C entry takes a float
    sigma2 = radius * radius / f(passes)
    L = f(math.sqrt(12.0 * float(sigma2) + 1.0))
    l = f(math.floor((float(L) - 1.0) / 2.0))
    a = (f(2) * l + f(1)) * (l * (l + f(1)) - f(3) * sigma2)
    a = a / (f(6) * (sigma2 - (l + f(1)) * (l + f(1))))
    return l + a


def blur_params(r: float):
    """→ (radius, ww, fw) of `ImagingHorizontalBoxBlur` for `GaussianBlur(r)`; r == 0 → the identity (0, 2²⁴, 0)"""
    rad = box_radius(r) if r != 0 else np.float32(0)
    radius = int(rad)
    ww = int(np.float32(1 << 24) / (rad * np.float32(2) + np.float32(1)))
    fw = ((1 << 24) - (radius * 2 + 1) * ww) // 2
    return radius, ww, fw


def _box_pass(x: np.ndarray, radius: int, ww: int, fw: int, axis: int) -> np.ndarray:
    n = x.shape[axis]
    v = x.astype(np.uint64)
    idx = np.arange(n)

    def tap(k):
        return np.take(v, np.clip(idx + k, 0, n - 1), axis=axis)

    acc = sum(tap(k) for k in range(-radius, radius + 1))
    bulk = acc * np.uint64(ww) + (tap(-radius - 1) + tap(radius + 1)) * np.uint64(fw)
    return ((bulk + np.uint64(1 << 23)) >> np.uint64(24)).astype(np.uint8)


def gaussian_blur(img: np.ndarray, r: float) -> np.ndarray:
    if r == 0:
        return img.copy()
    radius, ww, fw = blur_params(r)
    x = img
    for axis in (1, 1, 1, 0, 0, 0):
        x = _box_pass(x, radius, ww, fw, axis)
    return x
