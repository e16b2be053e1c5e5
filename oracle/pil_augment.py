"""Oracle (TEST INFRASTRUCTURE, never imported by the product path): numpy restatement of the reference's random training
augmentation after `JointResize` (utils/joint_transforms.py:20-48, utils/dataset.py:86-95), for fixed parameters:

  1. `RandomHorizontallyFlip`: `FLIP_LEFT_RIGHT` of image and mask;
  2. `RandomRotate(10)`: `img.rotate(deg, BILINEAR)` ("RGB") and `mask.rotate(deg, NEAREST)` ("L"), no expand, fill 0;
  3. `ColorJitter(0.1, 0.1, 0.1)` on the image: brightness, contrast and saturation in a given order, each
     `Image.blend(degenerate, img, factor)`.

Pillow's `rotate` builds an output → input affine matrix in Python (`rotate_matrix`) and resamples in C
(libImaging/Geometry.c): BILINEAR through the generic transform in float64, NEAREST through 16.16 fixed point.  Every
float operation below is one numpy call in Pillow's order, so none can be fused.  `Image.blend` computes in float32.
"""
from __future__ import annotations

import math

import numpy as np

BRIGHTNESS, CONTRAST, SATURATION = 0, 1, 2     # torchvision's ColorJitter function ids


def rotate_matrix(angle: float, w: int, h: int):
    """→ (the 6 coefficients of Pillow's `Image.rotate(angle)` matrix, identity), identity meaning Pillow copies"""
    angle = angle % 360.0
    if angle == 0:
        return [1.0, 0.0, 0.0, 0.0, 1.0, 0.0], True
    cx, cy = w / 2, h / 2
    angle = -math.radians(angle)
    m = [round(math.cos(angle), 15), round(math.sin(angle), 15), 0.0, round(-math.sin(angle), 15), round(math.cos(angle), 15), 0.0]
    m[2], m[5] = m[0] * -cx + m[1] * -cy + m[2], m[3] * -cx + m[4] * -cy + m[5]
    m[2] += cx
    m[5] += cy
    return m, False


def rotate_bilinear(img: np.ndarray, m) -> np.ndarray:
    """img uint8 [H, W] or [H, W, C]: the generic affine transform with the bilinear filter, fill 0"""
    h, w = img.shape[:2]
    x3 = img if img.ndim == 3 else img[:, :, None]
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    xs, ys = xs + 0.5, ys + 0.5
    xin = m[0] * xs
    xin = xin + m[1] * ys
    xin = xin + m[2]
    yin = m[3] * xs
    yin = yin + m[4] * ys
    yin = yin + m[5]
    inside = (xin >= 0.0) & (xin < w) & (yin >= 0.0) & (yin < h)
    xin = xin - 0.5
    yin = yin - 0.5
    x = np.floor(xin).astype(np.int64)
    y = np.floor(yin).astype(np.int64)
    dx = (xin - x)[..., None]
    dy = (yin - y)[..., None]
    x0, x1 = np.clip(x, 0, w - 1), np.clip(x + 1, 0, w - 1)
    src = x3.astype(np.int64)
    yc = np.clip(y, 0, h - 1)
    a, b = src[yc, x0], src[yc, x1]
    v1 = a + (b - a) * dx
    has2 = ((y + 1 >= 0) & (y + 1 < h))[..., None]
    y2 = np.clip(y + 1, 0, h - 1)
    a2, b2 = src[y2, x0], src[y2, x1]
    v2 = np.where(has2, a2 + (b2 - a2) * dx, v1)
    v = v1 + (v2 - v1) * dy
    out = np.where(inside[..., None], v.astype(np.uint8), 0).astype(np.uint8)
    return out if img.ndim == 3 else out[:, :, 0]


def rotate_nearest(img: np.ndarray, m) -> np.ndarray:
    """img uint8 [H, W]: the affine transform with nearest neighbour in 16.16 fixed point, fill 0"""
    h, w = img.shape[:2]

    def fix(v):
        return math.floor(v * 65536.0 + 0.5)

    a0, a1, a3, a4 = fix(m[0]), fix(m[1]), fix(m[3]), fix(m[4])
    a2, a5 = fix(m[2] + m[0] * 0.5 + m[1] * 0.5), fix(m[5] + m[3] * 0.5 + m[4] * 0.5)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.int64)
    xin = (a2 + ys * a1 + xs * a0) >> 16
    yin = (a5 + ys * a4 + xs * a3) >> 16
    inside = (xin >= 0) & (xin < w) & (yin >= 0) & (yin < h)
    out = np.zeros_like(img)
    out[inside] = img[yin[inside], xin[inside]]
    return out


def luma(img: np.ndarray) -> np.ndarray:
    """`convert("L")` of an RGB image: ITU-R 601-2 in 16-bit fixed point"""
    c = img.astype(np.int64)
    return ((c[..., 0] * 19595 + c[..., 1] * 38470 + c[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def blend(degenerate: np.ndarray, img: np.ndarray, factor) -> np.ndarray:
    """`Image.blend(degenerate, img, factor)`: float32 d + f·(x − d), clipped to [0, 255] and truncated"""
    d = degenerate.astype(np.float32)
    t = d + np.float32(factor) * (img.astype(np.int32) - degenerate.astype(np.int32)).astype(np.float32)
    return np.clip(t, 0.0, 255.0).astype(np.uint8)


def jitter_op(img: np.ndarray, op: int, factor) -> np.ndarray:
    if op == BRIGHTNESS:
        return blend(np.zeros_like(img), img, factor)
    if op == CONTRAST:
        mean = int(int(luma(img).astype(np.int64).sum()) / (img.shape[0] * img.shape[1]) + 0.5)
        return blend(np.full_like(img, mean), img, factor)
    if op == SATURATION:
        return blend(np.repeat(luma(img)[..., None], 3, axis=2), img, factor)
    raise ValueError(op)


def augment(img: np.ndarray, mask: np.ndarray, flip: bool, angle: float, order, factors):
    """img uint8 [H, W, 3], mask uint8 [H, W], both after JointResize; `order` the three op ids in application order,
    `factors` (brightness, contrast, saturation) → (image, mask)"""
    if flip:
        img, mask = img[:, ::-1], mask[:, ::-1]
    m, ident = rotate_matrix(angle, img.shape[1], img.shape[0])
    if ident:
        img, mask = img.copy(), mask.copy()
    else:
        img, mask = rotate_bilinear(img, m), rotate_nearest(mask, m)
    for op in order:
        img = jitter_op(img, op, factors[op])
    return img, mask
