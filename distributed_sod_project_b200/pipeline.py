"""Input-pipeline seam (SURVEY §8f.2): what the reference's `ImageFolder` + `create_loader` hand to the training loop
(utils/dataset.py:72-156, consumed at train.py:284-292), with the tensor-side work on the GPU.

Reference, per sample on DataLoader workers: PIL decode → joint resize / flip / rotate → ColorJitter → ToTensor →
Normalize; then the collate function stacks fp32 tensors and — for multi-scale training — resizes the stacked batch
with `F.interpolate` (bilinear image, nearest mask) on the CPU; the fp32 batch (16 B per pixel) is pinned and copied.

Here only decoding stays on the workers and the batch stays uint8 until it is on the device: `preprocess_batch` is ONE
kernel (csrc/pipeline.cu) doing ToTensor, Normalize, the optional horizontal flip and the collate's resize, and writing
the image channels-last.  4 B per pixel cross PCIe instead of 16.  `DevicePrefetcher` is the
`BackgroundGenerator(tr_loader, max_prefetch=2)` of train.py:285 with a copy stream: batch k+1 is uploaded and
pre-processed while iteration k runs.  For on-disk training sets `TrainPrefetcher` also runs the reference's
JointResize (`resize_u8`) and flip / rotate / ColorJitter (`augment_u8`) on the GPU, bit for bit as Pillow computes them,
or a configured chain of the reference's joint transforms (`parse_joint_transforms`: RandomScaleCrop, ScaleCenterCrop,
PaddingSquare and RandomGaussianBlur too, with `resize_nearest_u8`, `window_u8` and `gaussian_blur_u8`).
"""
from __future__ import annotations

import ctypes as C
import math
import random
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib

IMAGENET_MEAN = (0.485, 0.456, 0.406)     # utils/dataset.py:92
IMAGENET_STD = (0.229, 0.224, 0.225)


def preprocess_batch(img_u8: torch.Tensor, mask_u8: torch.Tensor | None = None, size: int | tuple[int, int] | None = None,
                     flip: torch.Tensor | None = None, dtype: torch.dtype = torch.float32,
                     mean=IMAGENET_MEAN, std=IMAGENET_STD):
    """img_u8 [N,H,W,3] uint8 (HWC, as PIL/numpy produce it), mask_u8 [N,H,W] uint8 or None, both on the GPU.
    Returns (image [N,3,S,S] `dtype`, channels-last; mask [N,1,S,S] fp32 or None): exactly
    `Normalize(ToTensor(img))` / `ToTensor(mask)` followed by the multi-scale collate's `interpolate` to `size`
    (utils/dataset.py:86-96,110-116,125-132).  `flip` (uint8 [N] on the GPU): mirror sample i left-right first."""
    if not img_u8.is_cuda:
        raise _lib.SodError("preprocess_batch needs CUDA tensors (no CPU fallback; keep torchvision transforms for CPU runs)")
    if img_u8.dtype != torch.uint8 or img_u8.dim() != 4 or img_u8.shape[-1] != 3:
        raise ValueError("img_u8 must be uint8 [N,H,W,3]")
    img_u8 = img_u8.contiguous()
    n, hs, ws, _ = img_u8.shape
    ho, wo = (hs, ws) if size is None else ((size, size) if isinstance(size, int) else tuple(size))
    out = torch.empty((n, ho, wo, 3), dtype=dtype, device=img_u8.device)
    m_out = None
    if mask_u8 is not None:
        if mask_u8.dtype != torch.uint8 or tuple(mask_u8.shape[-2:]) != (hs, ws) or mask_u8.numel() != n * hs * ws:
            raise ValueError("mask_u8 must be uint8 [N,H,W] matching the images")
        mask_u8 = mask_u8.contiguous()
        m_out = torch.empty((n, 1, ho, wo), dtype=torch.float32, device=img_u8.device)
    if flip is not None:
        flip = flip.to(device=img_u8.device, dtype=torch.uint8).contiguous()
        if flip.numel() != n:
            raise ValueError("flip must hold one flag per sample")
    rc = _lib.lib().sod_preprocess_batch(
        img_u8.data_ptr(), mask_u8.data_ptr() if mask_u8 is not None else None, flip.data_ptr() if flip is not None else None,
        out.data_ptr(), _lib.dtype_code(dtype), m_out.data_ptr() if m_out is not None else None, n, hs, ws, ho, wo,
        (C.c_float * 3)(*mean), (C.c_float * 3)(*std), _lib.stream_ptr())
    _lib.check(rc, "sod_preprocess_batch")
    _lib.count_launch()
    return out.permute(0, 3, 1, 2), m_out          # logical NCHW over channels-last storage


class Ragged:
    """A batch of uint8 images of different sizes, packed back to back with no padding: `data` (flat, CUDA), `hw`
    (int32 [n, 2] on the host), `channels` (1: "L" [h, w]; 3: "RGB" [h, w, 3]), and the device copies of the byte
    offsets and sizes that the kernels read."""

    def __init__(self, data: torch.Tensor, hw: torch.Tensor, channels: int):
        self.hw = hw.to(torch.int32).reshape(-1, 2).contiguous()
        self.channels = channels
        sizes = self.hw[:, 0].long() * self.hw[:, 1].long() * channels
        self.off = torch.cumsum(sizes, 0) - sizes                    # int64 [n], host
        if data.numel() != int(sizes.sum()):
            raise ValueError(f"ragged batch: {data.numel()} bytes for images of {int(sizes.sum())}")
        self.data = data.reshape(-1)
        dev = data.device
        self.off_d = self.off.to(dev, non_blocking=True)
        self.hw_d = self.hw.to(dev, non_blocking=True)

    @classmethod
    def empty(cls, hw: torch.Tensor, channels: int, device) -> "Ragged":
        hw = hw.to(torch.int32).reshape(-1, 2)
        n_bytes = int((hw[:, 0].long() * hw[:, 1].long()).sum()) * channels
        return cls(torch.empty(n_bytes, dtype=torch.uint8, device=device), hw, channels)

    @classmethod
    def stack(cls, images: torch.Tensor) -> "Ragged":
        """equal-size images uint8 [n, h, w] or [n, h, w, 3]"""
        ch = 1 if images.dim() == 3 else images.shape[-1]
        n, h, w = images.shape[:3]
        return cls(images.contiguous().reshape(-1), torch.tensor([[h, w]] * n, dtype=torch.int32), ch)

    def __len__(self) -> int:
        return self.hw.shape[0]

    def image(self, i: int) -> torch.Tensor:
        h, w = int(self.hw[i, 0]), int(self.hw[i, 1])
        o = int(self.off[i])
        v = self.data[o:o + h * w * self.channels]
        return v.view(h, w) if self.channels == 1 else v.view(h, w, self.channels)

    def as_batch(self) -> torch.Tensor:
        """view of an equal-size batch as [n, h, w] or [n, h, w, 3]"""
        h, w = int(self.hw[0, 0]), int(self.hw[0, 1])
        if not bool((self.hw == self.hw[0]).all()):
            raise ValueError("as_batch needs images of one size")
        return self.data.view(len(self), h, w) if self.channels == 1 else self.data.view(len(self), h, w, self.channels)


def resize_u8(src: Ragged, hw, resample: int = _lib.SOD_RESIZE_BICUBIC) -> Ragged:
    """Pillow's `Image.resize((w, h), resample)` (BILINEAR or BICUBIC, whole image, no reducing_gap) of every image of
    `src` to its size in `hw` (int32 [n, 2] or one (h, w) for all), bit for bit, in one batched call
    (csrc/resize.cu).  The reference uses it on predictions (`.resize(gt.size)`: BICUBIC, train.py:392-395) and, through
    torchvision `Resize((S, S))`, on test images (BILINEAR, utils/dataset.py:97-104)."""
    if not src.data.is_cuda:
        raise _lib.SodError("resize_u8 needs CUDA tensors (no CPU fallback)")
    hw = torch.as_tensor(hw, dtype=torch.int32)
    if hw.dim() == 1:
        hw = hw[None].expand(len(src), 2)
    hw = hw.contiguous()
    if hw.shape != (len(src), 2) or bool((hw <= 0).any()):
        raise ValueError("resize_u8: one positive (h, w) per image")
    out = Ragged.empty(hw, src.channels, src.data.device)
    lib = _lib.lib()
    ws_bytes = lib.sod_resize_u8_workspace_bytes(len(src), src.hw.data_ptr(), hw.data_ptr(), src.channels, resample)
    if ws_bytes == 0:
        raise _lib.SodError(f"sod_resize_u8: unsupported channels={src.channels} / resample={resample}")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=src.data.device)
    rc = lib.sod_resize_u8(src.data.data_ptr(), src.off_d.data_ptr(), src.hw_d.data_ptr(), out.data.data_ptr(),
                           out.off_d.data_ptr(), out.hw_d.data_ptr(), len(src), src.channels, resample, ws.data_ptr(),
                           ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "sod_resize_u8")
    _lib.count_launch(3)
    return out


@dataclass
class AugmentParams:
    """per-sample parameters of the reference's training augmentation for a batch of `size`² samples: `flip` (bool),
    `angle` (degrees, as `RandomRotate` draws it), `order` (the three ColorJitter op ids — 0 brightness, 1 contrast,
    2 saturation — in application order) and `factor` (float32 brightness, contrast, saturation factors)"""
    size: int
    flip: list
    angle: list
    order: list
    factor: list

    def __len__(self) -> int:
        return len(self.flip)

    def c_array(self):
        arr = (_lib.sod_augment_param * len(self))()
        for i, p in enumerate(arr):
            m, ident = rotate_matrix(self.angle[i], self.size, self.size)
            p.rot[:] = m
            p.flip, p.identity = int(bool(self.flip[i])), int(ident)
            p.ops[:] = [int(o) for o in self.order[i]]
            p.factor[:] = [float(f) for f in self.factor[i]]
        return arr


def rotate_matrix(angle: float, w: int, h: int):
    """Pillow's `Image.rotate(angle)` (no expand, centre, translate) output → input affine matrix, computed with
    Pillow's own formula → (6 coefficients, identity); identity when `angle % 360 == 0`, where Pillow copies"""
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


def draw_augment_params(n: int, size: int, rng: torch.Generator) -> AugmentParams:
    """the reference's random draws for n samples, from `rng`: flip with probability 0.5 (`RandomHorizontallyFlip`),
    angle = U[0, 1)·2·10 − 10 (`RandomRotate(10)`), a uniformly random order of brightness / contrast / saturation
    (torchvision's `randperm(4)` with hue absent) and three factors U[0.9, 1.1] in float32 (`ColorJitter(0.1, 0.1, 0.1)`)"""
    flip = (torch.rand(n, generator=rng, dtype=torch.float64) < 0.5).tolist()
    angle = [r * 2 * 10 - 10 for r in torch.rand(n, generator=rng, dtype=torch.float64).tolist()]
    order = torch.rand(n, 3, generator=rng).argsort(dim=1).tolist()
    factor = torch.empty(n, 3).uniform_(0.9, 1.1, generator=rng).tolist()
    return AugmentParams(size, flip, angle, order, factor)


def augment_u8(img_u8: torch.Tensor, mask_u8: torch.Tensor, params: AugmentParams):
    """the reference's `RandomHorizontallyFlip` → `RandomRotate(10)` → `ColorJitter(0.1, 0.1, 0.1)` on equal-size
    batches, img_u8 uint8 [n, S, S, 3] and mask_u8 uint8 [n, S, S] on the GPU, bit for bit as Pillow and torchvision
    compute them, with the parameters of `params` (csrc/augment.cu) → new (image, mask) tensors"""
    if not img_u8.is_cuda:
        raise _lib.SodError("augment_u8 needs CUDA tensors (no CPU fallback)")
    n, s = len(params), params.size
    if img_u8.dtype != torch.uint8 or tuple(img_u8.shape) != (n, s, s, 3):
        raise ValueError(f"img_u8 must be uint8 [{n}, {s}, {s}, 3]")
    if mask_u8.dtype != torch.uint8 or tuple(mask_u8.shape) != (n, s, s) or mask_u8.device != img_u8.device:
        raise ValueError(f"mask_u8 must be uint8 [{n}, {s}, {s}] on the images' device")
    img_u8, mask_u8 = img_u8.contiguous(), mask_u8.contiguous()
    img_out, mask_out = torch.empty_like(img_u8), torch.empty_like(mask_u8)
    lib = _lib.lib()
    ws_bytes = lib.sod_augment_u8_workspace_bytes(n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=img_u8.device)
    rc = lib.sod_augment_u8(img_u8.data_ptr(), mask_u8.data_ptr(), img_out.data_ptr(), mask_out.data_ptr(), n, s,
                            params.c_array(), ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "sod_augment_u8")
    _lib.count_launch(2)
    return img_out, mask_out


def resize_nearest_u8(src: Ragged, hw) -> Ragged:
    """Pillow's `Image.resize((w, h), NEAREST)` of every image of `src` to its size in `hw` (int32 [n, 2] or one (h, w)
    for all), bit for bit (csrc/joint.cu): the mask resize of `RandomScaleCrop` and `ScaleCenterCrop`"""
    if not src.data.is_cuda:
        raise _lib.SodError("resize_nearest_u8 needs CUDA tensors (no CPU fallback)")
    hw = torch.as_tensor(hw, dtype=torch.int32)
    if hw.dim() == 1:
        hw = hw[None].expand(len(src), 2)
    hw = hw.contiguous()
    if hw.shape != (len(src), 2) or bool((hw <= 0).any()):
        raise ValueError("resize_nearest_u8: one positive (h, w) per image")
    out = Ragged.empty(hw, src.channels, src.data.device)
    lib = _lib.lib()
    ws_bytes = lib.sod_resize_nearest_u8_workspace_bytes(len(src), src.hw.data_ptr(), hw.data_ptr(), src.channels)
    if ws_bytes == 0:
        raise _lib.SodError(f"sod_resize_nearest_u8: unsupported channels={src.channels}")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=src.data.device)
    rc = lib.sod_resize_nearest_u8(src.data.data_ptr(), src.off_d.data_ptr(), src.hw_d.data_ptr(), out.data.data_ptr(),
                                   out.off_d.data_ptr(), out.hw_d.data_ptr(), src.hw.data_ptr(), hw.data_ptr(), len(src),
                                   src.channels, ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "sod_resize_nearest_u8")
    _lib.count_launch(2)
    return out


def window_u8(src: Ragged, hw, offset) -> Ragged:
    """the (h, w) window (`hw`: int32 [n, 2] or one (h, w)) of every image of `src` whose top-left corner is source pixel
    `offset` (int32 [n, 2] rows, columns; may be negative), zeros outside the source (csrc/joint.cu): `Image.crop` of
    `RandomScaleCrop` / `ScaleCenterCrop` and the centred zero padding of `PaddingSquare`"""
    if not src.data.is_cuda:
        raise _lib.SodError("window_u8 needs CUDA tensors (no CPU fallback)")
    hw = torch.as_tensor(hw, dtype=torch.int32)
    if hw.dim() == 1:
        hw = hw[None].expand(len(src), 2)
    hw = hw.contiguous()
    offset = torch.as_tensor(offset, dtype=torch.int32).reshape(-1, 2).contiguous()
    if hw.shape != (len(src), 2) or offset.shape != (len(src), 2) or bool((hw <= 0).any()):
        raise ValueError("window_u8: one positive (h, w) and one (dy, dx) per image")
    out = Ragged.empty(hw, src.channels, src.data.device)
    lib = _lib.lib()
    ws_bytes = lib.sod_window_u8_workspace_bytes(len(src))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=src.data.device)
    rc = lib.sod_window_u8(src.data.data_ptr(), src.off_d.data_ptr(), src.hw_d.data_ptr(), out.data.data_ptr(),
                           out.off_d.data_ptr(), out.hw_d.data_ptr(), hw.data_ptr(), offset.data_ptr(), len(src),
                           src.channels, ws.data_ptr(), ws_bytes, _lib.stream_ptr())
    _lib.check(rc, "sod_window_u8")
    _lib.count_launch()
    return out


def blur_param(r: float):
    """Pillow's box parameters (radius, ww, fw) of `ImageFilter.GaussianBlur(r)` with its three passes
    (libImaging/BoxBlur.c `_gaussian_blur_radius` and `ImagingHorizontalBoxBlur`), in Pillow's float32 arithmetic;
    r == 0 (Pillow copies) and radii too small to change a pixel give the identity (0, 2²⁴, 0)"""
    f = np.float32
    if r == 0:
        rad = f(0)
    else:
        radius = f(r)                                          # GaussianBlur hands C a float
        sigma2 = radius * radius / f(3)
        L = f(math.sqrt(12.0 * float(sigma2) + 1.0))           # promoted to double, stored as float
        l = f(math.floor((float(L) - 1.0) / 2.0))
        a = (f(2) * l + f(1)) * (l * (l + f(1)) - f(3) * sigma2)
        a = a / (f(6) * (sigma2 - (l + f(1)) * (l + f(1))))
        rad = l + a
    ww = int(f(1 << 24) / (rad * f(2) + f(1)))
    return int(rad), ww, ((1 << 24) - (int(rad) * 2 + 1) * ww) // 2


def gaussian_blur_u8(img_u8: torch.Tensor, radius) -> torch.Tensor:
    """`img.filter(ImageFilter.GaussianBlur(r))` of every image of an equal-size batch, img_u8 uint8 [n, h, w, 3] or
    [n, h, w] on the GPU, one r per image (`radius`), bit for bit as Pillow computes it (csrc/joint.cu) → new tensor"""
    if not img_u8.is_cuda:
        raise _lib.SodError("gaussian_blur_u8 needs CUDA tensors (no CPU fallback)")
    if img_u8.dtype != torch.uint8 or img_u8.dim() not in (3, 4) or (img_u8.dim() == 4 and img_u8.shape[-1] != 3):
        raise ValueError("img_u8 must be uint8 [n, h, w, 3] or [n, h, w]")
    n, h, w = img_u8.shape[:3]
    ch = 1 if img_u8.dim() == 3 else 3
    if len(radius) != n:
        raise ValueError("gaussian_blur_u8: one radius per image")
    prm = (_lib.sod_blur_param * n)()
    for p, r in zip(prm, radius):
        p.radius, p.ww, p.fw = blur_param(float(r))
    img_u8 = img_u8.contiguous()
    out = torch.empty_like(img_u8)
    lib = _lib.lib()
    ws_bytes = lib.sod_gaussian_blur_u8_workspace_bytes(n, h, w, ch)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=img_u8.device)
    rc = lib.sod_gaussian_blur_u8(img_u8.data_ptr(), out.data_ptr(), n, h, w, ch, prm, ws.data_ptr(), ws_bytes,
                                  _lib.stream_ptr())
    _lib.check(rc, "sod_gaussian_blur_u8")
    _lib.count_launch(6)
    return out


# ---- the configurable joint-transform chain ------------------------------------------------------------------------
SIZE_STEPS = ("JointResize", "ScaleCenterCrop", "PaddingSquare")
_STAGE = {"JointResize": 0, "ScaleCenterCrop": 0, "PaddingSquare": 0, "RandomScaleCrop": 1, "RandomHorizontallyFlip": 2,
          "RandomRotate": 3, "RandomGaussianBlur": 4}
_ARGS = {"JointResize": ("size",), "ScaleCenterCrop": ("input_size",), "PaddingSquare": ("pad_size",),
         "RandomScaleCrop": ("input_size", "scale_factor"), "RandomHorizontallyFlip": (), "RandomRotate": ("degree",),
         "RandomGaussianBlur": ()}
JOINT_ORDER = ("exactly one size step first (JointResize | ScaleCenterCrop | PaddingSquare), then optionally "
               "RandomScaleCrop, then RandomHorizontallyFlip, RandomRotate and RandomGaussianBlur, each optional, in "
               "that order")


def default_joint_transforms(size: int) -> list:
    """the reference's chain (utils/dataset.py:87): JointResize(size) → RandomHorizontallyFlip → RandomRotate(10)"""
    return [["JointResize", size], ["RandomHorizontallyFlip"], ["RandomRotate", 10]]


def parse_joint_transforms(chain, size: int) -> list:
    """validate a `joint_transforms` list of [name, *args] entries (None: the reference's chain) for `size`² samples →
    the entries as [name, *args] lists.  Raises ValueError naming the offending entry."""
    if chain is None:
        return default_joint_transforms(size)
    if not isinstance(chain, (list, tuple)) or not chain:
        raise ValueError(f"joint_transforms must be a non-empty list of [name, *args] entries: {JOINT_ORDER}")
    out, stage, side = [], -1, None                       # side: the square side the chain has made so far
    for i, entry in enumerate(chain):
        where = f"joint_transforms[{i}] = {entry!r}"
        if not isinstance(entry, (list, tuple)) or not entry or entry[0] not in _STAGE:
            raise ValueError(f"{where}: not a known transform ({', '.join(_STAGE)}); accepted order: {JOINT_ORDER}")
        name, args = entry[0], list(entry[1:])
        if len(args) != len(_ARGS[name]):
            raise ValueError(f"{where}: {name} takes ({', '.join(_ARGS[name])}); accepted order: {JOINT_ORDER}")
        if (i == 0) != (_STAGE[name] == 0) or _STAGE[name] <= stage:
            raise ValueError(f"{where}: out of order; accepted order: {JOINT_ORDER}")
        for a, v in zip(_ARGS[name], args):
            if a in ("size", "input_size", "pad_size") and (isinstance(v, bool) or not isinstance(v, int) or v <= 0):
                raise ValueError(f"{where}: {a} must be a positive int")
            if a in ("scale_factor", "degree") and (isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v)):
                raise ValueError(f"{where}: {a} must be a finite number")
        if name == "RandomScaleCrop":
            if args[0] != side:
                raise ValueError(f"{where}: RandomScaleCrop needs a square input of its input_size {args[0]}, the chain "
                                 f"before it makes {side}²")
            if int(args[0] * args[1]) < args[0]:
                raise ValueError(f"{where}: scale_factor must be at least 1")
        if _STAGE[name] <= 1:
            side = args[0]
            if side != size:
                raise ValueError(f"{where}: makes {side}² samples but input_size is {size}; accepted order: {JOINT_ORDER}")
        stage = _STAGE[name]
        out.append([name, *args])
    return out


@dataclass
class JointParams:
    """per-sample draws of a joint-transform chain: `augment` (flip / rotate / jitter, as `draw_augment_params`),
    `crop` ((o, x1, y1) of `RandomScaleCrop` per sample, or None) and `blur` (the radius of `RandomGaussianBlur` per
    sample, 0.0 where it does not blur, or None)"""
    augment: AugmentParams
    crop: list | None
    blur: list | None


def draw_joint_params(n: int, chain: list, rng: torch.Generator) -> JointParams:
    """the draws of a parsed chain for n samples.  The reference chain's draws come first, in `draw_augment_params`'s
    order (flip, angle, jitter order, jitter factors), whether or not the chain flips or rotates, with the angle
    r·2·degree − degree; so a chain that only adds steps keeps the reference chain's flips, angles and jitter.  Then
    `RandomScaleCrop(S, f)`: a float64 U[0, 1) triple per sample, mapped to the inclusive integers o ∈ [S, int(S·f)],
    x1 ∈ [0, o − S], y1 ∈ [0, o − S] in that order; then `RandomGaussianBlur`: n float64 draws for "blur with probability
    0.5", then n radii U[0, 1) in float64."""
    steps = {e[0]: e[1:] for e in chain}
    size = chain[-1][1] if chain[-1][0] == "RandomScaleCrop" else chain[0][1]
    flip = (torch.rand(n, generator=rng, dtype=torch.float64) < 0.5).tolist()
    r = torch.rand(n, generator=rng, dtype=torch.float64).tolist()
    order = torch.rand(n, 3, generator=rng).argsort(dim=1).tolist()
    factor = torch.empty(n, 3).uniform_(0.9, 1.1, generator=rng).tolist()
    if "RandomHorizontallyFlip" not in steps:
        flip = [False] * n
    if "RandomRotate" in steps:
        degree = steps["RandomRotate"][0]
        angle = [v * 2 * degree - degree for v in r]
    else:
        angle = [0.0] * n
    crop = blur = None
    if "RandomScaleCrop" in steps:
        s, f = steps["RandomScaleCrop"]
        crop = []
        for u0, u1, u2 in torch.rand(n, 3, generator=rng, dtype=torch.float64).tolist():
            o = s + math.floor(u0 * (int(s * f) - s + 1))
            crop.append((o, math.floor(u1 * (o - s + 1)), math.floor(u2 * (o - s + 1))))
    if "RandomGaussianBlur" in steps:
        on = (torch.rand(n, generator=rng, dtype=torch.float64) < 0.5).tolist()
        radius = torch.rand(n, generator=rng, dtype=torch.float64).tolist()
        blur = [rr if b else 0.0 for b, rr in zip(on, radius)]
    return JointParams(AugmentParams(size, flip, angle, order, factor), crop, blur)


def scale_center_crop_geometry(h: int, w: int, s: int):
    """`ScaleCenterCrop(s)` of an h × w image → ((oh, ow) of the resize, (y1, x1) of the crop), with the reference's
    `int(1.0·w·oh/h)` and `int(round((w − s)/2.0))` (Python's round: half to even)"""
    if w > h:
        oh, ow = s, int(1.0 * w * s / h)
    else:
        ow, oh = s, int(1.0 * h * s / w)
    return (oh, ow), (int(round((oh - s) / 2.0)), int(round((ow - s) / 2.0)))


def padding_square_geometry(h: int, w: int):
    """`PaddingSquare` of an h × w image → (side, (dy, dx)): the image sits at ((side − h) // 2, (side − w) // 2) of a
    zero side × side square, side = max(h, w), i.e. the window of the image at minus those offsets"""
    side = max(h, w)
    return side, (-((side - h) // 2), -((side - w) // 2))


def joint_size_step(entry, img: Ragged, mask: Ragged):
    """the chain's size step on ragged image and mask batches of equal sizes → (image, mask) Ragged batches of S²"""
    name, s = entry[0], entry[1]
    hw = img.hw.tolist()
    if name == "JointResize":                              # Pillow's default BICUBIC for both
        return (resize_u8(img, (s, s), _lib.SOD_RESIZE_BICUBIC), resize_u8(mask, (s, s), _lib.SOD_RESIZE_BICUBIC))
    if name == "ScaleCenterCrop":                          # BILINEAR image, NEAREST mask, centre crop
        geo = [scale_center_crop_geometry(h, w, s) for h, w in hw]
        ohw, off = [g[0] for g in geo], [g[1] for g in geo]
        img = resize_u8(img, ohw, _lib.SOD_RESIZE_BILINEAR)
        mask = resize_nearest_u8(mask, ohw)
        return window_u8(img, (s, s), off), window_u8(mask, (s, s), off)
    # PaddingSquare: zero-pad to a square, then Image.resize's default BICUBIC for the image AND the mask
    geo = [padding_square_geometry(h, w) for h, w in hw]
    side, off = [[g[0], g[0]] for g in geo], [g[1] for g in geo]
    img, mask = window_u8(img, side, off), window_u8(mask, side, off)
    return (resize_u8(img, (s, s), _lib.SOD_RESIZE_BICUBIC), resize_u8(mask, (s, s), _lib.SOD_RESIZE_BICUBIC))


def random_scale_crop(img: Ragged, mask: Ragged, crop) -> tuple[Ragged, Ragged]:
    """`RandomScaleCrop` on S² batches with drawn (o, x1, y1) per sample: BILINEAR image / NEAREST mask to o², then the
    S² window at (y1, x1)"""
    s = int(img.hw[0, 0])
    ohw = [[o, o] for o, _, _ in crop]
    off = [[y1, x1] for _, x1, y1 in crop]
    img = resize_u8(img, ohw, _lib.SOD_RESIZE_BILINEAR)
    mask = resize_nearest_u8(mask, ohw)
    return window_u8(img, (s, s), off), window_u8(mask, (s, s), off)


def joint_chain_u8(chain: list, jp: JointParams, img: Ragged, mask: Ragged):
    """a parsed chain with its draws `jp` on ragged image / mask batches of equal sizes, then ColorJitter → (image uint8
    [n, S, S, 3], mask uint8 [n, S, S]): the size step and RandomScaleCrop on ragged batches, then flip / rotate with the
    jitter (one `augment_u8`), or, when the chain blurs, flip / rotate with jitter factors 1.0 (a byte identity), the
    blur, and the jitter alone with the identity rotation, as the reference jitters the blurred image"""
    img, mask = joint_size_step(chain[0], img, mask)
    if jp.crop is not None:
        img, mask = random_scale_crop(img, mask, jp.crop)
    img, mask = img.as_batch(), mask.as_batch()
    a = jp.augment
    if jp.blur is None:
        return augment_u8(img, mask, a)
    n = len(a)
    img, mask = augment_u8(img, mask, AugmentParams(a.size, a.flip, a.angle, a.order, [[1.0] * 3] * n))
    img = gaussian_blur_u8(img, jp.blur)
    return augment_u8(img, mask, AugmentParams(a.size, [False] * n, [0.0] * n, a.order, a.factor))


class DevicePrefetcher:
    """Wraps an iterable of host batches `(img_u8 [N,H,W,3], mask_u8 [N,H,W], names)` (pinned or not) and yields
    device batches `(image, mask, names)` in the training format, one batch ahead: upload + `preprocess_batch` of batch
    k+1 run on a side stream while the caller trains on batch k (the reference prefetches on a host thread,
    train.py:285; dead `DataPrefetcher`, utils/useful_but_dont_use.py:61-105, is the same idea).

    `size_list`: the multi-scale training sizes (config.py `size_list`); one size per batch, drawn from a generator
    seeded identically on every rank — the reference's collate draws with the worker's `random` module
    (utils/dataset.py:126), which is only consistent across ranks by accident of seeding."""

    def __init__(self, loader, size_list=None, dtype: torch.dtype = torch.float32, seed: int = 0, flip_prob: float = 0.0,
                 device: torch.device | None = None):
        self.loader, self.size_list, self.dtype, self.flip_prob = loader, size_list, dtype, flip_prob
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.rng = random.Random(seed)
        self.stream = torch.cuda.Stream(device=self.device)

    def __len__(self):
        return len(self.loader)

    def _stage(self, batch):
        img, mask, names = batch
        size = self.rng.choice(self.size_list) if self.size_list else None
        with torch.cuda.stream(self.stream):
            img_d = img.to(self.device, non_blocking=True)
            mask_d = mask.to(self.device, non_blocking=True)
            flip = None
            if self.flip_prob > 0:
                flip = torch.tensor([self.rng.random() < self.flip_prob for _ in range(img.shape[0])], dtype=torch.uint8).to(self.device, non_blocking=True)
            x, m = preprocess_batch(img_d, mask_d, size=size, flip=flip, dtype=self.dtype)
            ready = torch.cuda.Event()
            ready.record(self.stream)
        return x, m, names, ready, (img_d, mask_d)

    def __iter__(self):
        it = iter(self.loader)
        try:
            nxt = self._stage(next(it))
        except StopIteration:
            return
        while nxt is not None:
            x, m, names, ready, keep = nxt
            try:
                nxt = self._stage(next(it))          # queue the next upload before handing this batch out
            except StopIteration:
                nxt = None
            torch.cuda.current_stream().wait_event(ready)
            for t in (x, m, *keep):
                t.record_stream(torch.cuda.current_stream())
            yield x, m, names


class TrainPrefetcher(DevicePrefetcher):
    """`DevicePrefetcher` for on-disk training sets: wraps a DataLoader of ragged `data.EvalBatch` batches (decoded at
    the original size) and runs the reference's whole per-sample chain on the side stream, one batch ahead: H2D,
    `JointResize(size)` (Pillow BICUBIC for image and mask, `resize_u8`), flip / rotate / ColorJitter (`augment_u8`),
    then `preprocess_batch` (ToTensor, Normalize, the multi-scale collate; no flip).  Yields `(image, mask, names)`.

    `joint_transforms` (a list of [name, *args] entries, see `parse_joint_transforms`; None: the reference's chain)
    selects the joint transforms in place of JointResize → flip → rotate: a size step (JointResize, ScaleCenterCrop or
    PaddingSquare), optionally RandomScaleCrop, then flip, rotate and RandomGaussianBlur.  ColorJitter always follows.
    The reference's chain, given or not, runs exactly the code and draws above.

    Deviation from the reference, on purpose: the augmentation parameters are drawn in the main process from a generator
    seeded by (seed, epoch, rank) (`set_epoch`), not by each DataLoader worker's `random` state, so a run is reproducible
    whatever `num_workers` is.  The distributions are the reference's (`draw_augment_params`, `draw_joint_params`)."""

    def __init__(self, loader, size: int, size_list=None, dtype: torch.dtype = torch.float32, seed: int = 0, rank: int = 0,
                 device: torch.device | None = None, joint_transforms=None):
        super().__init__(loader, size_list=size_list, dtype=dtype, seed=seed, device=device)
        self.size, self.seed, self.rank = size, seed, rank
        self.chain = parse_joint_transforms(joint_transforms, size)
        self.default_chain = self.chain == default_joint_transforms(size)
        self.set_epoch(0)

    def set_epoch(self, epoch: int) -> None:
        """the sampler's shuffle and the drawn parameters of `epoch`; the multi-scale size sequence is the same on every rank"""
        sampler = getattr(self.loader, "sampler", None)
        if hasattr(sampler, "set_epoch"):
            sampler.set_epoch(epoch)
        self.rng.seed(self.seed + epoch)
        state = np.random.SeedSequence([self.seed, epoch, self.rank]).generate_state(2, dtype=np.uint32)
        self.gen = torch.Generator().manual_seed(int(state[0]) << 32 | int(state[1]))

    def _stage(self, batch):
        if not self.default_chain:
            return self._stage_chain(batch)
        size = self.rng.choice(self.size_list) if self.size_list else None
        params = draw_augment_params(len(batch), self.size, self.gen)
        with torch.cuda.stream(self.stream):
            img = Ragged(batch.img.to(self.device, non_blocking=True), batch.img_hw, 3)
            mask = Ragged(batch.gt.to(self.device, non_blocking=True), batch.gt_hw, 1)
            img = resize_u8(img, (self.size, self.size), _lib.SOD_RESIZE_BICUBIC).as_batch()
            mask = resize_u8(mask, (self.size, self.size), _lib.SOD_RESIZE_BICUBIC).as_batch()
            img, mask = augment_u8(img, mask, params)
            x, m = preprocess_batch(img, mask, size=size, dtype=self.dtype)
            ready = torch.cuda.Event()
            ready.record(self.stream)
        return x, m, batch.names, ready, ()

    def _stage_chain(self, batch):
        """`_stage` for a configured chain (`joint_chain_u8`)"""
        size = self.rng.choice(self.size_list) if self.size_list else None
        if not torch.equal(batch.img_hw, batch.gt_hw):
            raise ValueError(f"joint_transforms: image and mask sizes differ in {batch.names}")
        jp = draw_joint_params(len(batch), self.chain, self.gen)
        with torch.cuda.stream(self.stream):
            img = Ragged(batch.img.to(self.device, non_blocking=True), batch.img_hw, 3)
            mask = Ragged(batch.gt.to(self.device, non_blocking=True), batch.gt_hw, 1)
            img, mask = joint_chain_u8(self.chain, jp, img, mask)
            x, m = preprocess_batch(img, mask, size=size, dtype=self.dtype)
            ready = torch.cuda.Event()
            ready.record(self.stream)
        return x, m, batch.names, ready, ()
