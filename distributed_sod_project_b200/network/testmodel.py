"""`res50` / `cp_res50`: the TestModel plugin pair of the reference (network/TestModel.py:17-185), and
`wsgn_res50` / `cp_wsgn_res50`: the same models on the reference's weight-standardised GroupNorm ResNet-50
(`backbone.wsgn.from_wsgn.Backbone_ResNet50_in3`, the one-import swap in network/TestModel.py:11), and
`wsgn_resnext50` / `cp_wsgn_resnext50`: the same on its weight-standardised GroupNorm ResNeXt-50 32×4d
(`Backbone_ResNeXt50_in3`, built as `l_resnext50(pretrained, baseWidth=4, cardinality=32)`: the reference's builder
omits those two arguments, and its X-50-GN-WS release is 32×4d), and
`vgg16` / `cp_vgg16`: the same decoder on the reference's VGG16-BN (`backbone.origin.from_origin.Backbone_VGG16_in3`), whose
five slices carry 64 … 512 channels at strides 1 … 16.

Zero-arg factories looked up by name from `user_config["model"]` (reference train.py:141):
ResNet-50 encoder → five 1×1 "trans" convs to 64 ch → top-down decoder of SIM + ConvBNReLU with
bilinear upsample-add → 1×1 classifier → logits [N,1,H,W].

`cp_res50` wraps the same twelve segments in `torch.utils.checkpoint` (reference
network/TestModel.py:51-66): activations are recomputed in backward, so every BN forward — and,
distributed, its statistics exchange and running-stat update — runs twice per iteration (SURVEY Q3).
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.utils.checkpoint import checkpoint

from .blocks import (SIM, VGG16_SLICES, ConvBNReLU, WSConv2d, bilinear, group_norm32, resnet50_stages, upsample_add,
                     vgg16_bn_slices)

_TAPS = (32, 16, 8, 4, 2)                       # encoder strides tapped, deepest first
_TAP_CHANNELS = {32: 2048, 16: 1024, 8: 512, 4: 256, 2: 64}


class _TestModel(nn.Module):
    recompute = False  # cp_res50 flips this
    backbone = staticmethod(resnet50_stages)
    tap_channels = _TAP_CHANNELS                # channels of each backbone slice, keyed by its position name

    def __init__(self):
        super().__init__()
        self.div_2, self.div_4, self.div_8, self.div_16, self.div_32 = self.backbone()
        for s in _TAPS:
            setattr(self, f"trans{s}", nn.Conv2d(self.tap_channels[s], 64, 1, 1))
        for s in _TAPS:
            setattr(self, f"sim{s}", SIM(64, 32))
        for s in _TAPS:
            setattr(self, f"upconv{s}", ConvBNReLU(64, 32 if s == 2 else 64, 3, 1, 1))
        self.upconv1 = ConvBNReLU(32, 32, 3, 1, 1)
        self.classifier = nn.Conv2d(32, 1, 1)

    # -- segments (each is one checkpoint unit in cp_res50) -------------------------------------
    def _encode(self, stride: int, x):
        return getattr(self, f"div_{stride}")(x)

    def _project(self, f2, f4, f8, f16, f32):
        return self.trans2(f2), self.trans4(f4), self.trans8(f8), self.trans16(f16), self.trans32(f32)

    def _decode(self, stride: int, lateral, coarser=None):
        x = lateral if coarser is None else upsample_add(coarser, lateral)
        sim, up = getattr(self, f"sim{stride}"), getattr(self, f"upconv{stride}")
        return up(sim(x) + x)

    def _head(self, d2):
        return self.classifier(self.upconv1(bilinear(d2, scale_factor=2)))

    def _run(self, fn, *args):
        if self.recompute and torch.is_grad_enabled():
            # preserve_rng_state=False: the segments hold no dropout / RNG op, and saving the CUDA RNG state is not
            # allowed while a CUDA graph is being captured (the default config captures cp_res50 iterations)
            return checkpoint(fn, *args, use_reentrant=False, preserve_rng_state=False)
        return fn(*args)

    def forward(self, image: torch.Tensor) -> torch.Tensor:
        feats, x = {}, image
        for s in (2, 4, 8, 16, 32):
            x = self._run(lambda t, s=s: self._encode(s, t), x)
            feats[s] = x
        lat = dict(zip((2, 4, 8, 16, 32), self._run(self._project, *(feats[s] for s in (2, 4, 8, 16, 32)))))
        d = None
        for s in _TAPS:
            d = self._run(lambda a, b=None, s=s: self._decode(s, a, b), lat[s], *(() if d is None else (d,)))
        return self._run(self._head, d)


class res50(_TestModel):
    """Plain variant (reference network/TestModel.py:129-185)."""


class cp_res50(_TestModel):
    """Activation-checkpointed variant (reference network/TestModel.py:17-127)."""

    recompute = True


def _wsgn_backbone():
    return resnet50_stages(conv=WSConv2d, norm=group_norm32, imagenet_fc=True)


class wsgn_res50(_TestModel):
    """Plain variant on the weight-standardised GroupNorm(32) ResNet-50 (reference backbone/wsgn/from_wsgn.py:8-16):
    for micro-batch training, where per-GPU batches are too small for BatchNorm.  The decoder keeps BatchNorm."""

    backbone = staticmethod(_wsgn_backbone)


class cp_wsgn_res50(wsgn_res50):
    """Activation-checkpointed twin of `wsgn_res50`, as `cp_res50` is to `res50`."""

    recompute = True


def _wsgn_resnext_backbone():
    return resnet50_stages(conv=WSConv2d, norm=group_norm32, imagenet_fc=True, cardinality=32, base_width=4)


class wsgn_resnext50(_TestModel):
    """Plain variant on the weight-standardised GroupNorm(32) ResNeXt-50 32×4d (reference
    backbone/wsgn/from_wsgn.py:19-27, resnext.py): every bottleneck's 3x3 is a 32-group convolution."""

    backbone = staticmethod(_wsgn_resnext_backbone)


class cp_wsgn_resnext50(wsgn_resnext50):
    """Activation-checkpointed twin of `wsgn_resnext50`."""

    recompute = True


class vgg16(_TestModel):
    """Plain variant on VGG16-BN (reference backbone/origin/from_origin.py:18-25).  `div_2` … `div_32` name slice
    positions; their strides are 1, 2, 4, 8 and 16.  `div_2` is already at full resolution, so the head has no ×2
    up-sample."""

    backbone = staticmethod(vgg16_bn_slices)
    tap_channels = {32: 512, 16: 512, 8: 256, 4: 128, 2: 64}

    def _head(self, d2):
        return self.classifier(self.upconv1(d2))


class cp_vgg16(vgg16):
    """Activation-checkpointed twin of `vgg16`, with the same twelve segments as `cp_res50`."""

    recompute = True


_RESNET_REMAP = {"conv1.": "div_2.0.", "bn1.": "div_2.1.", "layer1.": "div_4.1.", "layer2.": "div_8.",
                 "layer3.": "div_16.", "layer4.": "div_32."}


def _resnet_remap(k: str) -> str | None:
    """torchvision / WS-GN ResNet key → `div_*` key by its first matching prefix, else None"""
    for old, new in _RESNET_REMAP.items():
        if k.startswith(old):
            return new + k[len(old):]
    return None


def _vgg_remap(k: str) -> str | None:
    """torchvision `vgg16_bn` key `features.{i}.*` → `div_*.{i - a}.*` of the slice that holds features[i], else None"""
    if not k.startswith("features."):
        return None
    idx, _, rest = k[len("features."):].partition(".")
    if not idx.isdigit():
        return None
    for name, (a, b) in zip(("div_2", "div_4", "div_8", "div_16", "div_32"), VGG16_SLICES):
        if a <= int(idx) < b:
            return f"{name}.{int(idx) - a}.{rest}"
    return None


def load_pretrained_backbone(model: _TestModel, path: str) -> list[str]:
    """Load ResNet-50 weights from a local file into `div_*` (the reference downloads them,
    backbone/origin/resnet.py:199-217 and backbone/wsgn/customized_func.py:32-43; no network here): torchvision's
    format, or the WS-GN release's — tensors under "state_dict", keys prefixed `module.` (stripped as the reference's
    `load_pretrained_params` does).  Keeps the reference's filter-then-update semantics: unknown keys are ignored.
    For `vgg16` / `cp_vgg16` it reads torchvision's `vgg16_bn` file: `features.{i}.*` goes to the slice holding
    features[i], `classifier.*` is ignored.  Returns loaded keys."""
    src = torch.load(path, map_location="cpu")
    if isinstance(src.get("state_dict"), dict):
        src = src["state_dict"]
    src = {k[len("module."):] if k.startswith("module.") else k: v for k, v in src.items()}
    rename = _vgg_remap if isinstance(model, vgg16) else _resnet_remap
    own = model.state_dict()
    picked = {}
    for k, v in src.items():
        nk = rename(k)
        if nk in own and own[nk].shape == v.shape:
            picked[nk] = v
    own.update(picked)
    model.load_state_dict(own)
    return sorted(picked)
