"""Building blocks of the TestModel plugin family (`res50`, `cp_res50`, and their WS-GN and VGG16-BN variants).

Written from scratch for this repo; the *contract* it keeps is the reference's
(lartpang/Distributed-SOD-Project):

* parameter / buffer names and registration order of `network/TestModel.py:17-185`,
  `module/BaseBlocks.py:10-40`, `module/MyLightModule.py:11-54`,
  `backbone/origin/resnet.py:61-156`, `backbone/origin/from_origin.py:7-15`
  (so reference checkpoints load, and `make_optimizer("f3_trick")` groups by the same
  `div_2` / `div*` prefixes, `utils/pipeline_ops.py:295-303`);
* RNG consumption order at construction, so that `init_seed(0)` followed by the factory call
  yields bit-identical initial weights to the reference (checked by
  tests/test_host_cpu.py::test_model_plugin_is_bit_identical_to_reference against vectors of the reference's model).

Every BatchNorm site goes through :func:`bn_act`, which is where the engine hooks in:
after `convert_syncbn_model` the BN modules expose `fused_forward`, and the (pre-add → BN →
residual-add → ReLU) chain becomes one hand-written sm_90a kernel instead of up to four
torch elementwise kernels.  On a stock `nn.BatchNorm2d` the same helper runs plain torch ops.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F


def bn_act(bn: nn.Module, x: torch.Tensor, *, relu: bool = True,
           pre_add: torch.Tensor | None = None, residual: torch.Tensor | None = None) -> torch.Tensor:
    """y = act( BN(x [+ pre_add]) [+ residual] ).

    pre_add  : the SIM pattern `relu(bn(a + b))` (reference module/MyLightModule.py:46-52)
    residual : the bottleneck pattern `relu(bn3(.) + identity)` (reference backbone/origin/resnet.py:87-94)
    """
    fused = getattr(bn, "fused_forward", None)
    if fused is not None:
        return fused(x, pre_add=pre_add, residual=residual, relu=relu)
    if pre_add is not None:
        x = x + pre_add
    y = bn(x)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


def _conv_nobias(conv: nn.Conv2d, x: torch.Tensor):
    """(conv(x) WITHOUT its bias, the bias tensor that has to be added later or None)"""
    if conv.bias is None:
        return conv(x), None
    if hasattr(conv, "_sod_w16") and torch.is_autocast_enabled() and x.is_cuda:    # bf16 shadow weights (amp.py)
        return conv._conv_forward(x, conv._sod_w16, None), conv._sod_b16
    return conv._conv_forward(x, conv.weight, None), conv.bias


def conv_bn_act(conv: nn.Conv2d, bn: nn.Module, x: torch.Tensor, *, relu: bool = True, pre=None,
                residual: torch.Tensor | None = None) -> torch.Tensor:
    """y = act( BN( conv(x) [+ pre_conv(pre_x)] ) [+ residual] ) with `pre = (pre_conv, pre_x)`.

    On the engine the convolution biases are not added by a separate elementwise pass (and their gradients not
    reduced by a separate kernel): the SyncBN kernel folds them in (`conv_bias=`) and its backward produces Σ dz."""
    fused = getattr(bn, "fused_forward", None)
    if fused is not None and x.is_cuda:
        a, b1 = _conv_nobias(conv, x)
        p, b2 = _conv_nobias(pre[0], pre[1]) if pre is not None else (None, None)
        return fused(a, pre_add=p, residual=residual, relu=relu, conv_bias=(b1, b2))
    return bn_act(bn, conv(x), relu=relu, pre_add=None if pre is None else pre[0](pre[1]), residual=residual)


# torch.autocast lists upsample_bilinear2d as an fp32 op: under bf16 autocast every interpolate becomes
# cast-up → fp32 kernel → fp32 result that then drags the following adds into fp32 (≈2 ms of casts per iteration on
# the TestModel).  The engine sets this flag so the interpolation runs natively in the activation dtype
# (the kernel still accumulates in fp32 internally; only the stored result is rounded to bf16).
INTERPOLATE_IN_ACTIVATION_DTYPE = False


def bilinear(x: torch.Tensor, **kw) -> torch.Tensor:
    """`cus_sample` of the reference (utils/tensor_ops.py:12-18): bilinear, align_corners=False."""
    if len(kw) != 1 or next(iter(kw)) not in ("size", "scale_factor"):
        raise ValueError("bilinear() takes exactly one of size= / scale_factor=")
    if x.is_cuda:
        from .. import resample                      # engine: deterministic channels-last ×2 kernel
        out_hw = kw["size"] if "size" in kw else ((int(x.shape[2] * kw["scale_factor"]), int(x.shape[3] * kw["scale_factor"]))
                                                  if kw["scale_factor"] == 2 else None)
        if out_hw is not None:
            y = resample.upsample2x(x, out_hw)
            if y is not None:
                return y
    if INTERPOLATE_IN_ACTIVATION_DTYPE and x.is_cuda and x.dtype != torch.float32 and torch.is_autocast_enabled():
        with torch.autocast("cuda", enabled=False):
            return F.interpolate(x, mode="bilinear", align_corners=False, **kw)
    return F.interpolate(x, mode="bilinear", align_corners=False, **kw)


def avgpool2(pool: nn.Module, x: torch.Tensor) -> torch.Tensor:
    """`h2l_pool` of the reference's SIM (module/MyLightModule.py:14): AvgPool2d((2,2), stride=2)"""
    if x.is_cuda:
        from .. import resample
        y = resample.avgpool2x2(x)
        if y is not None:
            return y
    return pool(x)


def upsample_add(*feats: torch.Tensor) -> torch.Tensor:
    """Sum of all inputs resized to the last one's spatial size (utils/tensor_ops.py:21-25)."""
    base = feats[-1]
    for f in feats[:-1]:
        fused = None
        if f.is_cuda:
            from .. import resample
            fused = resample.upsample2x_add(f, base)       # one kernel: bilinear ×2 of f, plus base
        base = fused if fused is not None else base + bilinear(f, size=base.shape[2:])
    return base


class ConvBNReLU(nn.Module):
    """Conv(bias=False) → BN → ReLU held in a 3-slot Sequential called `basicconv`
    (names `basicconv.0.weight`, `basicconv.1.{weight,bias}`; reference module/BaseBlocks.py:25-37)."""

    def __init__(self, cin: int, cout: int, kernel_size: int, stride: int = 1, padding: int = 0):
        super().__init__()
        self.basicconv = nn.Sequential(
            nn.Conv2d(cin, cout, kernel_size, stride, padding, bias=False),
            nn.BatchNorm2d(cout),
            nn.ReLU(inplace=True),
        )

    def forward(self, x):
        conv, bn, _ = self.basicconv
        return bn_act(bn, conv(x), relu=True)


class Bottleneck(nn.Module):
    """1x1 → 3x3(stride) → 1x1(×4) residual unit with the torchvision-v1 naming
    (`conv1,bn1,conv2,bn2,conv3,bn3,relu,downsample`), stride on the 3x3.

    With `cardinality` C > 1 it is the ResNeXt unit of the reference (backbone/wsgn/resnext.py:21-52): the inner width
    is D·C with D = floor(planes·base_width / 64), and the 3x3 is a C-group convolution."""

    expansion = 4

    def __init__(self, cin: int, planes: int, stride: int, shortcut: nn.Module | None, conv=nn.Conv2d,
                 norm=nn.BatchNorm2d, cardinality: int = 1, base_width: int = 64):
        super().__init__()
        width = int(math.floor(planes * (base_width / 64))) * cardinality
        cout = planes * self.expansion
        specs = ((cin, width, 1, 1, 0, 1), (width, width, 3, stride, 1, cardinality), (width, cout, 1, 1, 0, 1))
        for i, (ci, co, k, s, p, g) in enumerate(specs, start=1):
            setattr(self, f"conv{i}", conv(ci, co, k, s, p, bias=False) if g == 1 else
                    conv(ci, co, k, s, p, groups=g, bias=False))
            setattr(self, f"bn{i}", norm(co))
        self.relu = nn.ReLU(inplace=True)
        self.downsample = shortcut
        self.stride = stride

    def forward(self, x):
        skip = x
        y = bn_act(self.bn1, self.conv1(x))
        y = bn_act(self.bn2, self.conv2(y))
        if self.downsample is not None:
            proj_conv, proj_bn = self.downsample
            skip = bn_act(proj_bn, proj_conv(x), relu=False)
        return bn_act(self.bn3, self.conv3(y), residual=skip)


class _Stem(nn.Sequential):
    """conv7x7/2 → BN → ReLU == `div_2` (names `div_2.0.weight`, `div_2.1.*`)."""

    def forward(self, x):
        return bn_act(self[1], self[0](x))


class _StemPool(nn.MaxPool2d):
    """the ResNet stem's MaxPool2d(3, 2, 1); routed to csrc/maxpool.cu when that kernel is enabled (the default)"""

    def forward(self, x):
        from .. import resample
        y = resample.maxpool3x3s2(x) if (self.kernel_size, self.stride, self.padding, self.dilation, self.ceil_mode) == (3, 2, 1, 1, False) else None
        return y if y is not None else super().forward(x)


_RESNET50_STAGES = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))  # (width, blocks, stride)


def resnet50_stages(conv=nn.Conv2d, norm=nn.BatchNorm2d, imagenet_fc: bool = False, cardinality: int = 1,
                    base_width: int = 64) -> tuple[nn.Module, nn.Module, nn.Module, nn.Module, nn.Module]:
    """ResNet-50 encoder sliced into the five strides the decoder taps
    (reference backbone/origin/from_origin.py:7-15): div_2 = stem, div_4 = maxpool+layer1,
    div_8/16/32 = layer2/3/4.  Random init only (no network in this environment; the reference
    would download ImageNet weights, backbone/origin/resnet.py:199-217) — use
    `load_pretrained_backbone` for a local file.

    `conv` / `norm` build every convolution (called as `conv(cin, cout, k, stride, padding, bias=False)`) and every
    normalisation layer (`norm(channels)`).  `imagenet_fc`: also build (and drop) the 2048→1000 classifier the
    weight-standardised ResNet constructs before its init loop (backbone/wsgn/resnet.py:105-107), so the random draws
    after it are the reference's.

    `cardinality` > 1 builds ResNeXt-50 (cardinality × base_width d) instead, with the reference ResNeXt's init
    expression `normal_(0, math.sqrt(2.0 / n))`, n = k·k·out_channels (backbone/wsgn/resnext.py:109-112).  It is the
    same distribution as He-normal fan_out, but for some n `sqrt(2/n)` and `sqrt(2)/sqrt(n)` differ in the last bit.
    """
    stem_conv = conv(3, 64, 7, 2, 3, bias=False)
    stem = _Stem(stem_conv, norm(64), nn.ReLU(inplace=True))
    pool = _StemPool(3, 2, 1)

    layers, cin = [], 64
    for width, depth, stride in _RESNET50_STAGES:
        blocks = []
        for b in range(depth):
            s = stride if b == 0 else 1
            shortcut = None
            if b == 0 and (s != 1 or cin != width * Bottleneck.expansion):
                # built *before* the unit's own convs: keeps the reference's RNG draw order
                shortcut = nn.Sequential(
                    conv(cin, width * Bottleneck.expansion, 1, s, bias=False),
                    norm(width * Bottleneck.expansion),
                )
            blocks.append(Bottleneck(cin, width, s, shortcut, conv=conv, norm=norm, cardinality=cardinality,
                                     base_width=base_width))
            cin = width * Bottleneck.expansion
        layers.append(nn.Sequential(*blocks))
    if imagenet_fc:
        nn.Linear(cin, 1000)

    # He-normal (fan_out) re-init of every conv in module-traversal order, BN γ=1 β=0 (GroupNorm keeps its own 1 / 0)
    for mod in [stem, *layers]:
        for m in mod.modules():
            if isinstance(m, nn.Conv2d) and cardinality > 1:
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                with torch.no_grad():
                    m.weight.normal_(0, math.sqrt(2.0 / n))
            elif isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
    return stem, nn.Sequential(pool, layers[0]), layers[1], layers[2], layers[3]


class _VGGPool(nn.MaxPool2d):
    """VGG16-BN's MaxPool2d(2, 2); routed to csrc/maxpool.cu when that kernel is enabled (the default)"""

    def forward(self, x):
        from .. import resample
        cover = (self.kernel_size, self.stride, self.padding, self.dilation, self.ceil_mode) == (2, 2, 0, 1, False)
        y = resample.maxpool2x2s2(x) if cover and not self.return_indices else None
        return y if y is not None else super().forward(x)


class _VGGSlice(nn.Sequential):
    """A slice of VGG16-BN's `features`, indexed from 0 as the reference's `nn.Sequential(*features[a:b])` is.  Each
    conv → BN → ReLU triple runs as `conv_bn_act`, so the engine folds the convolution's bias into the SyncBN kernel."""

    def forward(self, x):
        mods = list(self)
        i = 0
        while i < len(mods):
            if isinstance(mods[i], nn.Conv2d):
                x = conv_bn_act(mods[i], mods[i + 1], x)
                i += 3
            else:
                x = mods[i](x)
                i += 1
        return x


_VGG16_CFG = (64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512)   # "D", last "M" dropped
VGG16_SLICES = ((0, 6), (6, 13), (13, 23), (23, 33), (33, 43))    # features[a:b] of each of the five slices


def vgg16_bn_slices() -> tuple[nn.Module, nn.Module, nn.Module, nn.Module, nn.Module]:
    """VGG16-BN's `features` cut into the five slices the decoder taps (reference backbone/origin/from_origin.py:18-25):
    two conv–BN–ReLU triples at full resolution, then four slices that each open with a 2×2 max-pool.  The fifth pool
    (features[43]) is not part of the backbone.  Modules are built in `make_layers` order (backbone/origin/vgg.py) and
    nothing is re-initialised: the reference builds with `pretrained=True`, which passes `init_weights=False`, so its
    convolutions keep torch's default init (kaiming-uniform weights, uniform biases) and its BatchNorms 1 / 0.  Random init
    only (no network here) — use `load_pretrained_backbone` for torchvision's `vgg16_bn` file."""
    layers, cin = [], 3
    for v in _VGG16_CFG:
        if v == "M":
            layers.append(_VGGPool(2, 2))
        else:
            layers += [nn.Conv2d(cin, v, 3, padding=1), nn.BatchNorm2d(v), nn.ReLU(inplace=True)]
            cin = v
    return tuple(_VGGSlice(*layers[a:b]) for a, b in VGG16_SLICES)


class WSConv2d(nn.Conv2d):
    """Weight-standardised convolution of the WS-GN backbone (reference backbone/wsgn/customized_func.py:12-25): each
    filter is centred by the nested means over (C, R, S) and divided by its unbiased std + 1e-5 before the convolution.
    This is the plain-torch form (CPU, and the stock CUDA model); the engine swaps in `wsgn.FusedWSConv2d`, which runs
    the same map as one sm_90a kernel per direction.  The amp shadow weights and the optimizer's 16-bit gradient ranges
    leave these convolutions out: their gradient reaches the fp32 master through the standardisation."""

    eps = 1e-5

    def standardized_weight(self) -> torch.Tensor:
        w = self.weight
        w = w - w.mean(dim=1, keepdim=True).mean(dim=2, keepdim=True).mean(dim=3, keepdim=True)
        std = w.reshape(w.size(0), -1).std(dim=1).view(-1, 1, 1, 1) + self.eps
        return w / std.expand_as(w)

    def forward(self, x):
        return self._conv_forward(x, self.standardized_weight(), self.bias)


def group_norm32(channels: int) -> nn.GroupNorm:
    """the WS-GN backbone's `BatchNorm2d` (reference backbone/wsgn/customized_func.py:28-29): GroupNorm(32, C), eps 1e-5"""
    return nn.GroupNorm(32, channels)


class SIM(nn.Module):
    """Two-resolution interaction block: a full-res (`h`, `hc` channels) and a half-res
    (`l`, `lc` channels) stream exchange features twice and merge back to full-res
    (reference module/MyLightModule.py:11-54).  Attribute names are the checkpoint contract."""

    # (name, in, out) in registration order; 'h'/'l' resolved to channel counts
    _LAYOUT = (
        ("h2l_0", "h", "l"), ("h2h_0", "h", "h"), ("bnl_0", None, "l"), ("bnh_0", None, "h"),
        ("h2h_1", "h", "h"), ("h2l_1", "h", "l"), ("l2h_1", "l", "h"), ("l2l_1", "l", "l"),
        ("bnl_1", None, "l"), ("bnh_1", None, "h"),
        ("h2h_2", "h", "h"), ("l2h_2", "l", "h"), ("bnh_2", None, "h"),
    )

    def __init__(self, hc: int, lc: int):
        super().__init__()
        ch = {"h": hc, "l": lc}
        self.h2l_pool = nn.AvgPool2d((2, 2), stride=2)
        for name, src, dst in self._LAYOUT:
            if src is None:
                self.add_module(name, nn.BatchNorm2d(ch[dst]))
            else:
                self.add_module(name, nn.Conv2d(ch[src], ch[dst], 3, 1, 1))
        self.relu = nn.ReLU(True)

    def forward(self, x):
        hw = x.shape[2:]
        down = lambda t: avgpool2(self.h2l_pool, t)  # noqa: E731
        # stage 0: split into the two streams
        xh = conv_bn_act(self.h2h_0, self.bnh_0, x)
        xl = conv_bn_act(self.h2l_0, self.bnl_0, down(x))
        # stage 1: cross exchange
        h_new = conv_bn_act(self.h2h_1, self.bnh_1, xh, pre=(self.l2h_1, bilinear(xl, size=hw)))
        l_new = conv_bn_act(self.l2l_1, self.bnl_1, xl, pre=(self.h2l_1, down(xh)))
        # stage 2: merge to full-res
        return conv_bn_act(self.h2h_2, self.bnh_2, h_new, pre=(self.l2h_2, bilinear(l_new, size=hw)))
