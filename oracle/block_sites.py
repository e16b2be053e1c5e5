"""Block "sites" of the five TestModel models (`res50`, `vgg16`, `wsgn_res50`, `wsgn_resnext50`, `aim_res50`): each model
cut into the pieces `_TestModel.forward` strings together, so that each can be run and differentiated on its own
(tests/test_block_sites_cpu.py, tests/test_gpu_block_seams.py).  Every function takes the model's name, `res50` by
default.

A site owns the parameters and buffers under its module paths (every one of the model's belongs to exactly one site),
takes its inputs at image size S from `shapes(S, batch)` and runs as `run(mods, *inputs)`, `mods` mapping each path to a
module — the engine's own, or the float64 copies `stock_twin` makes.  `dispatch(site, S, amp, model_name)` says which
backward nodes of the engine's autograd seam (`_SyncBNFnBackward`, `_Up2xBackward`, `_GroupNormFnBackward`, …) its
forward must create: that follows the predicates of `resample.py` (C % 8 == 0; ×2 exactly; even H and W for the 2×2
average pool; `conv_bias`: C a power of two times 8, only reached by the `trans*` convolutions under amp shadow weights)
and of `wsgn.py` (the grouped-convolution kernels run only where `grouped_conv_on_kernels` holds) at the shapes the site
sees.

* `wsgn_res50` / `wsgn_resnext50` have `res50`'s sites (paths, shapes, representatives); their backbone norms are
  GroupNorm(32) and their convolutions weight-standardised, their decoder is `res50`'s.
* `vgg16`'s backbone sites are its five slices `div_2` … `div_32`, at strides 1 … 16; `div_4` … `div_32` open with a 2×2
  max-pool.  Its decoder sites carry `res50`'s names at half `res50`'s stride, and its head has no ×2 up-sample.
* `aim_res50` has `res50`'s backbone, SIM, upconv, upsample_add and head sites; its five `trans*` convolutions are
  replaced by the LightAIM neck's blocks `trans.conv0` … `trans.conv4` (`NECK_TAPS`), each taking two or three
  backbone taps (post-ReLU, so drawn non-negative: `relu_inputs`).  A neck site's `stride` is that of its output.
"""
from __future__ import annotations

import copy
from dataclasses import dataclass, field
from typing import Callable

import torch
import torch.nn as nn

TAPS = (32, 16, 8, 4, 2)
TAP_CHANNELS = {32: 2048, 16: 1024, 8: 512, 4: 256, 2: 64}
STAGES = ((4, 64, 3), (8, 128, 4), (16, 256, 6), (32, 512, 3))     # (stride, width, units) of ResNet-50
SIZES = (256, 288, 320, 352, 384)                                  # 288 / 352: odd 9×9 / 11×11 stride-32 map
MODELS = ("res50", "vgg16", "wsgn_res50", "wsgn_resnext50")     # the backbones, each with every decoder site
NECK_MODELS = ("aim_res50",)                                      # res50 with the LightAIM neck in place of trans*
ALL_MODELS = MODELS + NECK_MODELS                                 # every model with a site table
WSGN = ("wsgn_res50", "wsgn_resnext50")
VGG_TAP_CHANNELS = {32: 512, 16: 512, 8: 256, 4: 128, 2: 64}       # `vgg16.tap_channels`
VGG_SLICE_IN = {2: 3, 4: 64, 8: 128, 16: 256, 32: 512}             # input channels of slice div_s, at stride s // 4 (div_2: 1)

BN, UP, AVG, MAX, CONVB, LOSS = ("_SyncBNFnBackward", "_Up2xBackward", "_AvgPool2x2Backward", "_MaxPool3x3s2Backward",
                                 "_ConvBiasBackward", "_FusedLossFnBackward")
GN, WS, WSG, MAX2 = "_GroupNormFnBackward", "_WSFnBackward", "_WSGroupConvFnBackward", "_MaxPool2x2s2Backward"
NEAR = "_UpNearest2xBackward"
SEAM_NODES = (BN, UP, AVG, MAX, CONVB, GN, WS, WSG, MAX2, NEAR)
# LightAIM: block i of `trans` → (the backbone strides it takes, in argument order; the stride of its output)
NECK_TAPS = {0: ((2, 4), 2), 1: ((2, 4, 8), 4), 2: ((4, 8, 16), 8), 3: ((8, 16, 32), 16), 4: ((16, 32), 32)}
# per block: (BatchNorms, nearest ×2 up-samples, 2×2 average pools) of its forward — Conv2nV1 (blocks 0 and 4, main
# stream 0 / 1) and Conv3nV1 (blocks 1 … 3)
NECK_NODES = {0: (6, 2, 1), 1: (8, 3, 3), 2: (8, 3, 3), 3: (8, 3, 3), 4: (6, 1, 2)}


@dataclass(frozen=True)
class Site:
    name: str
    paths: tuple[str, ...]                    # module paths of the model whose parameters / buffers the site owns
    shapes: Callable[[int, int], list]        # (S, batch) → input shapes
    run: Callable                             # run(mods, *inputs) → output
    kind: str                                 # stem | pool | down | plain | vpool | trans | sim | upconv | upadd | head
    stride: int                               # stride of the site's input
    representative: bool = True               # GPU grid (`grid`); the other plain bottlenecks repeat a tested one
    loss: bool = False                        # head: the fused BCE + CEL loss follows
    input_grad: tuple[bool, ...] = field(default=(True,))
    relu_inputs: bool = False                 # the inputs are post-ReLU maps: draw them non-negative


def _bottleneck_site(stride, unit, cin, width, down):
    path = f"div_4.1.{unit}" if stride == 4 else f"div_{stride}.{unit}"
    s_in = stride // 2 if down else stride
    return Site(name=path, paths=(path,), shapes=lambda S, b, c=cin, s=s_in: [(b, c, S // s, S // s)],
                run=lambda mods, x, p=path: mods[p](x), kind="down" if down else "plain", stride=s_in,
                representative=down or unit == 1)


def _sim_run(s):
    def run(mods, x):
        return mods[f"sim{s}"](x) + x                 # `_decode`: up(sim(x) + x); the sum is the upconv's input
    return run


def _upadd_run(mods, coarse, lateral):
    from distributed_sod_project_b200.network.blocks import upsample_add
    return upsample_add(coarse, lateral)


def _head_run(mods, d2):
    from distributed_sod_project_b200.network.blocks import bilinear
    return mods["classifier"](mods["upconv1"](bilinear(d2, scale_factor=2)))


def _vgg_head_run(mods, d2):
    return mods["classifier"](mods["upconv1"](d2))       # `vgg16._head`: d2 is already at full resolution


def _check(model_name):
    if model_name not in ALL_MODELS:
        raise ValueError(f"no site table for model {model_name!r}; one of {ALL_MODELS}")


def _resnet_backbone() -> list[Site]:
    out = [Site("stem", ("div_2",), lambda S, b: [(b, 3, S, S)], lambda mods, x: mods["div_2"](x), "stem", 1),
           Site("pool+div_4.1.0", ("div_4.0", "div_4.1.0"), lambda S, b: [(b, 64, S // 2, S // 2)],
                lambda mods, x: mods["div_4.1.0"](mods["div_4.0"](x)), "pool", 2)]
    cin = 64
    for stride, width, units in STAGES:
        for u in range(units):
            if not (stride == 4 and u == 0):
                out.append(_bottleneck_site(stride, u, cin, width, down=u == 0))
            cin = 4 * width
    return out


def _vgg_backbone() -> list[Site]:
    out = []
    for s in reversed(TAPS):
        st = max(s // 4, 1)                  # div_2 and div_4 both see the full-resolution map
        out.append(Site(f"div_{s}", (f"div_{s}",), lambda S, b, c=VGG_SLICE_IN[s], st=st: [(b, c, S // st, S // st)],
                        lambda mods, x, s=s: mods[f"div_{s}"](x), "stem" if s == 2 else "vpool", st))
    return out


def _neck_site(i) -> Site:
    path = f"trans.conv{i}"
    taps, out = NECK_TAPS[i]
    return Site(path, (path,), lambda S, b, taps=taps: [(b, TAP_CHANNELS[t], S // t, S // t) for t in taps],
                lambda mods, *xs, p=path: mods[p](*xs), "neck", out, input_grad=(True,) * len(taps), relu_inputs=True)


def _decoder(tap_channels, half, trans=True) -> list[Site]:
    """trans* … head; `half`: every tap sits at half `res50`'s stride (vgg16); `trans`: with the five trans* sites"""
    st = {s: s // 2 if half else s for s in TAPS}
    out = []
    for s in TAPS if trans else ():
        out.append(Site(f"trans{s}", (f"trans{s}",), lambda S, b, s=s: [(b, tap_channels[s], S // st[s], S // st[s])],
                        lambda mods, x, s=s: mods[f"trans{s}"](x), "trans", st[s]))
    for s in TAPS:
        out.append(Site(f"sim{s}", (f"sim{s}",), lambda S, b, s=s: [(b, 64, S // st[s], S // st[s])], _sim_run(s), "sim",
                        st[s]))
    for s in TAPS:
        out.append(Site(f"upconv{s}", (f"upconv{s}",), lambda S, b, s=s: [(b, 64, S // st[s], S // st[s])],
                        lambda mods, x, s=s: mods[f"upconv{s}"](x), "upconv", st[s]))
    for s in TAPS[1:]:
        out.append(Site(f"upsample_add{s}", (), lambda S, b, s=s: [(b, 64, S // (2 * st[s]), S // (2 * st[s])),
                                                                   (b, 64, S // st[s], S // st[s])],
                        _upadd_run, "upadd", st[s], input_grad=(True, True)))
    h = st[2]                                # the head's input d2: up-sampled ×2 inside (res50), or not (vgg16)
    out.append(Site("head", ("upconv1", "classifier"), lambda S, b: [(b, 32, S // h, S // h)],
                    _vgg_head_run if half else _head_run, "head", h, loss=True))
    return out


def sites(model_name: str = "res50") -> list[Site]:
    _check(model_name)
    if model_name == "vgg16":
        return _vgg_backbone() + _decoder(VGG_TAP_CHANNELS, half=True)
    if model_name == "aim_res50":
        return _resnet_backbone() + [_neck_site(i) for i in NECK_TAPS] + _decoder(TAP_CHANNELS, half=False, trans=False)
    return _resnet_backbone() + _decoder(TAP_CHANNELS, half=False)


def grid(model_name: str = "res50") -> list[Site]:
    """the sites the GPU grid runs: the representative ones, without the WS-GN models' decoder (`res50`'s code at
    `res50`'s shapes, which the `res50` rows already run); for `aim_res50` its five neck sites alone (the rest is
    `res50`'s code at `res50`'s shapes)"""
    if model_name == "aim_res50":
        return [s for s in sites(model_name) if s.kind == "neck"]
    decoder = ("trans", "sim", "upconv", "upadd", "head")
    return [s for s in sites(model_name) if s.representative and not (model_name in WSGN and s.kind in decoder)]


def by_name(model_name: str = "res50") -> dict[str, Site]:
    return {s.name: s for s in sites(model_name)}


def modules(model: nn.Module, site: Site) -> dict[str, nn.Module]:
    return {p: model.get_submodule(p) for p in site.paths}


def owner(name: str, model_name: str = "res50") -> list[str]:
    """the sites a parameter / buffer name of the model belongs to"""
    return [s.name for s in sites(model_name) if any(name.startswith(p + ".") for p in s.paths)]


def _grouped_conv_on_kernels(site: Site) -> bool:
    """`wsgn.grouped_conv_on_kernels` for the ResNeXt-50 32×4d unit of `site`: its 3×3 has width / 16 channels in each
    of its 32 groups (width 64 … 512 by stage) and stride 2 in the first unit of stages 8 … 32; the kernels take 8
    channels per group at stride 2, so the first unit of stage 8 alone"""
    if site.kind != "down":
        return False
    stride = int(site.name.split(".")[0][len("div_"):])
    return dict((s, w) for s, w, _ in STAGES)[stride] // 16 == 8


def dispatch(site: Site, size: int, amp: bool, model_name: str = "res50") -> dict[str, bool]:
    """backward node → present, for the engine's forward of `site` at image size `size` (amp: 16-bit shadow weights).

    The LightAIM neck sites (`aim_res50`) take every map at strides 2 … 16 through their 2×2 average pools; at every
    size of SIZES (multiples of 32) those maps are even — only the stride-32 map is odd, 9² at 288² and 11² at 352², and
    no neck block pools it — so every neck pool runs on the kernel.  Their nearest ×2 up-samples take any H, W and C % 8
    == 0 (64 channels, 1024 in block 4).  Under amp the 1×1 `identity` convolution, called as a module, takes
    `conv_bias` (C = 64); the 3×3 ones fold their biases into the SyncBN kernel.  `counts` gives the numbers."""
    _check(model_name)
    if site.kind == "neck":
        want = dict.fromkeys(SEAM_NODES, False)
        want[BN] = want[NEAR] = want[AVG] = True
        want[CONVB] = amp
        return want
    hw = size // site.stride
    want = dict.fromkeys(SEAM_NODES, False)
    backbone = site.kind in ("stem", "pool", "down", "plain", "vpool")
    if site.kind in ("sim", "upconv", "head") or (backbone and model_name not in WSGN):
        want[BN] = True
    if backbone and model_name in WSGN:
        want[GN] = want[WS] = True   # every norm is GroupNorm(32), every convolution weight-standardised
        want[WSG] = model_name == "wsgn_resnext50" and _grouped_conv_on_kernels(site)
    if site.kind == "pool":
        want[MAX] = True
    if site.kind == "vpool":
        want[MAX2] = True            # C = 64 … 512 and H, W ≥ 2 at every VGG pool
    if site.kind == "sim":
        even = hw % 2 == 0           # avgpool2 needs even H, W; the ×2 bilinear back to hw exists only then (vgg16: at
        want[AVG] = want[UP] = even  # strides 1 … 16 of 256² … 384² always even)
    if site.kind == "upadd" or (site.kind == "head" and model_name != "vgg16"):
        want[UP] = True              # vgg16's head has no ×2 up-sample
    if site.kind == "trans":
        want[CONVB] = amp            # C = 64: sod_colsum's bias gradient, reached through the shadow-weight forward
    return want                      # head: the classifier's C = 1 never takes `conv_bias`


def counts(site: Site, amp: bool) -> dict[str, int]:
    """backward node → how many the engine's forward of the neck site `site` creates (`dispatch` says which)"""
    if site.kind != "neck":
        raise ValueError(f"{site.name}: node counts are kept for the neck sites only")
    n_bn, n_near, n_avg = NECK_NODES[int(site.name[len("trans.conv"):])]
    return {BN: n_bn, NEAR: n_near, AVG: n_avg, CONVB: 1 if amp else 0}


def stock_twin(site: Site, model: nn.Module | None = None, dtype: torch.dtype = torch.float64,
               model_name: str = "res50") -> dict[str, nn.Module]:
    """copies of the site's modules from a stock model (`nn.BatchNorm2d`, `nn.GroupNorm` and `WSConv2d` as built, no
    amp), in `dtype` (float64 by default).  `model`: the stock model to copy from, else `init_seed(0)` + the factory
    `model_name`, the engine's starting point.  Run them with `resample.ENABLED` off (see `stock_modules`)."""
    _check(model_name)
    if model is None:
        from distributed_sod_project_b200 import network
        from distributed_sod_project_b200.utils import init_seed
        init_seed(0)
        model = getattr(network, model_name)()
    return {p: copy.deepcopy(m).to(dtype) for p, m in modules(model, site).items()}


def reference_loss(logits, mask, eps=1e-6):
    """BCEWithLogits(mean) + CEL (oracle/loss.py) in the dtype of the inputs"""
    import torch.nn.functional as F
    bce = F.binary_cross_entropy_with_logits(logits, mask)
    p = torch.sigmoid(logits)
    inter = p * mask
    cel = ((p - inter).sum() + (mask - inter).sum()) / (p.sum() + mask.sum() + eps)
    return bce + cel


class stock_modules:
    """context: the model's own torch ops (no resampling / max-pool / column-sum kernels)"""

    def __enter__(self):
        from distributed_sod_project_b200 import resample
        from distributed_sod_project_b200.network import blocks
        self.old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = False, False
        return self

    def __exit__(self, *exc):
        from distributed_sod_project_b200 import resample
        from distributed_sod_project_b200.network import blocks
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = self.old
        return False


def compose(model: nn.Module, image: torch.Tensor, model_name: str = "res50") -> torch.Tensor:
    """`_TestModel.forward` restated site by site (every site, in model order)"""
    table = by_name(model_name)

    def run(name, *xs):
        site = table[name]
        return site.run(modules(model, site), *xs)

    if model_name == "vgg16":
        feats, x = {}, image
        for s in reversed(TAPS):
            x = feats[s] = run(f"div_{s}", x)
    else:
        x = run("stem", image)
        feats = {2: x}
        x = run("pool+div_4.1.0", x)
        for u in range(1, 3):
            x = run(f"div_4.1.{u}", x)
        feats[4] = x
        for stride, _, units in STAGES[1:]:
            for u in range(units):
                x = run(f"div_{stride}.{u}", x)
            feats[stride] = x
    if model_name == "aim_res50":
        lat = {out: run(f"trans.conv{i}", *(feats[t] for t in taps)) for i, (taps, out) in NECK_TAPS.items()}
    else:
        lat = {s: run(f"trans{s}", feats[s]) for s in (2, 4, 8, 16, 32)}
    d = None
    for s in TAPS:
        x = lat[s] if d is None else run(f"upsample_add{s}", d, lat[s])
        d = run(f"upconv{s}", run(f"sim{s}", x))
    return run("head", d)
