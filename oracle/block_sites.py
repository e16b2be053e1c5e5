"""Block "sites" of `res50`: the model cut into the pieces `_TestModel.forward` strings together, so that each can be run
and differentiated on its own (tests/test_block_sites_cpu.py, tests/test_gpu_block_seams.py).

A site owns the parameters and buffers under its module paths (every one of the model's belongs to exactly one site),
takes its inputs at image size S from `shapes(S, batch)` and runs as `run(mods, *inputs)`, `mods` mapping each path to a
module — the engine's own, or the float64 copies `stock_twin` makes.  `dispatch(site, S, amp)` says which backward nodes
of the engine's autograd seam (`_SyncBNFnBackward`, `_Up2xBackward`, …) its forward must create: that follows the
predicates of `resample.py` (C % 8 == 0; ×2 exactly; even H and W for the 2×2 pool; `conv_bias`: C a power of two times
8, only reached by the `trans*` convolutions under amp shadow weights) at the shapes the site sees.
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

BN, UP, AVG, MAX, CONVB, LOSS = ("_SyncBNFnBackward", "_Up2xBackward", "_AvgPool2x2Backward", "_MaxPool3x3s2Backward",
                                 "_ConvBiasBackward", "_FusedLossFnBackward")
SEAM_NODES = (BN, UP, AVG, MAX, CONVB)


@dataclass(frozen=True)
class Site:
    name: str
    paths: tuple[str, ...]                    # module paths of res50 whose parameters / buffers the site owns
    shapes: Callable[[int, int], list]        # (S, batch) → input shapes
    run: Callable                             # run(mods, *inputs) → output
    kind: str                                 # stem | pool | down | plain | trans | sim | upconv | upadd | head
    stride: int                               # stride of the site's input
    representative: bool = True               # in the GPU grid (the other plain bottlenecks repeat a tested one)
    loss: bool = False                        # head: the fused BCE + CEL loss follows
    input_grad: tuple[bool, ...] = field(default=(True,))


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


def sites() -> list[Site]:
    out = [Site("stem", ("div_2",), lambda S, b: [(b, 3, S, S)], lambda mods, x: mods["div_2"](x), "stem", 1),
           Site("pool+div_4.1.0", ("div_4.0", "div_4.1.0"), lambda S, b: [(b, 64, S // 2, S // 2)],
                lambda mods, x: mods["div_4.1.0"](mods["div_4.0"](x)), "pool", 2)]
    cin = 64
    for stride, width, units in STAGES:
        for u in range(units):
            if not (stride == 4 and u == 0):
                out.append(_bottleneck_site(stride, u, cin, width, down=u == 0))
            cin = 4 * width
    for s in TAPS:
        out.append(Site(f"trans{s}", (f"trans{s}",), lambda S, b, s=s: [(b, TAP_CHANNELS[s], S // s, S // s)],
                        lambda mods, x, s=s: mods[f"trans{s}"](x), "trans", s))
    for s in TAPS:
        out.append(Site(f"sim{s}", (f"sim{s}",), lambda S, b, s=s: [(b, 64, S // s, S // s)], _sim_run(s), "sim", s))
    for s in TAPS:
        out.append(Site(f"upconv{s}", (f"upconv{s}",), lambda S, b, s=s: [(b, 64, S // s, S // s)],
                        lambda mods, x, s=s: mods[f"upconv{s}"](x), "upconv", s))
    for s in TAPS[1:]:
        out.append(Site(f"upsample_add{s}", (), lambda S, b, s=s: [(b, 64, S // (2 * s), S // (2 * s)), (b, 64, S // s, S // s)],
                        _upadd_run, "upadd", s, input_grad=(True, True)))
    out.append(Site("head", ("upconv1", "classifier"), lambda S, b: [(b, 32, S // 2, S // 2)], _head_run, "head", 2,
                    loss=True))
    return out


def by_name() -> dict[str, Site]:
    return {s.name: s for s in sites()}


def modules(model: nn.Module, site: Site) -> dict[str, nn.Module]:
    return {p: model.get_submodule(p) for p in site.paths}


def owner(name: str) -> list[str]:
    """the sites a parameter / buffer name of res50 belongs to"""
    return [s.name for s in sites() if any(name.startswith(p + ".") for p in s.paths)]


def dispatch(site: Site, size: int, amp: bool) -> dict[str, bool]:
    """backward node → present, for the engine's forward of `site` at image size `size` (amp: 16-bit shadow weights)"""
    hw = size // site.stride
    want = dict.fromkeys(SEAM_NODES, False)
    if site.kind in ("stem", "pool", "down", "plain", "sim", "upconv", "head"):
        want[BN] = True
    if site.kind == "pool":
        want[MAX] = True
    if site.kind == "sim":
        even = hw % 2 == 0           # avgpool2 needs even H, W; the ×2 bilinear back to hw exists only then
        want[AVG] = want[UP] = even
    if site.kind in ("upadd", "head"):
        want[UP] = True
    if site.kind == "trans":
        want[CONVB] = amp            # C = 64: sod_colsum's bias gradient, reached through the shadow-weight forward
    return want                      # head: the classifier's C = 1 never takes `conv_bias`


def stock_twin(site: Site, model: nn.Module | None = None, dtype: torch.dtype = torch.float64) -> dict[str, nn.Module]:
    """copies of the site's modules from a stock `res50` (`nn.BatchNorm2d` as built, no amp), in `dtype` (float64 by
    default).  `model`: the stock model to copy from, else `init_seed(0)` + `res50()`, the engine's starting point.
    Run them with `resample.ENABLED` off (see `stock_modules`)."""
    if model is None:
        from distributed_sod_project_b200 import network
        from distributed_sod_project_b200.utils import init_seed
        init_seed(0)
        model = network.res50()
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


def compose(model: nn.Module, image: torch.Tensor) -> torch.Tensor:
    """`_TestModel.forward` restated site by site (every site, in model order)"""
    table = by_name()

    def run(name, *xs):
        site = table[name]
        return site.run(modules(model, site), *xs)

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
    lat = {s: run(f"trans{s}", feats[s]) for s in (2, 4, 8, 16, 32)}
    d = None
    for s in TAPS:
        x = lat[s] if d is None else run(f"upsample_add{s}", d, lat[s])
        d = run(f"upconv{s}", run(f"sim{s}", x))
    return run("head", d)
