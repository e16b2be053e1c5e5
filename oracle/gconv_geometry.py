"""Launch geometry of csrc/gconv.cu (the 32-group 3×3 convolutions), restated for tests.

Every grid is a function of the shape only (never of the SM count), so a result is the same on every card.
* fwd / dgrad, 16-bit: one CTA per (group, pixels_per_cta(cpg) output pixels); the warps walk 16-pixel m-tiles, the
  last of which may be partly outside the image ("tail"), and the last CTA may own fewer m-tiles ("partial").
* fp32: one thread per (output pixel, group), CTAs of 128 pixels.
* wgrad: the N·Ho·Wo pixels in S chunks of pc pixels (pc a multiple of 32, the last chunk possibly shorter), one CTA
  per (chunk, group); the S fp32 partials are added in chunk order by a second launch.
"""
from __future__ import annotations

GROUPS = 32
CPG = (4, 8, 16, 32)
THREADS, WARPS, TILES_PER_WARP = 128, 4, 8
WG_PIXELS, WG_MIN_CHUNK, WG_MAX_SPLIT = 32, 512, 32


def out_size(h: int, stride: int) -> int:
    return (h - 1) // stride + 1


def pixels_per_cta(cpg: int) -> int:
    return 16 * WARPS * TILES_PER_WARP // max(1, cpg // 8)


def wgrad_geometry(pixels: int) -> tuple[int, int]:
    """(S, pc): chunks and pixels per chunk"""
    s = min(max(-(-pixels // WG_MIN_CHUNK), 1), WG_MAX_SPLIT)
    per = -(-pixels // s)
    pc = -(-per // WG_PIXELS) * WG_PIXELS
    return -(-pixels // pc), pc


def regime(n: int, h: int, w: int, cpg: int, stride: int, out_hw: tuple[int, int] | None = None) -> tuple:
    """(wgrad split, last chunk, last m-tile, last CTA) of one launch over an output of n × out_hw pixels (the
    convolution's output for fwd / wgrad, the input size for dgrad)"""
    oh, ow = out_hw if out_hw is not None else (out_size(h, stride), out_size(w, stride))
    p = n * oh * ow
    s, pc = wgrad_geometry(p)
    split = "single" if s == 1 else ("capped" if s == WG_MAX_SPLIT and -(-p // WG_MIN_CHUNK) > WG_MAX_SPLIT else "split")
    last = "even" if p % pc == 0 else "short"
    tile = "whole" if p % 16 == 0 else "tail"
    cta = "full" if p % pixels_per_cta(cpg) == 0 else "partial"
    return split, last, tile, cta


def regime_cases():
    """(n, h, w, cpg, stride) shapes that reach every cell of `regime` for every cpg, both strides"""
    shapes = ((1, 1, 1), (1, 2, 2), (2, 11, 11), (1, 16, 32), (2, 40, 40), (16, 80, 80), (3, 7, 5), (4, 64, 64))
    out = []
    for cpg in CPG:
        for stride in (1, 2):
            for n, h, w in shapes:
                out.append((n, h, w, cpg, stride, regime(n, h, w, cpg, stride)))
    return out
