"""ORACLE (test infrastructure only): the launch geometry of csrc/joint.cu, restated.

`sod_resize_nearest_u8` (its copy kernel), `sod_window_u8` and each of the six `sod_gaussian_blur_u8` passes run
(n, per) CTAs of 256 threads; CTA y of image b does the output bytes y·256 + t, then + per·256, … of its image, with

    per = clamp(min(⌈8·#SMs / n⌉, ⌈largest image's bytes / 256⌉), 1, 128).

So an image of `bytes` output bytes is covered in one pass when bytes ≤ per·256 (a partial pass when per·256 − bytes
leaves whole CTAs or threads idle), or by ⌈bytes / (per·256)⌉ grid-stride passes whose last is a tail unless it divides
exactly.  The NEAREST tables are one thread per image and axis, whatever the sizes.

`regime(per, bytes)` names the cell of one image, `per_of(n, max_bytes, sm)` the launch's CTAs per image.
"""
from __future__ import annotations

THREADS = 256
CTAS_PER_SM = 8
MAX_PER = 128
REGIMES = ("one pass, idle CTAs", "one pass", "passes + tail", "passes exact")


def cdiv(a, b):
    return -(-a // b)


def per_of(n: int, max_bytes: int, sm: int) -> int:
    return max(1, min(cdiv(CTAS_PER_SM * sm, n), cdiv(max_bytes, THREADS), MAX_PER))


def regime(per: int, nbytes: int) -> str:
    span = per * THREADS
    if nbytes <= span:
        return "one pass" if cdiv(nbytes, THREADS) == per else "one pass, idle CTAs"
    return "passes exact" if nbytes % span == 0 else "passes + tail"


def cells(n: int, image_bytes, sm: int) -> set:
    """the regimes a launch over images of `image_bytes` output bytes each reaches"""
    per = per_of(n, max(image_bytes), sm)
    return {regime(per, b) for b in image_bytes}
