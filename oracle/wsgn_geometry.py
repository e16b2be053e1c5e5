"""ORACLE (test infrastructure only): the launch geometry of the GroupNorm kernels, restated from csrc/wsgn.cu
`gn_geometry`, with the SM count as an argument, so the tests can ask which regime a launch takes on any GPU.

A sample's H·W rows are split over S CTAs of 256 threads; a thread owns 8 channels (L = C/8 lanes) and R = 256/L row
phases walk the CTA's chunk.  The regime axes:
* split: "one" (S == 1: the sample's own CTA merges its single partial) or "many" (S > 1);
* tail: "even" (every CTA has rc rows) or "short" (the last CTA of a sample has fewer);
* phases: "idle" (a CTA has fewer rows than R: some row phases see no row) or "full";
* lanes: R > 1 (several rows per pass) or R == 1 (C = 2048: one row per pass).
"""
from __future__ import annotations

from dataclasses import dataclass

THREADS = 256
MAX_SPLIT = 1024
CHANNELS = (64, 128, 256, 512, 1024, 2048)          # the backbone's GroupNorm widths (C/G = 2 … 64)


@dataclass(frozen=True)
class Geom:
    L: int
    R: int
    S: int
    rc: int


def make_geom(n: int, hw: int, c: int, sm_count: int) -> Geom:
    L = c // 8
    R = THREADS // L
    want = (2 * sm_count + n - 1) // n
    min_rows = 8 * R
    most = (hw + min_rows - 1) // min_rows
    s = max(1, min(want, most, MAX_SPLIT))
    rc = (hw + s - 1) // s
    return Geom(L, R, (hw + rc - 1) // rc, rc)


def classify(n: int, hw: int, c: int, sm_count: int) -> tuple[str, str, str, str]:
    g = make_geom(n, hw, c, sm_count)
    last = hw - (g.S - 1) * g.rc
    return ("one" if g.S == 1 else "many", "even" if last == g.rc else "short",
            "idle" if last < g.R else "full", "multi" if g.R > 1 else "single")


def regime_cases(sm_count: int) -> list[tuple[int, int, int, tuple]]:
    """(n, h, w, c) shapes, one per regime cell reachable on this SM count, smallest first: the search walks the
    backbone's channel widths, batch sizes 1-16 and square sizes from 1 to 192 (the stem at a 384² input)"""
    found: dict = {}
    for c in CHANNELS:
        for n in (1, 2, 3, 16):
            for side in list(range(1, 24)) + [40, 80, 96, 160, 192]:
                cell = classify(n, side * side, c, sm_count)
                if cell not in found:
                    found[cell] = (n, side, side, c)
    return [(*v, k) for k, v in sorted(found.items())]
