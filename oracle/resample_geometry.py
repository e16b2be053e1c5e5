"""ORACLE (test infrastructure only): the launch geometry of the resampling kernels, restated from csrc/resample.cu,
csrc/maxpool.cu and csrc/nearest.cu.

* The eight grid-stride kernels (bilinear ×2, 2×2 average pool, 3×3/2 max pool and nearest ×2, forward and backward) run
  `grid_for` CTAs of 256 threads, at most 16 per SM, and thread t handles the 16-byte channel packets t, t + T, t + 2T, …
  of the tensor it writes (T = grid·256).  The forward of the bilinear up-sample and the backward of the average pool
  write the larger tensor, the max pool's two kernels and the other two the smaller one; the nearest kernels run one
  thread per packet of the smaller (input) side in both directions, the forward writing its four copies, the backward
  gathering its four taps.  So the packet count P of a shape differs by kernel.  `classify` puts P in a
  wave regime: a partial wave below the cap, exactly one full pass, one full pass plus a ragged one, two or more passes
  ragged or exact.
* `sod_colsum` runs min(⌈rows/8R⌉, 2·#SMs, 296) CTAs of 256 threads, L = C/8 lanes by R = 256/L rows.  Thread (b, r0)
  sums the rows b·R + r0 + j·step (step = grid·R) for j < q, in groups of four, (v0 + v1) + (v2 + v3), while four remain,
  then one by one (q mod 4 of them); q = 0 for a thread whose first row is past the end.  Each CTA sums its R row
  partials in order and the last CTA sums the CTA partials in CTA order.  `colsum_replay` repeats that in fp32: it only
  adds, so numpy float32 gives the kernel's bits.
* `select` / `select_colsum` find the smallest shape reaching a regime cell on a given SM count.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

K_THREADS = 256            # resample.cu, maxpool.cu and nearest.cu kThreads
K_CTAS_PER_SM = 16         # grid_for's cap: 16·#SMs CTAs
COLSUM_THREADS = 256
COLSUM_PASSES = 8          # at least eight row passes per CTA before the grid grows
COLSUM_CTAS_PER_SM = 2
COLSUM_MAX_GRID = 296
COLSUM_MAX_C = 2048
COLSUM_UNROLL = 4

KERNELS = ("upsample_fwd", "upsample_bwd", "avgpool_fwd", "avgpool_bwd", "maxpool_fwd", "maxpool_bwd")   # what res50 runs
NEAREST_KERNELS = ("nearest_fwd", "nearest_bwd")                  # the LightAIM neck's (aim_res50)
GRID_STRIDE_KERNELS = KERNELS + NEAREST_KERNELS                   # all eight
DTYPES = ("float32", "bfloat16", "float16")
WAVES = ("partial", "1", "1+ragged", ">=2 ragged", ">=2 exact")
LANES = tuple(1 << k for k in range(9))                   # L = C/8 = 1 … 256
COLSUM_AXES = dict(L=LANES, grid=("below", "cap"), tail=(0, 1, 2, 3), idle=("yes",), rows=("1",))


# ---- the eight grid-stride kernels -------------------------------------------------------------------------------
def grid_for(packets, sm_count):
    return int(min(max(-(-packets // K_THREADS), 1), K_CTAS_PER_SM * sm_count))


def packets(kernel, shape):
    """16-byte packets the kernel's loop runs over for the forward input `shape` = (n, c, h, w) (the nearest kernels: one
    per input packet in both directions); the avg-pool needs even h, w"""
    n, c, h, w = shape
    c8 = c // 8
    if kernel == "upsample_fwd":
        return n * 2 * h * 2 * w * c8
    if kernel in ("upsample_bwd", "maxpool_bwd", "avgpool_bwd", "nearest_fwd", "nearest_bwd"):
        return n * h * w * c8
    if kernel == "avgpool_fwd":
        return n * (h // 2) * (w // 2) * c8
    if kernel == "maxpool_fwd":
        return n * ((h - 1) // 2 + 1) * ((w - 1) // 2 + 1) * c8
    raise KeyError(kernel)


def thread_packets(p, sm_count):
    """per thread of the grid, the packet indices its grid-stride loop visits (a list of arrays)"""
    total = grid_for(p, sm_count) * K_THREADS
    return [np.arange(t, p, total) for t in range(total)]


def passes(p, sm_count):
    """per thread, how many times its loop body runs"""
    total = grid_for(p, sm_count) * K_THREADS
    t = np.arange(total)
    return np.where(t < p, -(-(p - t) // total), 0)


def classify(p, sm_count):
    full = K_CTAS_PER_SM * sm_count * K_THREADS
    if p < full:
        return "partial"
    if p == full:
        return "1"
    if p < 2 * full:
        return "1+ragged"
    return ">=2 exact" if p % full == 0 else ">=2 ragged"


def _multiple(kernel):
    """P is a multiple of 4 where the kernel writes the ×2 side of the op (not the nearest kernels: one thread per input
    packet)"""
    return 4 if kernel in ("upsample_fwd", "avgpool_bwd") else 1


def _factor(b):
    """(n, c8, h, w) with n·c8·h·w = b: c8 the largest of 8, 4, 2, 1 dividing b, n = 2 where that leaves ≥ 8, and
    h ≥ w the most nearly square split (w = 1 for a prime)"""
    c8 = next(k for k in (8, 4, 2, 1) if b % k == 0)
    rest = b // c8
    n = 2 if rest % 2 == 0 and rest >= 8 else 1
    rest //= n
    w = max(d for d in range(1, int(rest ** 0.5) + 1) if rest % d == 0)
    return n, c8, rest // w, w


def shape_for(kernel, p):
    """a forward input shape (n, c, h, w) whose kernel writes exactly p packets"""
    m = _multiple(kernel)
    assert p % m == 0
    n, c8, h, w = _factor(p // m)
    if kernel.startswith("upsample"):
        shape = (n, 8 * c8, h, w)
    elif kernel.startswith("avgpool"):
        shape = (n, 8 * c8, 2 * h, 2 * w)
    elif kernel == "maxpool_fwd":
        shape = (n, 8 * c8, 2 * h, 2 * w - 1)                # even and odd input sizes
    else:
        shape = (n, 8 * c8, h, w)
    assert packets(kernel, shape) == p, (kernel, p, shape)
    return shape


def select(kernel, wave, sm_count):
    """the smallest forward input shape whose `kernel` launch is in `wave` on `sm_count` SMs.  "partial" asks for more
    than one CTA and a ragged last CTA (a one-CTA launch is the degenerate shapes' business)"""
    full = K_CTAS_PER_SM * sm_count * K_THREADS
    m = _multiple(kernel)
    p = {"partial": K_THREADS + m, "1": full, "1+ragged": full + m, ">=2 ragged": 2 * full + m, ">=2 exact": 2 * full}[wave]
    shape = shape_for(kernel, p)
    assert classify(packets(kernel, shape), sm_count) == wave
    return shape


# ---- sod_colsum ----------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class ColsumLaunch:
    rows: int
    L: int
    R: int
    grid: int
    cap: int
    step: int
    q: np.ndarray            # [grid, R]: rows each thread sums (its lanes share them)


def colsum_launch(rows, c, sm_count):
    assert rows > 0 and c % 8 == 0 and c <= COLSUM_MAX_C
    L = c // 8
    assert L & (L - 1) == 0
    R = COLSUM_THREADS // L
    cap = min(COLSUM_CTAS_PER_SM * sm_count, COLSUM_MAX_GRID)
    grid = min(max(-(-rows // (R * COLSUM_PASSES)), 1), cap)
    step = grid * R
    start = np.arange(grid)[:, None] * R + np.arange(R)[None, :]
    q = np.where(start < rows, -(-(rows - start) // step), 0)
    return ColsumLaunch(rows, L, R, grid, cap, step, q)


def colsum_thread_rows(g: ColsumLaunch):
    """per thread (b, r0), the rows it reads: the unrolled groups first, then the tail"""
    return {(b, r0): b * g.R + r0 + g.step * np.arange(int(g.q[b, r0])) for b in range(g.grid) for r0 in range(g.R)}


def classify_colsum(g: ColsumLaunch):
    live = g.q[g.q > 0]
    return dict(L=g.L, grid="cap" if g.grid == g.cap else "below", qmax=int(g.q.max()),
                tails=frozenset(int(v) for v in np.unique(live % COLSUM_UNROLL)), idle=bool((g.q == 0).any()),
                ragged=g.rows % g.step != 0, rows1=g.rows == 1)


def colsum_cells(g: ColsumLaunch):
    cls = classify_colsum(g)
    cells = {("L", g.L), ("grid", cls["grid"])} | {("tail", t) for t in cls["tails"]}
    if cls["idle"]:
        cells.add(("idle", "yes"))
    if cls["rows1"]:
        cells.add(("rows", "1"))
    return cells


def required_colsum_cells():
    return {(axis, v) for axis, vals in COLSUM_AXES.items() for v in vals}


# every L at the cap, with the largest per-thread row count 8 … 11 so that the q and q − 1 of its threads give all four
# tail residues; below the cap: one row (idle threads, one CTA), a one-CTA launch with idle threads and a full grid of
# eight passes per thread
COLSUM_SPECS = tuple(dict(L=L, grid="cap", qmax=8 + j % 4, ragged=j % 2 == 0) for j, L in enumerate(LANES)) + (
    dict(L=8, rows1=True),
    dict(L=1, grid="below", idle=True, rows1=False),
    dict(L=256, grid="below", qmax=8, ragged=False),
    dict(L=32, grid="below", qmax=5, ragged=True),
)


def select_colsum(want, sm_count):
    """the smallest row count whose launch at C = 8·want["L"] has every other property in `want`, or None"""
    c = 8 * want["L"]
    R = COLSUM_THREADS // want["L"]
    cap = min(COLSUM_CTAS_PER_SM * sm_count, COLSUM_MAX_GRID)
    hi = (want.get("qmax", 12) + 1) * cap * R
    for rows in range(1, hi + 1):
        # cheap rejections first: the grid, q of thread 0 (⌈rows/step⌉) and whether rows is a multiple of step
        grid = min(max(-(-rows // (R * COLSUM_PASSES)), 1), cap)
        if "grid" in want and (grid == cap) != (want["grid"] == "cap"):
            continue
        if "qmax" in want and -(-rows // (grid * R)) != want["qmax"]:
            continue
        if "ragged" in want and (rows % (grid * R) != 0) != want["ragged"]:
            continue
        cls = classify_colsum(colsum_launch(rows, c, sm_count))
        if all(cls[k] == v for k, v in want.items()):
            return rows
    return None


def colsum_replay(x, sm_count):
    """the kernel's fp32 sum of x ([rows, C], values exact in fp32) over rows, as a float32 [C] array"""
    x = np.asarray(x, np.float32)
    rows, c = x.shape
    g = colsum_launch(rows, c, sm_count)
    depth = int(g.q.max())
    xp = np.zeros((depth * g.step, c), np.float32)
    xp[:rows] = x
    v = xp.reshape(depth, g.grid, g.R, c)                   # v[j, b, r0] = row b·R + r0 + j·step
    q = g.q[:, :, None]
    groups = q // COLSUM_UNROLL
    a = np.zeros((g.grid, g.R, c), np.float32)
    for k in range(depth // COLSUM_UNROLL):
        j = COLSUM_UNROLL * k
        s = (v[j] + v[j + 1]) + (v[j + 2] + v[j + 3])
        a = np.where(k < groups, a + s, a)
    for j in range(depth):
        a = np.where((j >= COLSUM_UNROLL * groups) & (j < q), a + v[j], a)
    cta = np.zeros((g.grid, c), np.float32)
    for r0 in range(g.R):
        cta = cta + a[:, r0]
    out = np.zeros(c, np.float32)
    for b in range(g.grid):
        out = out + cta[b]
    return out
