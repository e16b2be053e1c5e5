"""ORACLE (test infrastructure only): the weighted F-measure of the reference (utils/saliency_metric.py:232-303) on
scipy's exact nearest-foreground indices, restated in numpy, and the launch geometry of csrc/wfm.cu.

Feature transform.  `scipy.ndimage.distance_transform_edt(~fg, return_indices=True)` runs two separable passes, a 1-D
lower-envelope sweep over every line: first along axis 0 (each column), then along axis 1 (each row).  A site is a
foreground pixel (pass 1) or the site pass 1 found for a column (pass 2), at position s along the line, with squared
distance R(s) to the line: 0 in pass 1, (row_of_site - y)² in pass 2.
* envelope build, in line order: for a new site w with v on top of the stack and u below it, a = v - u, b = w - v,
  c = a + b; pop v while c·R(v) - b·R(u) - a·R(w) - a·b·c > 0; then push w;
* query, in line order, with a pointer l from the first stacked site: move l on only while the next site is strictly
  nearer (squared distance); a tie keeps the current site.
With R ≡ 0 (pass 1) the pop test is -a·b·c > 0, never true: every site stays, and the query picks the nearest foreground
pixel of the column, the upper one on a tie — which is what the column kernel computes with two sweeps and no stack.
Every quantity is an integer far below 2⁵³, so the device does the same comparisons exactly in int64.

`feature_transform(fg)` returns scipy's (row, col) index arrays (-1 where there is no foreground at all) and the
float64 distances; `wfm(pred_u8, gt_u8)` is `metrics._wfm_host` on top of it.

Launch geometry (csrc/wfm.cu; sizes known on the host, grids sized by the largest image of the batch):
* column pass: (⌈max w/128⌉, n) CTAs of 128 threads, one thread per (image, column).  Cells: a full last column block
  (w % 128 == 0), a tail block (w % 128 != 0), idle CTAs of a narrower image in a ragged batch, several blocks per image.
* row pass: (⌈max h/128⌉, n) CTAs of 4 warps, one thread per (image, row); each warp stages 32 rows × 32 columns of
  pass 1's output in shared memory at a time.  Cells: a partial warp (h % 32 != 0), idle warps (⌈h/32⌉ % 4 != 0), a tail
  column chunk (w % 32 != 0), a single chunk (w ≤ 32), idle CTAs of a shorter image.
* weighted-error pass: (max tiles, n) CTAs of 256 threads, one per 32 × 32 tile of an image (⌈h/32⌉·⌈w/32⌉ tiles);
  the last CTA of an image to finish adds its tiles' partial sums in a fixed tree order.  Cells: a tail row tile
  (h % 32), a tail column tile (w % 32), one tile, idle CTAs of a smaller image, more CTAs than fit on the device at once.
"""
from __future__ import annotations

import numpy as np

COL_THREADS = 128
ROW_THREADS = 128
ROW_WARP_ROWS = 32
ROW_CHUNK = 32
TILE = 32
TILE_THREADS = 256
MAX_THREADS_PER_SM = 2048
MAX_WIDTH = 1 << 21                # wider images are refused: keeps the envelope test's int64 terms below 2⁶³

LOG_HALF_OVER_5 = np.log(0.5) / 5  # B = 2 - exp(log(0.5)/5 · Dst) on the background


def gaussian_kernel() -> np.ndarray:
    """the reference's 7×7 MATLAB-style Gaussian with σ = 5 (utils/saliency_metric.py:279-283), float64"""
    ax = np.arange(-3, 4, dtype=np.float64)
    k = np.exp(-(ax[None, :] ** 2 + ax[:, None] ** 2) / (2.0 * 5 * 5))
    k[k < np.finfo(k.dtype).eps * k.max()] = 0
    return k / k.sum()


def coefficients() -> np.ndarray:
    """the 50 doubles the WFM entries take: the 7×7 kernel row-major, then log(0.5)/5"""
    return np.concatenate([gaussian_kernel().reshape(-1), [LOG_HALF_OVER_5]]).astype(np.float64)


# ---- feature transform ----------------------------------------------------------------------------------------------
def envelope_1d(pos: np.ndarray, r: np.ndarray, n: int) -> np.ndarray:
    """one line of n pixels with sites at increasing positions `pos` and perpendicular squared distances `r`: the index
    into `pos` of the site scipy assigns to every pixel (-1 for every pixel when there is no site)"""
    if len(pos) == 0:
        return np.full(n, -1, dtype=np.int64)
    stack: list[int] = []
    for k in range(len(pos)):
        w = int(pos[k])
        while len(stack) >= 2:
            v, u = int(pos[stack[-1]]), int(pos[stack[-2]])
            a, b = v - u, w - v
            c = a + b
            if c * int(r[stack[-1]]) - b * int(r[stack[-2]]) - a * int(r[k]) - a * b * c > 0:
                stack.pop()
            else:
                break
        stack.append(k)
    out = np.empty(n, dtype=np.int64)
    l = 0
    for x in range(n):
        while l + 1 < len(stack):
            cur, nxt = stack[l], stack[l + 1]
            dc = (int(pos[cur]) - x) ** 2 + int(r[cur])
            dn = (int(pos[nxt]) - x) ** 2 + int(r[nxt])
            if dn < dc:
                l += 1
            else:
                break
        out[x] = stack[l]
    return out


def feature_transform(fg: np.ndarray):
    """fg: bool [h, w].  Returns (iy, ix, dist): scipy's `distance_transform_edt(~fg, return_indices=True)` indices and
    distances, with -1 indices and inf distance everywhere when fg is empty (scipy leaves those undefined)."""
    fg = np.asarray(fg, dtype=bool)
    h, w = fg.shape
    col = np.full((h, w), -1, dtype=np.int64)              # pass 1: row of the column's site
    for x in range(w):
        pos = np.nonzero(fg[:, x])[0]
        k = envelope_1d(pos, np.zeros(len(pos), dtype=np.int64), h)
        col[:, x] = np.where(k >= 0, pos[np.maximum(k, 0)] if len(pos) else -1, -1)
    iy = np.full((h, w), -1, dtype=np.int64)
    ix = np.full((h, w), -1, dtype=np.int64)
    for y in range(h):
        pos = np.nonzero(col[y] >= 0)[0]
        r = (col[y, pos] - y) ** 2
        k = envelope_1d(pos, r, w)
        if len(pos):
            ix[y] = pos[k]
            iy[y] = col[y, ix[y]]
    yy, xx = np.mgrid[0:h, 0:w]
    d2 = (iy - yy) ** 2 + (ix - xx) ** 2
    dist = np.where(iy >= 0, np.sqrt(d2.astype(np.float64)), np.inf)
    return iy, ix, dist


def column_nearest(fg: np.ndarray) -> np.ndarray:
    """pass 1 as the column kernel computes it: nearest foreground row of each column, the upper one on a tie, -1 when
    the column has none"""
    fg = np.asarray(fg, dtype=bool)
    h, w = fg.shape
    out = np.full((h, w), -1, dtype=np.int64)
    for x in range(w):
        above = -1
        ab = np.empty(h, dtype=np.int64)
        for y in range(h):
            if fg[y, x]:
                above = y
            ab[y] = above
        below = -1
        for y in range(h - 1, -1, -1):
            if fg[y, x]:
                below = y
            a = ab[y]
            out[y, x] = below if a < 0 or (below >= 0 and below - y < y - a) else a
    return out


# ---- the metric -----------------------------------------------------------------------------------------------------
def normalise(pred_u8: np.ndarray, gt_u8: np.ndarray):
    """the rules of metrics._wfm_host: gt / (max + 1e-8) > 0.5 and (u - min)/(max - min), or u/255 when max == min"""
    gt = gt_u8 / (gt_u8.max() + 1e-8) > 0.5
    mx, mn = int(pred_u8.max()), int(pred_u8.min())
    pred = pred_u8 / 255 if mx == mn else (pred_u8.astype(np.float64) - mn) / (mx - mn)
    return pred, gt


def wfm_sums(pred_u8: np.ndarray, gt_u8: np.ndarray):
    """(ΣEw[gt], ΣEw[~gt], n_fg) of one image, float64 — what the device reduces per image"""
    from scipy.ndimage import convolve
    pred, gt = normalise(pred_u8, gt_u8)
    if not gt.any():
        return 0.0, 0.0, 0.0
    iy, ix, dst = feature_transform(gt)
    err = np.abs(pred - gt)
    et = err[iy, ix]                                        # foreground pixels map to themselves
    ea = convolve(et, weights=gaussian_kernel(), mode="constant", cval=0)
    min_e = np.where(gt & (ea < err), ea, err)
    ew = min_e * np.where(gt, 1.0, 2 - np.exp(LOG_HALF_OVER_5 * dst))
    return float(ew[gt].sum()), float(ew[~gt].sum()), float(gt.sum())


def q_from_sums(s_fg: float, s_bg: float, n_fg: float, beta: float = 1, eps: float = 1e-6) -> float:
    """Q of utils/saliency_metric.py:292-301 from the three sums (0 without foreground)"""
    if n_fg == 0:
        return 0.0
    tpw = n_fg - s_fg
    r = 1 - s_fg / n_fg
    p = tpw / (eps + tpw + s_bg)
    return float((1 + beta) * r * p / (eps + r + beta * p))


def wfm(pred_u8: np.ndarray, gt_u8: np.ndarray, beta: float = 1) -> float:
    return q_from_sums(*wfm_sums(pred_u8, gt_u8), beta=beta)


# ---- test masks ------------------------------------------------------------------------------------------------------
def mask_families(rng):
    """(name, fg bool [h, w]) test masks rich in ties: lattices, discs, symmetric point pairs, single pixels, full
    masks, rows or columns without foreground, 1×N and N×1, scattered points and random densities"""
    out = []
    for h, w in ((1, 1), (1, 17), (17, 1), (2, 2), (9, 13), (31, 8), (40, 40)):
        yy, xx = np.mgrid[0:h, 0:w]
        for s in (2, 3, 5):
            out.append((f"lattice{s} {h}x{w}", (yy % s == 0) & (xx % s == 0)))
        out.append((f"disc {h}x{w}", (yy - (h - 1) / 2) ** 2 + (xx - (w - 1) / 2) ** 2 <= (min(h, w) / 3) ** 2))
        out.append((f"random {h}x{w}", rng.random((h, w)) < 0.2))
        pair = np.zeros((h, w), bool)
        pair[0, 0] = pair[h - 1, w - 1] = True                  # symmetric pair: the centre line ties
        out.append((f"corners {h}x{w}", pair))
        pair = np.zeros((h, w), bool)
        pair[h // 2, 0] = pair[h // 2, w - 1] = True
        out.append((f"row pair {h}x{w}", pair))
        pair = np.zeros((h, w), bool)
        pair[0, w // 2] = pair[h - 1, w // 2] = True
        out.append((f"column pair {h}x{w}", pair))
        single = np.zeros((h, w), bool)
        single[h // 3, w // 2] = True
        out.append((f"single {h}x{w}", single))
        out.append((f"full {h}x{w}", np.ones((h, w), bool)))
        rows = rng.random((h, w)) < 0.3
        rows[::2] = False                                       # rows (and often columns) without foreground
        rows[h // 2, w // 2] = True
        out.append((f"empty rows {h}x{w}", rows))
        cols = rng.random((h, w)) < 0.3
        cols[:, 1::3] = False
        cols[h // 2, 0] = True
        out.append((f"empty columns {h}x{w}", cols))
    for k in range(12):                                         # three scattered points and random densities
        h, w = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        m = np.zeros((h, w), bool)
        for _ in range(3):
            m[rng.integers(0, h), rng.integers(0, w)] = True
        out.append((f"points {h}x{w}", m))
        out.append((f"density {h}x{w}", rng.random((h, w)) < rng.uniform(0.01, 0.6)))
    return [(n, m) for n, m in out if m.any()]


# ---- launch geometry ------------------------------------------------------------------------------------------------
def cdiv(a, b):
    return -(-a // b)


def tiles(h, w):
    return cdiv(h, TILE) * cdiv(w, TILE)


def grids(hw):
    """CTAs of the three launches for images of sizes hw [(h, w), ...]: {kernel: (grid_x, n, threads)}"""
    n = len(hw)
    mh, mw = max(h for h, _ in hw), max(w for _, w in hw)
    return {"column": (cdiv(mw, COL_THREADS), n, COL_THREADS),
            "row": (cdiv(mh, ROW_THREADS), n, ROW_THREADS),
            "weighted": (max(tiles(h, w) for h, w in hw), n, TILE_THREADS)}


def cells(hw, sm: int):
    """the regime cells a call over images of sizes hw reaches on `sm` SMs, as (kernel, cell) pairs"""
    g = grids(hw)
    out = set()
    out.add(("batch", "one image" if len(hw) == 1 else "many images"))
    for h, w in hw:
        out.add(("column", "tail block" if w % COL_THREADS else "full block"))
        if w > COL_THREADS:
            out.add(("column", "several blocks"))
        if cdiv(w, COL_THREADS) < g["column"][0]:
            out.add(("column", "idle CTA"))
        out.add(("row", "partial warp" if h % ROW_WARP_ROWS else "full warps"))
        if cdiv(h, ROW_WARP_ROWS) % (ROW_THREADS // 32):
            out.add(("row", "idle warp"))
        out.add(("row", "tail chunk" if w % ROW_CHUNK else "full chunks"))
        if w <= ROW_CHUNK:
            out.add(("row", "single chunk"))
        if cdiv(h, ROW_THREADS) < g["row"][0]:
            out.add(("row", "idle CTA"))
        if h % TILE:
            out.add(("weighted", "tail row tile"))
        if w % TILE:
            out.add(("weighted", "tail column tile"))
        if tiles(h, w) == 1:
            out.add(("weighted", "one tile"))
        if tiles(h, w) < g["weighted"][0]:
            out.add(("weighted", "idle CTA"))
    for k, (gx, n, threads) in g.items():
        if gx * n > sm * (MAX_THREADS_PER_SM // threads):
            out.add((k, "beyond one wave"))
    return out


REQUIRED = (("batch", "one image"), ("batch", "many images"),
            ("column", "tail block"), ("column", "full block"), ("column", "several blocks"), ("column", "idle CTA"),
            ("column", "beyond one wave"),
            ("row", "partial warp"), ("row", "full warps"), ("row", "idle warp"), ("row", "tail chunk"),
            ("row", "full chunks"), ("row", "single chunk"), ("row", "idle CTA"), ("row", "beyond one wave"),
            ("weighted", "tail row tile"), ("weighted", "tail column tile"), ("weighted", "one tile"),
            ("weighted", "idle CTA"), ("weighted", "beyond one wave"))


def select(cell, sm: int):
    """a small list of image sizes whose call reaches `cell` on `sm` SMs"""
    kernel, name = cell
    if cell == ("batch", "one image"):
        return [(5, 7)]
    if name == "beyond one wave":
        # enough images for the kernel's CTAs to exceed one wave at the thread limit
        per = {"column": (40, 129), "row": (129, 40), "weighted": (64, 64)}[kernel]
        g = grids([per])[kernel]
        resident = sm * (MAX_THREADS_PER_SM // g[2])
        return [per] * (resident // g[0] + 1)
    table = {
        ("batch", "many images"): [(9, 11), (13, 6)],
        ("column", "tail block"): [(6, 130)],
        ("column", "full block"): [(5, 128)],
        ("column", "several blocks"): [(4, 300)],
        ("column", "idle CTA"): [(7, 260), (9, 20)],
        ("row", "partial warp"): [(45, 9)],
        ("row", "full warps"): [(64, 9)],
        ("row", "idle warp"): [(70, 12)],
        ("row", "tail chunk"): [(40, 75)],
        ("row", "full chunks"): [(40, 64)],
        ("row", "single chunk"): [(50, 17)],
        ("row", "idle CTA"): [(300, 20), (12, 20)],
        ("weighted", "tail row tile"): [(70, 64)],
        ("weighted", "tail column tile"): [(64, 70)],
        ("weighted", "one tile"): [(20, 30)],
        ("weighted", "idle CTA"): [(100, 100), (31, 33)],
    }
    return table[cell]
