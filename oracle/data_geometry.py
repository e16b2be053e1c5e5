"""ORACLE (test infrastructure only): the launch geometry of the data-side kernels, restated from csrc/pipeline.cu,
csrc/resize.cu and csrc/augment.cu.

* `preprocess_kernel` (`sod_preprocess_batch`) runs min(⌈N·Ho·Wo/256⌉, 16·#SMs) CTAs of 256 threads over the output
  pixels, grid-stride: one pass covers 16·#SMs·256 pixels (540,672 on 132 SMs).  `quantize_kernel`
  (`sod_saliency_quantize`) is the same loop over n elements with a cap of 8·#SMs CTAs.  Both are classified by wave as
  in oracle/resample_geometry.py: a partial wave below the cap, exactly one pass, one pass plus a ragged one, two or more
  passes ragged or exact.  Pre-processing also has a mode per call (identity, both axes up, both down, one axis resized).
* `metric_head_kernel` runs one 512-thread CTA per image; a thread strides ⌈h·w/512⌉ times, and h·w < 512 leaves
  threads idle.
* `metric_hist_kernel` runs `per` CTAs of 256 threads per image, grid-stride over the image's pixels.  The fixed-size
  entry takes per = clamp(⌈h·w/4096⌉, 1, 64), so a thread makes at most 16 passes until h·w > 63·4096 = 258,048, where
  per is capped at 64 and each CTA strides further.  The ragged entry cannot read the sizes: per = clamp(⌈4·#SMs/n⌉, 1,
  64), so every image gets the same per, 64 for n ≤ 8 on 132 SMs and 1 for n ≥ 4·#SMs.
* `sod_resize_u8` launches three kernels over (n, per) CTAs, per = clamp(⌈8·#SMs/n⌉, 1, 128); CTA y of an image does
  the rows y, y + per, … of each pass.  per = 1 (n ≥ 8·#SMs) makes one CTA do every row of its image.  Which passes
  run depends on the sizes alone: a copy when nothing changes, the horizontal or the vertical pass alone when only one
  axis changes, both otherwise.
* `sod_augment_u8` launches two kernels over n × ⌈S/r⌉ CTAs of 256 threads, r = 1024 // S rows per tile, or r = 1 when
  S ≥ 1024, where a tile is one row and each thread loops ⌈S/256⌉ times.

`cells(kernel, shape, sm)` names the regime cells one launch reaches, `required(kernel, sm)` the cells a device must
reach, and `select(kernel, cell, sm)` the smallest shape reaching a cell on `sm` SMs.
"""
from __future__ import annotations

THREADS = 256                       # preprocess, quantize, hist, resize and augment CTAs
PREP_CTAS_PER_SM = 16
QUANT_CTAS_PER_SM = 8
HEAD_THREADS = 512
HIST_PX_PER_CTA = 4096              # fixed-size entry: 256 threads × 16 pixels
HIST_MAX_PER = 64
HIST_RAGGED_CTAS_PER_SM = 4
RESIZE_CTAS_PER_SM = 8
RESIZE_MAX_PER = 128
AUG_PIXELS_PER_CTA = 1024

KERNELS = ("preprocess", "quantize", "head", "hist_fixed", "hist_ragged", "resize", "augment")
WAVES = ("partial", "1", "1+ragged", ">=2 ragged", ">=2 exact")
PREP_MODES = ("identity", "up", "down", "mixed")


def cdiv(a, b):
    return -(-a // b)


# ---- grid-stride waves (preprocess, quantize) -----------------------------------------------------------------------
def _cap(kernel, sm):
    return (PREP_CTAS_PER_SM if kernel == "preprocess" else QUANT_CTAS_PER_SM) * sm


def grid(kernel, total, sm):
    """CTAs of a preprocess / quantize launch over `total` elements"""
    return min(cdiv(total, THREADS), _cap(kernel, sm))


def full_pass(kernel, sm):
    return _cap(kernel, sm) * THREADS


def wave(kernel, total, sm):
    full = full_pass(kernel, sm)
    if total < full:
        return "partial"
    if total == full:
        return "1"
    if total < 2 * full:
        return "1+ragged"
    return ">=2 exact" if total % full == 0 else ">=2 ragged"


def thread_elements(kernel, total, sm):
    """per thread, the element indices its grid-stride loop visits"""
    step = grid(kernel, total, sm) * THREADS
    return [range(t, total, step) for t in range(step)]


def prep_mode(hs, ws, ho, wo):
    if (hs, ws) == (ho, wo):
        return "identity"
    if hs < ho and ws < wo:
        return "up"
    if hs > ho and ws > wo:
        return "down"
    return "mixed"


def _out_split(total):
    """(n, ho, wo) with n·ho·wo = total: the largest image of at most 4096 pixels dividing total, both sides ≥ 2 and
    as square as possible"""
    for hw in range(min(total, 4096), 3, -1):
        sides = [d for d in range(2, int(hw ** 0.5) + 1) if hw % d == 0]
        if total % hw == 0 and sides:
            return total // hw, sides[-1], hw // sides[-1]
    raise ValueError(total)


def _prep_source(mode, ho, wo):
    if mode == "identity":
        return ho, wo
    if mode == "up":
        return max(1, ho * 5 // 8), max(1, wo * 5 // 8)
    if mode == "down":
        return ho * 3 // 2 + 1, wo * 3 // 2 + 1
    return ho * 3 // 2 + 1, wo                          # mixed: rows resized, columns not


# ---- metric kernels -----------------------------------------------------------------------------------------------
def head_cell(hw):
    if hw < HEAD_THREADS:
        return "idle"
    if hw == HEAD_THREADS:
        return "1"
    return ">=1000" if hw >= 1000 * HEAD_THREADS else "ragged"


def hist_fixed_per(hw):
    return max(1, min(cdiv(hw, HIST_PX_PER_CTA), HIST_MAX_PER))


def hist_fixed_cell(hw):
    per = hist_fixed_per(hw)
    if per == 1:
        return "idle" if hw < THREADS else "1"
    return "cap" if per == HIST_MAX_PER else "mid"


def hist_ragged_per(n, sm):
    return max(1, min(cdiv(HIST_RAGGED_CTAS_PER_SM * sm, n), HIST_MAX_PER))


def hist_ragged_cell(n, sm):
    per = hist_ragged_per(n, sm)
    if per == 1:
        return "1"
    return "max" if per == hist_ragged_per(1, sm) else "mid"


# ---- resize -------------------------------------------------------------------------------------------------------
def resize_per(n, sm):
    return max(1, min(cdiv(RESIZE_CTAS_PER_SM * sm, n), RESIZE_MAX_PER))


def resize_cell(n, sm):
    per = resize_per(n, sm)
    if per == 1:
        return "1"
    return "max" if per == resize_per(1, sm) else "mid"


def resize_passes(ih, iw, oh, ow):
    if (ih, iw) == (oh, ow):
        return "copy"
    if ih == oh:
        return "h"
    if iw == ow:
        return "v"
    return "hv"


# ---- augment ------------------------------------------------------------------------------------------------------
def aug_rows_per_tile(s):
    return 1 if s >= AUG_PIXELS_PER_CTA else AUG_PIXELS_PER_CTA // s


def aug_grid(n, s):
    return n, cdiv(s, aug_rows_per_tile(s))


def aug_cell(s):
    r = aug_rows_per_tile(s)
    if r == 1:
        return "row" if s == AUG_PIXELS_PER_CTA else "row-loop"
    return "tile exact" if s % r == 0 else "tile ragged"


# ---- cells --------------------------------------------------------------------------------------------------------
def cells(kernel, shape, sm):
    """the regime cells one launch reaches.  Shapes: preprocess (n, hs, ws, ho, wo); quantize (numel,); head, hist_fixed
    and hist_ragged [(h, w), …] per image; resize (n, passes); augment (n, S)"""
    if kernel == "preprocess":
        n, hs, ws, ho, wo = shape
        out = {("wave", wave(kernel, n * ho * wo, sm), prep_mode(hs, ws, ho, wo))}
        if (hs, ws) == (1, 1):
            out.add(("source", "1x1"))
        if (ho, wo) == (1, 1):
            out.add(("output", "1x1"))
        return out
    if kernel == "quantize":
        return {("wave", wave(kernel, shape[0], sm))}
    if kernel == "head":
        return {("image", head_cell(h * w)) for h, w in shape}
    if kernel == "hist_fixed":
        return {("image", hist_fixed_cell(h * w)) for h, w in shape}
    if kernel == "hist_ragged":
        return {("per", hist_ragged_cell(len(shape), sm))}
    if kernel == "resize":
        n, passes = shape
        return {("per", resize_cell(n, sm))} | {("passes", p) for p in passes}
    if kernel == "augment":
        n, s = shape
        return {("tile", aug_cell(s)), ("n", "1" if n == 1 else ">1")}
    raise KeyError(kernel)


def required(kernel, sm):
    if kernel == "preprocess":
        return {("wave", w, m) for w in WAVES for m in PREP_MODES} | {("source", "1x1"), ("output", "1x1")}
    if kernel == "quantize":
        return {("wave", w) for w in WAVES}
    if kernel == "head":
        return {("image", c) for c in ("idle", "1", "ragged", ">=1000")}
    if kernel == "hist_fixed":
        return {("image", c) for c in ("idle", "1", "mid", "cap")}
    if kernel == "hist_ragged":
        return {("per", c) for c in ("1", "mid", "max")}
    if kernel == "resize":
        return {("per", c) for c in ("1", "mid", "max")} | {("passes", p) for p in ("copy", "h", "v", "hv")}
    if kernel == "augment":
        return {("tile", c) for c in ("tile exact", "tile ragged", "row", "row-loop")} | {("n", "1"), ("n", ">1")}
    raise KeyError(kernel)


def _smallest_n(pred):
    n = 1
    while not pred(n):
        n += 1
    return n


def select(kernel, cell, sm):
    """the smallest shape (in the `cells` convention) whose launch reaches `cell` on `sm` SMs.  Pre-processing totals
    move in steps of 64 output pixels, so that a batch splits into images of at least 2 × 2 (one pass is 64² · #SMs)"""
    if kernel in ("preprocess", "quantize"):
        if cell[0] != "wave":
            assert kernel == "preprocess"
            return (1, 1, 1, 5, 7) if cell == ("source", "1x1") else (1, 5, 7, 1, 1)
        w = cell[1]
        full = full_pass(kernel, sm)
        m = 64 if kernel == "preprocess" else 1
        total = {"partial": THREADS + m, "1": full, "1+ragged": full + m, ">=2 ragged": 2 * full + m, ">=2 exact": 2 * full}[w]
        if kernel == "quantize":
            return (total,)
        n, ho, wo = _out_split(total)
        hs, ws = _prep_source(cell[2], ho, wo)
        shape = (n, hs, ws, ho, wo)
    elif kernel == "head":
        hw = {"idle": 1, "1": HEAD_THREADS, "ragged": HEAD_THREADS + 1, ">=1000": 1000 * HEAD_THREADS}[cell[1]]
        shape = [{1: (1, 1), HEAD_THREADS: (16, 32), HEAD_THREADS + 1: (1, 513), 1000 * HEAD_THREADS: (800, 640)}[hw]]
    elif kernel == "hist_fixed":
        shape = [{"idle": (1, 1), "1": (16, 16), "mid": (64, 65), "cap": (63 * 64 + 1, 64)}[cell[1]]]
    elif kernel == "hist_ragged":
        want = cell[1]
        n = _smallest_n(lambda k: hist_ragged_cell(k, sm) == want)
        shape = [(1, 1)] * n
    elif kernel == "resize":
        if cell[0] == "per":
            n = _smallest_n(lambda k: resize_cell(k, sm) == cell[1])
            shape = (n, ("copy",))
        else:
            shape = (1, (cell[1],))
    elif kernel == "augment":
        if cell[0] == "n":
            shape = (1 if cell[1] == "1" else 2, 1)
        else:
            # S = 32: 32 tiles of 32 rows; S = 33: 31 rows and a last tile of 2 (S < 32 is one partial tile)
            shape = (1, {"tile exact": 32, "tile ragged": 33, "row": 1024, "row-loop": 1025}[cell[1]])
    else:
        raise KeyError(kernel)
    assert cell in cells(kernel, shape, sm), (kernel, cell, sm, shape)
    return shape
