"""ORACLE (test infrastructure only): the launch geometry of the fused BCE+CEL kernels, restated from csrc/loss.cu.

`launch` is the host function `launch_loss` with the device (SM count, opt-in shared memory per block) as arguments
instead of a query, and with the per-CTA slices the kernels derive from it, so the tests can ask which kernel a launch
runs and which branches each CTA takes on any GPU:

* the grid is min(⌈n/4096⌉, #SMs) CTAs, each owning `per_cta` elements (⌈n/grid⌉ rounded up to 8) of the
  16-byte-packet part [0, n & ~7); the scalar tail [n & ~7, n) belongs to CTA 0;
* `need` 4096-element chunks per CTA fit in shared memory up to the resident limit (min(budget / chunk bytes, 12)):
  then `loss_bce_cel_kernel` holds the whole slice; beyond it (or always with mode 2) `loss_stream_kernel` runs its ring
  of NS stages, and chunks [0, nres0) of a CTA are streamed a second time in phase 2; mode 1 refuses instead.

On top of it `classify` gives the regime of a launch (one value per axis of AXES) and `select` the smallest n that
reaches a requested regime on a given device.

Property (tests/test_loss_geometry_model.py): for n ≥ 8 no CTA is ever empty, since (grid − 1)·per_cta < n & ~7.
"""
from __future__ import annotations

from dataclasses import dataclass
from functools import lru_cache

import numpy as np

K_THREADS = 512
K_CHUNK = 4096
K_MAX_RESIDENT = 12
K_MAX_STREAM_STAGES = 12
K_MAX_GRID = 1024
RESIDENT_RESERVE = 128 + 1024          # mbarriers + static shared memory of loss_bce_cel_kernel
STREAM_RESERVE = 256 + 1024            # full/empty mbarriers + static shared memory of loss_stream_kernel

# (logits, mask) element types of the ten kernel instances: five dtype pairs × two kernels
PAIRS = (("float32", "float32"), ("bfloat16", "float32"), ("float16", "float32"),
         ("bfloat16", "bfloat16"), ("float16", "float16"))
DTYPE_BYTES = {"float32": 4, "bfloat16": 2, "float16": 2}
FEW_MAX = 8


@dataclass(frozen=True)
class Launch:
    n: int
    mode: int
    kernel: str              # "resident", "streamed" or "refused" (mode 1 on a slice beyond the resident window)
    grid: int
    per_cta: int
    need: int                # chunks of a full slice
    resident_limit: int      # chunks the resident kernel can hold (before the clamp to `need`; 0 in mode 2)
    resident: int            # min(resident_limit, need): the resident kernel's chunk count
    ns: int                  # ring stages of the streamed kernel (0 otherwise)
    chunks: tuple            # per CTA: chunk count
    nres0: tuple             # per CTA: chunks streamed again in phase 2 (streamed kernel; 0 otherwise)
    partial: tuple           # per CTA: its last chunk holds fewer than 4096 elements
    tail: int                # n − (n & ~7), computed by CTA 0 in both phases


def resident_limit(sx, sm, max_smem_optin):
    return min((max_smem_optin - RESIDENT_RESERVE) // (K_CHUNK * (sx + sm)), K_MAX_RESIDENT)


def stream_stages(sx, sm, max_smem_optin):
    return min((max_smem_optin - STREAM_RESERVE) // (K_CHUNK * (sx + sm)), K_MAX_STREAM_STAGES)


def launch(n, sx, sm, mode, sm_count, max_smem_optin):
    """csrc/loss.cu launch_loss for n elements, sx-byte logits and sm-byte mask; None where it returns SOD_EUNSUPPORTED
    for want of two ring stages"""
    assert n > 0 and mode in (0, 1, 2)
    limit = 0 if mode == 2 else resident_limit(sx, sm, max_smem_optin)
    grid = min(max(-(-n // K_CHUNK), 1), sm_count)
    assert grid <= K_MAX_GRID
    per_cta = (-(-n // grid) + 7) & ~7
    need = -(-per_cta // K_CHUNK)
    resident = min(limit, need)
    ns = 0
    if need > resident:
        if mode == 1:
            kernel = "refused"
        else:
            ns = stream_stages(sx, sm, max_smem_optin)
            if ns < 2:
                return None
            kernel = "streamed"
    else:
        kernel = "resident"
    nvec = n & ~7
    chunks, nres0, partial = [], [], []
    for b in range(grid):
        e0 = min(b * per_cta, nvec)
        e1 = min(b * per_cta + per_cta, nvec)
        c = -(-(e1 - e0) // K_CHUNK)
        chunks.append(c)
        nres0.append(c - ns if kernel == "streamed" and c > ns else 0)
        partial.append((e1 - e0) % K_CHUNK != 0)
    return Launch(n, mode, kernel, grid, per_cta, need, limit, resident, ns, tuple(chunks), tuple(nres0), tuple(partial),
                  n - nvec)


# ---- regimes ---------------------------------------------------------------------------------------------------------
AXES = dict(
    kernel=("resident", "streamed"),
    chunks=("1", "2..limit-1", "limit", "<NS-1", "NS-1", "NS", "NS+1", "2NS+1", ">=3NS"),
    ctas=("1", "few", "grid"),
    last=("equal", "fewer", "partial"),
    tail=("0", "1-7", "n<8"),
    mode=(0, 2),
)
RESIDENT_CHUNKS = ("1", "2..limit-1", "limit")
STREAMED_CHUNKS = ("<NS-1", "NS-1", "NS", "NS+1", "2NS+1", ">=3NS")


def classify(g: Launch, sm_count):
    """the regime of a launch, one value per axis (None: a value no axis tracks).  `chunks` is CTA 0's chunk count (the
    most any CTA has): against the resident limit for the resident kernel, against NS for the streamed one; `last`
    compares the last CTA with CTA 0 ("partial": as many chunks, the last one partial)."""
    c0 = g.chunks[0]
    if c0 == 0:
        ch = None                                   # n < 8: the scalar tail is the whole tensor
    elif g.kernel == "resident":
        ch = "1" if c0 == 1 else ("limit" if c0 == g.resident_limit else "2..limit-1")
    elif g.kernel == "streamed":
        ns = g.ns
        ch = {ns - 1: "NS-1", ns: "NS", ns + 1: "NS+1", 2 * ns + 1: "2NS+1"}.get(c0)
        if ch is None:
            ch = "<NS-1" if c0 < ns - 1 else (">=3NS" if c0 >= 3 * ns else None)
    else:
        ch = None
    if c0 == 0:
        last = None
    elif g.chunks[-1] < c0:
        last = "fewer"
    else:
        last = "partial" if g.partial[-1] else "equal"
    ctas = "1" if g.grid == 1 else ("grid" if g.grid == sm_count else ("few" if g.grid <= FEW_MAX else "many"))
    tail = "n<8" if g.n < 8 else ("0" if g.tail == 0 else "1-7")
    return dict(kernel=g.kernel, chunks=ch, ctas=ctas, last=last, tail=tail, mode=g.mode)


def matches(cls, want):
    return all(cls[k] == v for k, v in want.items())


def reachable(kernel, axis, value):
    """whether a cell (kernel, axis value) can occur at all: the resident kernel runs in mode 0 only and counts chunks
    against its limit, the streamed kernel against NS"""
    if axis == "chunks":
        return value in (RESIDENT_CHUNKS if kernel == "resident" else STREAMED_CHUNKS)
    if axis == "mode":
        return kernel == "streamed" or value == 0
    if axis == "kernel":
        return value == kernel
    return True


# ---- the selector: the same rules on arrays of n, so a whole range of n is classified at once -----------------------
CHUNK_CODES = {v: i for i, v in enumerate(AXES["chunks"])}


def regimes(n, sx, sm, mode, sm_count, max_smem_optin):
    """`classify(launch(n, …))` for an int64 array of n, as integer codes: dict axis → array of indices into AXES[axis]
    (−1: None; see _UNTRACKED for values no regime targets).  Only CTA 0 and the last CTA are needed: every CTA but the last owns `per_cta`."""
    n = np.asarray(n, np.int64)
    limit = 0 if mode == 2 else resident_limit(sx, sm, max_smem_optin)
    ns = stream_stages(sx, sm, max_smem_optin)
    grid = np.clip(-(-n // K_CHUNK), 1, sm_count)
    per = ((-(-n // grid)) + 7) & ~7
    need = -(-per // K_CHUNK)
    nvec = n & ~7
    c0 = -(-np.minimum(per, nvec) // K_CHUNK)
    rest = nvec - np.minimum((grid - 1) * per, nvec)          # elements of the last CTA
    clast = -(-rest // K_CHUNK)
    plast = rest % K_CHUNK != 0
    beyond = need > limit
    kernel = np.where(beyond, 2 if mode == 1 else 1, 0)
    res_ch = np.where(c0 == 1, CHUNK_CODES["1"], np.where(c0 == limit, CHUNK_CODES["limit"], CHUNK_CODES["2..limit-1"]))
    st_ch = np.full_like(c0, -1)
    st_ch = np.where(c0 >= 3 * ns, CHUNK_CODES[">=3NS"], st_ch)
    st_ch = np.where(c0 < ns - 1, CHUNK_CODES["<NS-1"], st_ch)
    for k, name in ((ns - 1, "NS-1"), (ns, "NS"), (ns + 1, "NS+1"), (2 * ns + 1, "2NS+1")):
        st_ch = np.where(c0 == k, CHUNK_CODES[name], st_ch)
    chunks = np.where(kernel == 0, res_ch, np.where(kernel == 1, st_ch, -1))
    chunks = np.where(c0 == 0, -1, chunks)
    last = np.where(clast < c0, 1, np.where(plast, 2, 0))
    last = np.where(c0 == 0, -1, last)
    ctas = np.where(grid == 1, 0, np.where(grid == sm_count, 2, np.where(grid <= FEW_MAX, 1, 3)))
    tail = np.where(n < 8, 2, np.where(n % 8 == 0, 0, 1))
    return dict(kernel=kernel, chunks=chunks, ctas=ctas, last=last, tail=tail, mode=np.full_like(n, _code("mode", mode)))


_UNTRACKED = {("kernel", "refused"): 2, ("ctas", "many"): 3, ("mode", 1): 2}


def _code(axis, value):
    return _UNTRACKED.get((axis, value)) or AXES[axis].index(value)


def _chunk_range(want, sx, sm, mode, max_smem_optin):
    """the CTA-0 chunk counts [lo, hi] a wanted regime can have (chunks grow with n, so n outside them cannot match)"""
    limit = 0 if mode == 2 else resident_limit(sx, sm, max_smem_optin)
    ns = stream_stages(sx, sm, max_smem_optin)
    top = 3 * max(ns, limit) + 1
    ch = want.get("chunks")
    if ch is None:
        return 1, top
    return {"1": (1, 1), "2..limit-1": (2, limit - 1), "limit": (limit, limit), "<NS-1": (1, ns - 2), "NS-1": (ns - 1, ns - 1),
            "NS": (ns, ns), "NS+1": (ns + 1, ns + 1), "2NS+1": (2 * ns + 1, 2 * ns + 1), ">=3NS": (3 * ns, 3 * ns + 1)}[ch]


def select(want, sx, sm, sm_count, max_smem_optin, block=1 << 20):
    """smallest n ≥ 1 whose launch has every axis value in `want` (a partial `classify` dict; mode 0 unless `want` names
    one), or None if no n up to 3·max(NS, limit) + 1 chunks per CTA has it"""
    return _select(tuple(sorted(want.items())), sx, sm, sm_count, max_smem_optin, block)


@lru_cache(maxsize=None)
def _select(want_items, sx, sm, sm_count, max_smem_optin, block):
    want = dict(want_items)
    mode = want.get("mode", 0)
    ka, kb = _chunk_range(want, sx, sm, mode, max_smem_optin)
    if ka > kb:
        return None
    # CTA 0 has k chunks only if ⌈n/grid⌉ > (k − 1)·4096 − 8, and a full grid is needed for more than one
    lo = 1 if ka == 1 else sm_count * ((ka - 1) * K_CHUNK - 8) + 1
    hi = sm_count * kb * K_CHUNK + 8 * sm_count
    for start in range(lo, hi + 1, block):
        n = np.arange(start, min(start + block, hi + 1), dtype=np.int64)
        r = regimes(n, sx, sm, mode, sm_count, max_smem_optin)
        ok = np.ones(n.shape, bool)
        for axis, value in want.items():
            ok &= r[axis] == _code(axis, value)
        hit = np.flatnonzero(ok)
        if hit.size:
            return int(n[hit[0]])
    return None


# ---- the covering set: every kernel instance meets every reachable regime axis value --------------------------------
# Mode 0 unless stated.  Resident specs reach chunks 1 / 2…limit−1 / = limit, 1 / a few / a full grid of CTAs, a last CTA
# equal / shorter by chunks / ending in a partial chunk, and tails of 0, 1–7 and the whole tensor; the streamed specs the
# same with chunks < NS−1, NS−1, NS (mode 2 only: mode 0 streams from limit + 1 = NS + 1 on), NS+1 (the resident →
# streamed boundary), 2NS+1 and ≥ 3NS.
SPECS = (
    dict(kernel="resident", tail="n<8"),
    dict(kernel="resident", ctas="1", last="equal"),
    dict(kernel="resident", ctas="few", last="partial", tail="1-7"),
    dict(kernel="resident", chunks="1", ctas="grid", last="partial"),
    dict(kernel="resident", chunks="2..limit-1", last="fewer", tail="1-7"),
    dict(kernel="resident", chunks="limit", last="equal", tail="0"),
    dict(kernel="streamed", mode=2, tail="n<8"),
    dict(kernel="streamed", mode=2, ctas="1", tail="1-7"),
    dict(kernel="streamed", mode=2, ctas="few", last="equal"),
    dict(kernel="streamed", mode=2, chunks="NS-1", last="fewer", tail="1-7"),
    dict(kernel="streamed", mode=2, chunks="NS", last="partial"),
    dict(kernel="streamed", mode=0, chunks="NS+1", last="equal", tail="0"),
    dict(kernel="streamed", mode=0, chunks="2NS+1", last="fewer", tail="1-7"),
    dict(kernel="streamed", mode=2, chunks=">=3NS", last="partial", tail="1-7"),
)


@dataclass(frozen=True)
class Case:
    id: str
    tx: str                  # logits dtype
    tm: str                  # mask dtype
    spec: int

    @property
    def mode(self):
        return SPECS[self.spec].get("mode", 0)


def covering_cases():
    return [Case(f"{tx}-{tm}-s{j}", tx, tm, j) for tx, tm in PAIRS for j in range(len(SPECS))]


def resolve(case: Case, sm_count, max_smem_optin):
    """(n, launch) of the case on this device; n is None if its regime is unreachable"""
    sx, sm = DTYPE_BYTES[case.tx], DTYPE_BYTES[case.tm]
    n = select(SPECS[case.spec], sx, sm, sm_count, max_smem_optin)
    return n, (None if n is None else launch(n, sx, sm, case.mode, sm_count, max_smem_optin))


def instance(kernel, tx, tm):
    name = {"resident": "loss_bce_cel_kernel", "streamed": "loss_stream_kernel"}[kernel]
    return f"{name}<{tx},{tm}>"


def cells(case: Case, g: Launch, sm_count):
    cls = classify(g, sm_count)
    inst = instance(g.kernel, case.tx, case.tm)
    return {(inst, axis, v) for axis, v in cls.items() if v is not None}


def required_cells():
    """every reachable (instance, axis, value) of the ten instances"""
    return {(instance(k, tx, tm), axis, v) for tx, tm in PAIRS for k in AXES["kernel"] for axis, vals in AXES.items()
            for v in vals if reachable(k, axis, v)}
