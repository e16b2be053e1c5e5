"""ORACLE (test infrastructure only): the launch geometry of the world-1 optimizer and gradient kernels, restated from
the host side of csrc/sgd.cu with the SM count as an argument.

* `local_step_kernel` (`sod_sgd_momentum`, `sod_adam` and their `*_scaler` forms) runs min(⌈nvec/2048⌉, 2·#SMs) CTAs of
  512 threads over nvec = n/4 float4 vectors.  With T = grid·512, thread t visits t + k·4T + u·T for u < 4 while
  t + k·4T < nvec (each vector still bounds-checked): one pass covers 4T vectors.  Cells: one CTA (nvec ≤ 2048), several
  CTAs with a ragged last one, the cap reached in exactly one pass (nvec = 4T), the cap reached with a partly live unroll
  group (nvec < 4T), two or more passes exact or ragged.  A segment edge b (in vectors) falls inside one thread's unroll
  group (`unroll`: b mod T ≠ 0 and ⌊b/T⌋ mod 4 < 3, so the cursor advances between u and u + 1), at a CTA edge
  (b mod 512 = 0), at a T boundary or at a pass boundary (b mod 4T = 0).
* `grad_gather16_kernel` (`sod_grad_gather16[_checked]`) splits each item into 8192-element chunks; one launch per batch of
  160 items runs min(chunks, 8·#SMs) CTAs of 256 threads, CTA c doing chunks c, c + grid, …  Inside a chunk a 16-byte
  aligned source is copied as uint4 vectors and then a scalar tail of numel mod 8 (at the item's last chunk); any other
  source (src mod 16 ∈ {2, …, 14}) element by element.
* `grad_check_ranges_kernel` (`sod_grad_check_ranges`): the same split with 4096-element chunks, min(chunks, 4·#SMs) CTAs
  and batches of 128 ranges; empty ranges take no chunk, and a batch of empty ranges launches nothing.
* `grad_nonfinite_kernel` and `grad_merge16_kernel`: min(⌈nvec/1024⌉, cap) CTAs of 256 threads, cap 4·#SMs and 8·#SMs,
  grid-stride by grid·256 vectors — so a thread makes up to four passes below the cap and more once the cap is reached.

`step_cells` / `gather_cells` / `check_cells` / `flat_cells` classify one launch, and `select(kind, cell, sm)` returns the
smallest shape reaching a cell on `sm` SMs.
"""
from __future__ import annotations

STEP_THREADS = 512
STEP_UNROLL = 4
STEP_CTAS_PER_SM = 2
GATHER_THREADS = 256
GATHER_CHUNK = 8192
GATHER_CTAS_PER_SM = 8
GATHER_MAX_ITEMS = 160
CHECK_THREADS = 256
CHECK_CHUNK = 4096
CHECK_CTAS_PER_SM = 4
CHECK_MAX_RANGES = 128
FLAT_THREADS = 256
FLAT_VEC_PER_CTA = 1024
NONFINITE_CTAS_PER_SM = 4
MERGE_CTAS_PER_SM = 8

STEP_CELLS = ("1cta", "ctas ragged", "cap 1 pass", "cap partial group", ">=2 passes exact", ">=2 passes ragged")
EDGE_CLASSES = ("unroll", "cta", "T", "pass")
GATHER_CELLS = ("small", "tail", "misaligned", "2 passes", "2 launches")
CHECK_CELLS = ("empty", "all-empty batch", "2 passes", "2 launches")
FLAT_CELLS = ("1 pass", "below cap", "cap")


def cdiv(a, b):
    return -(-a // b)


# ---- local step ----------------------------------------------------------------------------------------------------
def step_grid(nvec, sm):
    return min(cdiv(nvec, STEP_THREADS * STEP_UNROLL), STEP_CTAS_PER_SM * sm)


def step_stride(nvec, sm):
    return step_grid(nvec, sm) * STEP_THREADS


def step_visits(nvec, sm):
    """per thread, the vectors it visits in order"""
    T = step_stride(nvec, sm)
    out = []
    for t in range(T):
        v = []
        for i0 in range(t, nvec, STEP_UNROLL * T):
            v.extend(i for i in range(i0, i0 + STEP_UNROLL * T, T) if i < nvec)
        out.append(v)
    return out


def step_cells(nvec, sm):
    g, T = step_grid(nvec, sm), step_stride(nvec, sm)
    cap, full = STEP_CTAS_PER_SM * sm, STEP_UNROLL * step_stride(nvec, sm)
    cells = set()
    if g == 1:
        cells.add("1cta")
    if g > 1 and nvec % (STEP_THREADS * STEP_UNROLL) and nvec < full:
        cells.add("ctas ragged")
    if g == cap and nvec == full:
        cells.add("cap 1 pass")
    if g == cap and nvec < full:
        cells.add("cap partial group")
    if nvec >= 2 * full and nvec % full == 0:
        cells.add(">=2 passes exact")
    if nvec > full and nvec % full:
        cells.add(">=2 passes ragged")
    return cells


def edge_class(b, nvec, sm):
    """where a segment edge at vector b (0 < b < nvec) falls in the visit order, or None"""
    T = step_stride(nvec, sm)
    if b % (STEP_UNROLL * T) == 0:
        return "pass"
    if b % T == 0:
        return "T"
    if b % STEP_THREADS == 0:
        return "cta"
    if (b // T) % STEP_UNROLL < STEP_UNROLL - 1:
        return "unroll"
    return None


def edge_at(cls, nvec, sm):
    """the smallest edge 0 < b < nvec of class `cls`, or None"""
    T = step_stride(nvec, sm)
    cand = {"pass": [STEP_UNROLL * T], "T": [T, 2 * T, 3 * T], "cta": [STEP_THREADS * k for k in range(1, 4)],
            "unroll": [1, T // 2 + 1]}[cls]
    for b in cand:
        if 0 < b < nvec and edge_class(b, nvec, sm) == cls:
            return b
    return None


# ---- gather / check ranges -----------------------------------------------------------------------------------------
def batches(count, per):
    return [range(b, min(b + per, count)) for b in range(0, count, per)]


def gather_launches(numels, sm):
    """per launch: (items, chunk prefix sums, grid)"""
    out = []
    for bt in batches(len(numels), GATHER_MAX_ITEMS):
        c0 = [0]
        for i in bt:
            c0.append(c0[-1] + cdiv(numels[i], GATHER_CHUNK))
        out.append((list(bt), c0, min(c0[-1], GATHER_CTAS_PER_SM * sm)))
    return out


def gather_chunk_cta(numels, sm):
    """(launch, item, chunk of the item) → (CTA, pass) of every chunk"""
    out = {}
    for li, (items, c0, grid) in enumerate(gather_launches(numels, sm)):
        for k, i in enumerate(items):
            for c in range(c0[k], c0[k + 1]):
                out[(li, i, c - c0[k])] = (c % grid, c // grid)
    return out


def gather_elements(numel, src_misalign_bytes):
    """per chunk of one item: (vector element ranges, scalar element indices) in the chunk's own order"""
    out = []
    for first in range(0, numel, GATHER_CHUNK):
        cnt = min(GATHER_CHUNK, numel - first)
        if src_misalign_bytes % 16 == 0:
            nv = cnt >> 3
            out.append(([range(first + 8 * i, first + 8 * i + 8) for i in range(nv)], list(range(first + 8 * nv, first + cnt))))
        else:
            out.append(([], list(range(first, first + cnt))))
    return out


def gather_cells(numels, misalign, sm):
    cells = set()
    if any(x < 8 for x in numels):
        cells.add("small")
    if any(x % 8 for x in numels):
        cells.add("tail")
    if any(m % 16 for m in misalign):
        cells.add("misaligned")
    launches = gather_launches(numels, sm)
    if any(c0[-1] > grid for _, c0, grid in launches):
        cells.add("2 passes")
    if len(launches) > 1:
        cells.add("2 launches")
    return cells


def check_launches(lengths, sm):
    """per launch: (non-empty range indices, chunk prefix sums, grid); a batch without chunks launches nothing (None)"""
    out = []
    for bt in batches(len(lengths), CHECK_MAX_RANGES):
        live = [i for i in bt if lengths[i] > 0]
        c0 = [0]
        for i in live:
            c0.append(c0[-1] + cdiv(lengths[i], CHECK_CHUNK))
        out.append((live, c0, min(c0[-1], CHECK_CTAS_PER_SM * sm)) if c0[-1] else None)
    return out


def check_cells(lengths, sm):
    cells = set()
    if any(x == 0 for x in lengths):
        cells.add("empty")
    launches = check_launches(lengths, sm)
    if any(x is None for x in launches):
        cells.add("all-empty batch")
    if any(x is not None and x[1][-1] > x[2] for x in launches):
        cells.add("2 passes")
    if len(launches) > 1:
        cells.add("2 launches")
    return cells


# ---- nonfinite / merge ----------------------------------------------------------------------------------------------
def flat_cap(kind, sm):
    return (NONFINITE_CTAS_PER_SM if kind == "nonfinite" else MERGE_CTAS_PER_SM) * sm


def flat_grid(kind, nvec, sm):
    return min(cdiv(nvec, FLAT_VEC_PER_CTA), flat_cap(kind, sm))


def flat_visits(kind, nvec, sm):
    stride = flat_grid(kind, nvec, sm) * FLAT_THREADS
    return [range(t, nvec, stride) for t in range(stride)]


def flat_cells(kind, nvec, sm):
    g = flat_grid(kind, nvec, sm)
    if nvec <= g * FLAT_THREADS:
        return {"1 pass"}
    return {"cap"} if g == flat_cap(kind, sm) else {"below cap"}


# ---- selection -----------------------------------------------------------------------------------------------------
def select(kind, cell, sm):
    """the smallest shape reaching `cell`: nvec (step, nonfinite, merge), a list of numels (gather) or of range lengths
    (check)"""
    if kind == "step":
        per, cap = STEP_THREADS * STEP_UNROLL, STEP_CTAS_PER_SM * sm
        full = cap * per
        nvec = {"1cta": 1, "ctas ragged": per + 1, "cap 1 pass": full, "cap partial group": (cap - 1) * per + 1,
                ">=2 passes exact": 2 * full, ">=2 passes ragged": full + 1}[cell]
        assert cell in step_cells(nvec, sm), (cell, nvec, sm)
        return nvec
    if kind in ("nonfinite", "merge"):
        nvec = {"1 pass": 1, "below cap": FLAT_THREADS + 1, "cap": flat_cap(kind, sm) * FLAT_VEC_PER_CTA + 1}[cell]
        assert flat_cells(kind, nvec, sm) == {cell}, (kind, cell, nvec, sm)
        return nvec
    if kind == "gather":
        shape = {"small": [3], "tail": [13], "misaligned": [24], "2 passes": [(GATHER_CTAS_PER_SM * sm + 1) * GATHER_CHUNK],
                 "2 launches": [8] * (GATHER_MAX_ITEMS + 1)}[cell]
        return shape
    if kind == "check":
        shape = {"empty": [0, 5], "all-empty batch": [0] * CHECK_MAX_RANGES + [5],
                 "2 passes": [(CHECK_CTAS_PER_SM * sm + 1) * CHECK_CHUNK], "2 launches": [1] * (CHECK_MAX_RANGES + 1)}[cell]
        assert cell in check_cells(shape, sm), (cell, sm)
        return shape
    raise KeyError(kind)
