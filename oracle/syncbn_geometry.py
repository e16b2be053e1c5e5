"""ORACLE (test infrastructure only): the launch geometry of the SyncBN kernels, restated from csrc/syncbn.cu.

`make_geom` is the host function of the same name with the device (SM count, opt-in shared memory per block) as
arguments instead of a query, so the tests can ask which code path a launch takes on any GPU.  On top of it:

* `fwd_site` / `bwd_site`: the stream count and chunk cap each call site passes (sod_syncbn_fwd: 1 + pre streams,
  32 KB chunks, 16 KB with a residual; sod_syncbn_bwd: dy, x, pre?, y? streams, 32 KB);
* `classify`: the ring regime of a geometry — chunks per full strip against the stage count NS, the length of the
  last strip, whether the last chunk is partial, how many strips — i.e. which branches of the ring protocol
  (tests/test_ring_protocol_model.py) and of the hop-1 exchange a launch exercises;
* `select`: the smallest row count (for a given C, or the smallest over a list of C) whose geometry has a requested
  regime, so a test reaches the same branches on a 132-SM H100 as on a 148-SM part.
"""
from __future__ import annotations

from dataclasses import dataclass
from functools import lru_cache

K_THREADS = 512
K_MAX_C = 2048
K_MAX_STAGES = 16
K_MAX_GRID = 160
K_RED_BYTES = 49152
K_SMEM_FIXED = 256 + K_RED_BYTES + 3 * K_MAX_C * 4
TRAFFIC_DIV = 4                       # SOD_BN_TRAFFIC_DIV default

CHANNELS = (8, 16, 64, 256, 2048)     # L = C/8 = 1 … 256: every branch of cta_reduce (the C axis of the regimes)
SEARCH_CHANNELS = (8, 16, 32, 64, 128, 256, 512, 1024, 2048)
N_CLASSES = ("1", "NS-1", "NS", "NS+1", "2NS+1")
LAST_CLASSES = ("equal", "one", "ns+1", "shorter")
STRIP_CLASSES = ("1", "few", "grid")   # few: 2-8 strips; "many" (9 … grid-1) is not a target
FEW_MAX = 8


@dataclass(frozen=True)
class Geom:
    C: int
    es: int
    chunk_bytes: int
    chunk_rows: int
    ppt: int
    nstream: int
    nstage: int
    strips: int
    chunks_per_strip: int
    rows: int
    total_chunks: int


def make_geom(rows, C, es, nstream, max_chunk, sm_count, max_smem_optin):
    """csrc/syncbn.cu make_geom; None where the host function returns SOD_EUNSUPPORTED"""
    chunk = max_chunk
    while nstream * chunk > 49152:
        chunk >>= 1
    L = C // 8
    if rows <= 0 or C <= 0 or C % 8 or C > K_MAX_C or (L & (L - 1)) or L > 256:
        return None
    while C * es > chunk:
        chunk *= 2
    chunk_rows = chunk // (C * es)
    ppt = -(-(chunk // (8 * es)) // K_THREADS)
    budget = max_smem_optin - K_SMEM_FIXED - 1024
    nstage = min(budget // (nstream * chunk), K_MAX_STAGES)
    if nstage < 2:
        return None
    total = -(-rows // chunk_rows)
    by_traffic = max((rows * C * es) // (TRAFFIC_DIV * 2 * C * 8), 1)
    cap = min(sm_count, K_MAX_GRID, by_traffic)
    strips = min(total, cap)
    cps = -(-total // strips)
    strips = -(-total // cps)
    return Geom(C, es, chunk, chunk_rows, ppt, nstream, nstage, strips, cps, rows, total)


def fwd_site(pre, res):
    """(nstream, max_chunk) of sod_syncbn_fwd"""
    return (2 if pre else 1), (16384 if res else 32768)


def bwd_site(pre, relu, xmask):
    """(nstream, max_chunk) of sod_syncbn_bwd: dy, x, then pre, then y unless the mask comes from x"""
    return 2 + int(pre) + int(relu and not xmask), 32768


def grid_cap(sm_count):
    return min(sm_count, K_MAX_GRID)


def classify(g: Geom, sm_count):
    """the regime of a launch (axis → class); `n` is None when chunks per strip is none of the tracked values"""
    NS, n = g.nstage, g.chunks_per_strip
    n_cls = {1: "1", NS - 1: "NS-1", NS: "NS", NS + 1: "NS+1", 2 * NS + 1: "2NS+1"}.get(n)
    last = g.total_chunks - (g.strips - 1) * n
    if last == n:
        last_cls = "equal"
    elif last == 1:
        last_cls = "one"
    elif last == NS + 1:
        last_cls = "ns+1"
    else:
        last_cls = "shorter"
    if g.strips == 1:
        strips_cls = "1"
    elif g.strips == grid_cap(sm_count):
        strips_cls = "grid"             # min(#SMs, 160) CTAs: above 128 the 5th hop-1b packet per lane is used
    else:
        strips_cls = "few" if g.strips <= FEW_MAX else "many"
    partial = g.rows % g.chunk_rows != 0
    return dict(n=n_cls, last=last_cls, partial=partial, strips=strips_cls, C=g.C)


def matches(cls, want):
    return all(cls[k] == v for k, v in want.items())


def select(want, es, nstream, max_chunk, sm_count, max_smem_optin):
    """smallest (by bytes) geometry whose regime has every axis value in `want` (a partial `classify` dict); `want["C"]`,
    if present, fixes C, else every channel count of SEARCH_CHANNELS is tried.  Returns None if no row count reaches it."""
    return _select(tuple(sorted(want.items())), es, nstream, max_chunk, sm_count, max_smem_optin)


@lru_cache(maxsize=None)
def _select(want_items, es, nstream, max_chunk, sm_count, max_smem_optin):
    want = dict(want_items)
    best = None
    for C in ((want["C"],) if "C" in want else SEARCH_CHANNELS):
        g0 = make_geom(1, C, es, nstream, max_chunk, sm_count, max_smem_optin)
        if g0 is None:
            continue
        cr = g0.chunk_rows
        max_total = grid_cap(sm_count) * (2 * g0.nstage + 1)      # beyond: more than 2NS+1 chunks per strip
        # rows grow with the chunk count: the first total chunk count that matches gives the smallest tensor for this C
        for total in range(1, max_total + 1):
            if best is not None and (total - 1) * cr * C >= best.rows * best.C:
                break
            cands = [total * cr]
            if cr > 1:
                cands = [(total - 1) * cr + 1, (total - 1) * cr + cr // 2, total * cr - 1, total * cr]
            hit = None
            for rows in cands:
                g = make_geom(rows, C, es, nstream, max_chunk, sm_count, max_smem_optin)
                if g is not None and matches(classify(g, sm_count), want):
                    hit = g
                    break
            if hit is not None:
                if best is None or hit.rows * C < best.rows * best.C:
                    best = hit
                break
    return best


def shape_of(g: Geom):
    """an (N, C, H, W) with N·H·W = rows: two images when the row count is even, so N > 1 is exercised"""
    if g.rows % 2 == 0 and g.rows > 2:
        return (2, g.C, g.rows // 2, 1)
    return (1, g.C, g.rows, 1)


# ---- the covering set: every kernel instance meets every regime axis value ------------------------------------------
# One spec per row; together they reach every value of every axis (chunks per strip, last strip, last chunk, strips, C).
SPECS = (
    dict(n="1", strips="grid", C=8),
    dict(n="NS-1", last="one", C=16),
    dict(n="NS", partial=True, last="shorter", C=64),
    dict(n="NS+1", last="equal", partial=False, C=256),
    dict(n="NS+1", strips="few"),
    dict(n="2NS+1", last="ns+1"),
    dict(strips="1", C=2048),
)
AXES = dict(n=N_CLASSES, last=LAST_CLASSES, partial=(False, True), strips=STRIP_CLASSES, C=CHANNELS)
DTYPE_BYTES = {"float32": 4, "bfloat16": 2, "float16": 2}
FWD_SITES = (dict(pre=False, res=False), dict(pre=True, res=False), dict(pre=False, res=True), dict(pre=True, res=True))
# backward call sites: 2 (dy, x), 3 (+ y), 4 (+ pre + y) streams; the mask-from-x variant drops the y stream
BWD_SITES = (dict(pre=False, relu=False, res=False), dict(pre=False, relu=True, res=True),
             dict(pre=True, relu=True, res=True), dict(pre=True, relu=True, res=False))
BWD_SITES_XMASK = (dict(pre=False, relu=True, res=False), dict(pre=True, relu=True, res=False))


@dataclass(frozen=True)
class Case:
    id: str
    kind: str            # "fwd": training + eval forward; "bwd": training forward + backward (the backward is the target)
    dtype: str
    pre: bool
    res: bool
    relu: bool
    spec: int
    xmask: bool = False  # SOD_BN_BWD_MASK_FROM_X requested (used when relu and no residual)
    hint: bool = False   # SOD_BN_L2_HINTS
    nbias: int = 0       # folded conv biases
    bias_fp32: bool = False
    into: bool = False   # γ/β gradients accumulated into bound .grad buffers


def covering_cases():
    cases = []
    for dt in DTYPE_BYTES:
        for si, site in enumerate(FWD_SITES):
            for j in range(len(SPECS)):
                cases.append(Case(f"fwd-{dt}-pre{int(site['pre'])}res{int(site['res'])}-s{j}", "fwd", dt, site["pre"], site["res"],
                                  relu=(j + si) % 2 == 0, spec=j, nbias=j % 3, bias_fp32=j % 2 == 1))
        for fold in (False, True):
            for hint in (False, True):
                for xmask in (False, True):
                    i = 2 * fold + hint
                    sites = BWD_SITES_XMASK if xmask else BWD_SITES
                    for j in range(len(SPECS)):
                        site = sites[(i + j) % len(sites)]
                        cases.append(Case(f"bwd-{dt}-f{int(fold)}h{int(hint)}x{int(xmask)}-pre{int(site['pre'])}relu{int(site['relu'])}"
                                          f"res{int(site['res'])}-s{j}", "bwd", dt, site["pre"], site["res"], site["relu"], spec=j,
                                          xmask=xmask, hint=hint, nbias=(1 + j % 2) if fold else 0, bias_fp32=fold and (j // 2) % 2 == 1,
                                          into=(i + j) % 3 == 0))
    return cases


def target_site(case: Case):
    """(nstream, max_chunk) of the launch whose regime the case selects"""
    if case.kind == "fwd":
        return fwd_site(case.pre, case.res)
    return bwd_site(case.pre, case.relu, case.xmask and case.relu and not case.res)


def resolve(case: Case, sm_count, max_smem_optin):
    """the target launch's geometry on this device (None: the spec is unreachable)"""
    return select(SPECS[case.spec], DTYPE_BYTES[case.dtype], *target_site(case), sm_count, max_smem_optin)


def instances(case: Case, g: Geom):
    """names of the kernel instances the target launch runs (the forward's template depends on the geometry: PPT)"""
    if case.kind == "fwd":
        name = f"syncbn_fwd_kernel<{case.dtype},{g.ppt},{str(case.res).lower()}>"
        return (name + " train", name + " eval")
    return (f"syncbn_bwd_kernel<{case.dtype},{24 if case.nbias else 16},{str(case.xmask).lower()},{str(case.hint).lower()}>",)


def cells(case: Case, g: Geom, sm_count):
    cls = classify(g, sm_count)
    return {(inst, axis, cls[axis]) for inst in instances(case, g) for axis in AXES}


def required_cells(case_cells):
    """every axis value for every instance that appears in `case_cells`"""
    return {(inst, axis, v) for inst in {c[0] for c in case_cells} for axis, vals in AXES.items() for v in vals}
