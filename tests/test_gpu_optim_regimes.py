"""The optimizer-step, gradient-gather, overflow-check and merge kernels of csrc/sgd.cu in every launch regime of this GPU,
bit for bit against the fp32 replay of oracle/optim_replay.py or exact copies, through the C ABI.

oracle/optim_geometry.py picks, for the device the test runs on, the shapes that reach each regime cell: the step
kernel's single CTA, several CTAs with a ragged last one, the 2·#SMs cap reached in exactly one pass or with a partly
live unroll group, and two or more grid-stride passes (exact and ragged); segment edges inside one thread's unroll group,
at a CTA edge, at a T = grid·512 boundary and at a pass boundary; the gather's scalar tails, misaligned sources, second
grid-stride pass and second launch; the range check's empty ranges, all-empty batch, second pass and second launch; and
the nonfinite / merge kernels below and at their caps.  Outputs that a launch must not write are filled with a sentinel
first.  The last test asserts that every cell ran.

Bounds.  The world-1 step is exactly reproducible, so p, the optimizer state and the 16-bit shadow must equal the replay
bit for bit (non-finite values by class: CUDA's NaN payload is not numpy's).  The one assumption is the margin on
CUDA's double `pow` in Adam's bias corrections (oracle/optim_replay.py); every (lr, β, t) used here is checked against it
on the CPU by tests/test_optim_replay_cpu.py and again below.  Copies, merges and flags are exact.
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

from oracle import optim_geometry as geo
from oracle import optim_replay as rp

pytestmark = pytest.mark.gpu

RAN: set = set()
SENT16 = 0x5A5A
RULES = ("sgd", "nesterov", "adam")
G16 = (None, "bfloat16", "float16")
MODES = ("arg", "scaler")
SGD_LRS, WDS, MUS = (0.05, 0.01, 0.2, 1e-3), (5e-4, 0.0, 1e-2), (0.9, 0.5, 0.0, 0.99)
ADAM_LRS = (1e-3, 2e-3, 0.05, 0.1)              # tests/test_optim_replay_cpu.py LRS: all clear the pow margin
BETAS = ((0.9, 0.999), (0.8, 0.99), (0.5, 0.75), (0.95, 0.9999))
EPSS = (1e-8, 0.0, 1e-6)
STEPS = (0, 1, 10_000, 1_000_000)


def _sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _l():
    from distributed_sod_project_b200 import _lib
    return _lib


def L():
    return _l().lib()


def sp():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return t.data_ptr() if t is not None else None


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _same(got, want):
    """bit-equal, with any NaN equal to any NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    return (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))


def _assert_same(got, want, what):
    ok = _same(got, want)
    if not ok.all():
        i = int(np.flatnonzero(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.size} differ, first at {i}: {got[i]!r} vs {want[i]!r}")


def _f16(x, dtype):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(getattr(torch, dtype))


def _bits16(t):
    return t.contiguous().view(torch.int16).cpu().numpy().astype(np.uint16)


# ---------------------------------------------------------------------------------------------------------------------
# step kernels
# ---------------------------------------------------------------------------------------------------------------------
def _layout(nvec, sm, rule, nseg16=False):
    """segment table (element offsets) with edges of every class the shape allows, and the shape cells it reaches"""
    if nseg16:
        bounds = [0] + [nvec * k // 16 for k in range(1, 16)] + [nvec]
        raw = [(bounds[i], bounds[i + 1]) for i in range(16)]
    else:
        pts = {1, 2, nvec - 1} | {geo.edge_at(c, nvec, sm) for c in geo.EDGE_CLASSES}
        pts = sorted(b for b in pts if b is not None and 0 < b < nvec)
        bounds = [0] + pts + [nvec]
        raw = [(bounds[i], bounds[i + 1]) for i in range(len(bounds) - 1)]
    table, shapes = [], set()
    for i, (b, e) in enumerate(raw):
        if not nseg16 and i == 3 and len(raw) > 5:
            shapes.add("gap")
            continue
        flags = (rp.GRAD16 if i % 3 == 0 else 0) | (rp.FROZEN if i == 2 else 0)
        if rule == "nesterov" and i % 2 == 0:
            flags |= rp.NESTEROV
        table.append((b, e, flags, i))
        if not nseg16 and i == 1:
            table.append((e, e, 0, i + 100))
            shapes.add("empty")
    table = table[:16]
    segs = []
    for k, (b, e, flags, i) in enumerate(table):
        s = dict(begin=4 * b, end=4 * e, flags=flags, wd=float(np.float32(WDS[i % 3])))
        if rule == "adam":
            b1, b2 = BETAS[i % 4]
            s.update(lr=float(np.float32(ADAM_LRS[(i // 2) % 4])), beta1=b1, beta2=b2, eps=EPSS[i % 3])
        else:       # neighbours share lr but differ in wd and mu
            s.update(lr=float(np.float32(SGD_LRS[(i // 2) % 4])), mu=float(np.float32(MUS[i % 4])))
        if e - b == 1:
            shapes.add("float4")
        if flags & rp.FROZEN:
            shapes.add("frozen")
        segs.append(s)
    if segs and segs[-1]["end"] == 4 * nvec:
        shapes.add("ends at n")
    if nseg16 and len(segs) == 16:
        shapes.add("16 segments")
    edges = {geo.edge_class(x // 4, nvec, sm) for s in segs for x in (s["begin"], s["end"]) if 0 < x < 4 * nvec}
    return segs, shapes, edges - {None}


def _seg_array(rule, segs, lr_by_value):
    l = _l()
    if rule == "adam":
        arr = (l.sod_adam_segment * max(len(segs), 1))()
        for i, s in enumerate(segs):
            arr[i] = l.sod_adam_segment(s["begin"], s["end"], s["lr"] if lr_by_value else 123.0, s["wd"], s["beta1"], s["beta2"],
                                        s["eps"], s["flags"])
    else:
        arr = (l.sod_sgd_segment * max(len(segs), 1))()
        for i, s in enumerate(segs):
            arr[i] = l.sod_sgd_segment(s["begin"], s["end"], s["lr"] if lr_by_value else 123.0, s["wd"], s["mu"], s["flags"])
    return arr


def _inputs(n, rule, tier, g16, seed):
    rng = np.random.default_rng(seed)
    spread = lambda lo, hi: (rng.standard_normal(n) * np.exp2(rng.integers(lo, hi, n))).astype(np.float32)  # noqa: E731
    p, s0, g32 = spread(-6, 6), spread(-10, 2), spread(-12, 4)
    state = [s0] + ([np.abs(spread(-24, 0))] if rule == "adam" else [])
    h = spread(-12, 4) if g16 else None
    if tier == "special":
        k = max(n // 97, 1)
        idx = rng.permutation(n)[:12 * k].reshape(12, k) if n >= 12 * k else rng.integers(0, n, (12, k))
        g32[idx[0]], g32[idx[1]], g32[idx[2]] = np.inf, -np.inf, np.nan
        g32[idx[3]] = np.float32(1e-41) * np.sign(rng.standard_normal(k)).astype(np.float32)   # subnormal
        g32[idx[4]] = -0.0
        p[idx[5]] = (rng.choice([-1, 1], k) * np.exp2(rng.integers(16, 40, k))).astype(np.float32)  # beyond fp16
        p[idx[6]] = -0.0
        state[-1][idx[7]] = 0.0
        g32[idx[7]] = 0.0
        p[idx[7]] = 0.0
        if h is not None:
            h[idx[8]], h[idx[9]], h[idx[10]] = np.inf, np.nan, -np.inf
            h[idx[11]] = np.float32(6e-8 if g16 == "float16" else 1e-39)
    if tier == "ties":      # p at bf16 ties (low half 0x8000) and fp16 ties (low 13 bits 0x1000, fp16 normal range)
        sign = rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)
        bf = sign | (rng.integers(100, 150, n, dtype=np.uint32) << np.uint32(23)) | \
            (rng.integers(0, 1 << 7, n, dtype=np.uint32) << np.uint32(16)) | np.uint32(0x8000)
        hf = sign | (rng.integers(113, 142, n, dtype=np.uint32) << np.uint32(23)) | \
            (rng.integers(0, 1 << 10, n, dtype=np.uint32) << np.uint32(13)) | np.uint32(0x1000)
        p = np.where(rng.random(n) < 0.5, bf, hf).astype(np.uint32).view(np.float32)
    h16 = _f16(h, g16) if g16 else None
    return p, state, g32, h16


def _run_step(rule, cell_nvec, segs, tier, g16, mode, lr_dev, zero, seed, steps=None, expect=True):
    l = _l()
    n = 4 * cell_nvec
    p0, st0, g0, h0 = _inputs(n, rule, tier, g16, seed)
    if tier == "ties":
        segs = [dict(s, lr=0.0) for s in segs]
    dev = lambda a: torch.from_numpy(a.copy()).cuda()  # noqa: E731
    p, st, g = dev(p0), [dev(s) for s in st0], dev(g0)
    h = h0.cuda() if h0 is not None else None
    shadow = torch.full((n,), SENT16, dtype=torch.int16, device="cuda").view(getattr(torch, g16)) if g16 else None
    flags = (l.SOD_SGD_ZERO_GRAD if zero else 0) | (l.SOD_GRAD16_F16 if g16 == "float16" else 0)
    arr = _seg_array("adam" if rule == "adam" else "sgd", segs, not lr_dev)
    lr_t = torch.tensor([s["lr"] for s in segs] + [0.0] * (16 - len(segs)), dtype=torch.float32, device="cuda") if lr_dev else None
    steps = list(steps if steps is not None else [STEPS[i % 4] for i in range(len(segs))])
    step_dev = torch.zeros(l.SOD_ADAM_STEP_WORDS, dtype=torch.int32)
    step_dev[:len(steps)] = torch.tensor(steps, dtype=torch.int32)
    step_dev = step_dev.cuda()
    scale, gi, unsk = 3.0, 2, 1
    scaler = torch.zeros(l.SOD_LOSS_SCALER_WORDS, dtype=torch.int32)
    scaler[2], scaler[3] = unsk, gi
    scaler.view(torch.float32)[1] = scale
    scaler = scaler.cuda()
    inv = 0.3
    if rule == "adam":
        for s, c in zip(segs, steps):
            assert rp.adam_scalars_stable(s["lr"], s["beta1"], s["beta2"], c), (s, c)
        if mode == "scaler":
            rc = L().sod_adam_scaler(ptr(p), ptr(st[0]), ptr(st[1]), ptr(g), ptr(h), ptr(shadow), n, arr, len(segs), ptr(lr_t),
                                     ptr(step_dev), ptr(scaler), flags, sp())
        else:
            rc = L().sod_adam(ptr(p), ptr(st[0]), ptr(st[1]), ptr(g), ptr(h), ptr(shadow), n, arr, len(segs), ptr(lr_t),
                              ptr(step_dev), inv, None, flags, sp())
    else:
        if mode == "scaler":
            rc = L().sod_sgd_momentum_scaler(ptr(p), ptr(st[0]), ptr(g), ptr(h), ptr(shadow), n, arr, len(segs), ptr(lr_t),
                                             ptr(scaler), flags, sp())
        else:
            rc = L().sod_sgd_momentum(ptr(p), ptr(st[0]), ptr(g), ptr(h), ptr(shadow), n, arr, len(segs), ptr(lr_t), inv,
                                      None, flags, sp())
    assert rc == 0
    torch.cuda.synchronize()
    hv = h0.float().numpy() if h0 is not None else None
    kw = dict(scale=scale) if mode == "scaler" else dict(inv_scale=inv)
    we = rp.step("adam" if rule == "adam" else "sgd", p0, st0, g0, hv, segs, zero_grad=zero, steps=steps, **kw)
    wp, wst, wg, wh, upd = we
    _assert_same(p.cpu().numpy(), wp, "p")
    for k, (a, b) in enumerate(zip(st, wst)):
        _assert_same(a.cpu().numpy(), b, f"state {k}")
    _assert_same(g.cpu().numpy(), wg, "fp32 gradient")
    if h is not None:
        _assert_same(h.float().cpu().numpy(), wh, "16-bit gradient")
        sh = _bits16(shadow)
        want = _bits16(_f16(wp, g16))
        nan = np.isnan(wp) & upd
        assert np.array_equal(sh[upd & ~nan], want[upd & ~nan]), "shadow"
        assert np.all((sh[nan] & 0x7FFF) > (0x7F80 if g16 == "bfloat16" else 0x7C00)), "shadow NaN"
        assert np.all(sh[~upd] == SENT16), "shadow written outside the updated elements"
    sd = step_dev.cpu().tolist()
    if rule == "adam":
        assert sd[:len(steps)] == rp.next_steps(steps, segs, False) and sd[len(steps):] == [0] * (17 - len(steps))
    else:
        assert sd == steps + [0] * (17 - len(steps))
    sc = scaler.cpu()
    if mode == "scaler":
        assert (float(sc.view(torch.float32)[1]), int(sc[2])) == rp.scaler_next(scale, unsk, gi, False)
        assert int(sc[0]) == 0 and int(sc[4]) == 0
    else:
        assert float(sc.view(torch.float32)[1]) == scale and int(sc[2]) == unsk
    return upd


CASES = [(cell, rule, gi, mi) for cell in geo.STEP_CELLS for rule in RULES for gi in range(3) for mi in range(2)]


@pytest.mark.parametrize("cell,rule,gi,mi", CASES, ids=[f"{c}-{r}-{G16[g]}-{MODES[m]}" for c, r, g, m in CASES])
def test_step_regimes(cell, rule, gi, mi):
    sm = _sm()
    nvec = geo.select("step", cell, sm)
    if cell == ">=2 passes ragged":
        nvec += 7
    ri = RULES.index(rule)
    zero = (gi + ri) % 2 == 0
    lr_dev = (gi + mi + ri) % 2 == 1
    g16, mode = G16[gi], MODES[mi]
    segs, shapes, edges = _layout(nvec, sm, rule)
    tiers = ["random"]
    if cell in ("1cta", ">=2 passes ragged", "ctas ragged"):
        tiers.append("special")
    if cell == "cap partial group" and g16:
        tiers.append("ties")
    for tier in tiers:
        _run_step(rule, nvec, segs, tier, g16, mode, lr_dev, zero, _seed(cell, rule, gi, mi, tier))
        RAN.add(("tier", tier))
    RAN.update({("step", cell), ("step", rule, g16, mode), ("combo", rule, lr_dev, zero)})
    RAN.update(("edge", e) for e in edges)
    RAN.update(("shape", s) for s in shapes)


@pytest.mark.parametrize("rule", RULES)
def test_step_16_segments_and_none(rule):
    sm = _sm()
    nvec = geo.select("step", ">=2 passes ragged", sm) + 333
    segs, shapes, _ = _layout(nvec, sm, rule, nseg16=True)
    assert len(segs) == 16
    _run_step(rule, nvec, segs, "random", "bfloat16", "scaler", True, True, _seed("16", rule))
    # nseg = 0: nothing updated, gradients still cleared, the scaler still advances, no step count moves
    upd = _run_step(rule, 2048 + 5, [], "random", "float16", "scaler", False, True, _seed("0", rule))
    assert not upd.any()
    RAN.update(("shape", s) for s in shapes | {"nseg 0"})


def _adam_launch(nvec, segs, step_dev, found, seed):
    n = 4 * nvec
    p0, st0, g0, _ = _inputs(n, "adam", "random", None, seed)
    p, m, v, g = (torch.from_numpy(a.copy()).cuda() for a in (p0, st0[0], st0[1], g0))
    arr = _seg_array("adam", segs, True)
    rc = L().sod_adam(ptr(p), ptr(m), ptr(v), ptr(g), None, None, n, arr, len(segs), None, ptr(step_dev), 1.0, ptr(found),
                      _l().SOD_SGD_ZERO_GRAD, sp())
    assert rc == 0
    torch.cuda.synchronize()
    return (p0, st0, g0), (p, m, v, g)


def test_adam_step_counts_across_grids_and_a_skip():
    """counts 0, 1, 10⁴ and 10⁶ on one step_dev, advanced by launches of one CTA, a middle grid and the cap, with a
    skipped step in between: each launch uses the counts the last one left and re-arms the ticket"""
    sm = _sm()
    counts = [0, 1, 10_000, 1_000_000]
    step_dev = torch.zeros(17, dtype=torch.int32)
    step_dev[:4] = torch.tensor(counts, dtype=torch.int32)
    step_dev = step_dev.cuda()
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    for k, (cell, skip) in enumerate([("1cta", False), ("ctas ragged", False), ("ctas ragged", True), (">=2 passes exact", False)]):
        nvec = max(geo.select("step", cell, sm), 8)
        q = nvec // 4
        segs = [dict(begin=4 * i * q, end=4 * ((i + 1) * q if i < 3 else nvec), flags=0, wd=5e-4, lr=ADAM_LRS[i],
                     beta1=BETAS[i][0], beta2=BETAS[i][1], eps=1e-8) for i in range(4)]
        found.fill_(1 if skip else 0)
        (p0, st0, g0), (p, m, v, g) = _adam_launch(nvec, segs, step_dev, found, _seed("counts", k))
        wp, wst, _, _, _ = rp.step("adam", p0, st0, g0, None, segs, skip=skip, steps=counts)
        _assert_same(p.cpu().numpy(), wp, f"p after launch {k}")
        _assert_same(m.cpu().numpy(), wst[0], "m")
        _assert_same(v.cpu().numpy(), wst[1], "v")
        assert not g.any()
        counts = rp.next_steps(counts, segs, skip)
        assert step_dev.cpu().tolist() == counts + [0] * 13, k


# ---------------------------------------------------------------------------------------------------------------------
# the loss scaler
# ---------------------------------------------------------------------------------------------------------------------
def _scaler_step(scale, unskipped, gi, found, n=4 * 1031):
    l = _l()
    s = torch.zeros(l.SOD_LOSS_SCALER_WORDS, dtype=torch.int32)
    s[0], s[2], s[3] = found, unskipped, gi
    s.view(torch.float32)[1] = scale
    s = s.cuda()
    rng = np.random.default_rng(_seed("scaler", scale, gi, found))
    p0 = rng.standard_normal(n).astype(np.float32)
    g0 = (rng.standard_normal(n) * 1e3).astype(np.float32)
    p, v, g = torch.from_numpy(p0.copy()).cuda(), torch.zeros(n, device="cuda"), torch.from_numpy(g0.copy()).cuda()
    segs = [dict(begin=0, end=n, flags=0, lr=0.05, wd=0.0, mu=0.9)]
    assert L().sod_sgd_momentum_scaler(ptr(p), ptr(v), ptr(g), None, None, n, _seg_array("sgd", segs, True), 1, None, ptr(s),
                                       l.SOD_SGD_ZERO_GRAD, sp()) == 0
    torch.cuda.synchronize()
    wp, _, _, _, _ = rp.step("sgd", p0, [np.zeros(n, np.float32)], g0, None, segs, scale=scale, skip=bool(found))
    _assert_same(p.cpu().numpy(), wp, "p")
    w = s.cpu()
    assert int(w[0]) == found and int(w[4]) == 0
    return float(w.view(torch.float32)[1]), int(w[2])


def test_scaler_edges():
    f = lambda x: float(np.float32(x))                  # noqa: E731
    # a scale that is not a power of two: 1/scale rounds, and the step uses exactly that
    assert _scaler_step(3.0, 0, 2, 0) == (3.0, 1)
    assert _scaler_step(f(1 / 3), 1, 2, 0) == rp.scaler_next(f(1 / 3), 1, 2, False)
    assert _scaler_step(3.0, 5, 0, 0) == (3.0, 6)                    # growth_interval 0: never grows
    assert _scaler_step(3.0, 5, 1, 0) == (6.0, 6)                    # 1: every clean step
    assert _scaler_step(1.0, 4, 2, 1) == (1.0, 0) and _scaler_step(1.5, 4, 2, 1) == (1.0, 0)    # the floor
    assert _scaler_step(2.0 ** 23, 0, 1, 0) == (2.0 ** 24, 1)         # growth to the cap
    assert _scaler_step(2.0 ** 24, 0, 1, 0) == (2.0 ** 24, 1)         # and not past it
    s, u = 2.0 ** 40, 0                                               # a host-set scale beyond the cap halves down
    for k in range(3):
        s, u = _scaler_step(s, u, 1, 1)
        assert s == 2.0 ** (39 - k) and u == 0
    got = _scaler_step(2.0 ** 127, 0, 1, 0)                          # (unbounded doubling gave +inf here)
    assert got == (2.0 ** 24, 1) and np.isfinite(got[0])
    assert _scaler_step(got[0], got[1], 1, 0) == (2.0 ** 24, 2)       # and the next step is a normal one


# ---------------------------------------------------------------------------------------------------------------------
# gather
# ---------------------------------------------------------------------------------------------------------------------
class _Gather:
    """items over sources with chosen misalignment, packed into a sentinel-filled destination with 64-element padding"""

    def __init__(self, numels, misalign, dtype, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.dtype = getattr(torch, dtype)
        self.srcs, self.offs, self.numels = [], [], list(numels)
        off = 64
        for k, (x, mis) in enumerate(zip(numels, misalign)):
            base = (torch.randn(x + 8, generator=g, device="cuda") * 4).to(self.dtype)
            self.srcs.append(base[mis // 2: mis // 2 + x])
            self.offs.append(off)
            off += (x + 63) // 64 * 64 + 64
        self.total = off
        self.dst = torch.full((off,), SENT16, dtype=torch.int16, device="cuda").view(self.dtype)

    def items(self, bad=None):
        l = _l()
        arr = (l.sod_gather_item * len(self.srcs))()
        for k, (s, o, x) in enumerate(zip(self.srcs, self.offs, self.numels)):
            arr[k] = l.sod_gather_item(s.data_ptr(), o, x)
        if bad is not None:
            k, field, val = bad
            setattr(arr[k], field, val)
        return arr

    def run(self, checked=None, found=None, bad=None):
        arr = self.items(bad)
        if checked is None:
            return L().sod_grad_gather16(arr, len(self.srcs), ptr(self.dst), self.total, sp())
        return L().sod_grad_gather16_checked(arr, len(self.srcs), ptr(self.dst), self.total, checked, ptr(found), sp())

    def verify(self):
        torch.cuda.synchronize()
        d = _bits16(self.dst)
        pad = np.ones(self.total, bool)
        for s, o, x in zip(self.srcs, self.offs, self.numels):
            assert np.array_equal(d[o:o + x], _bits16(s)), (o, x)
            pad[o:o + x] = False
        assert np.all(d[pad] == SENT16)


def _gather_set(sm, dtype, seed):
    numels = list(range(1, 17)) + [8192, 8193, 8192 * 3 + 5]
    numels += [24 + k for k in range(7)]
    misalign = [0] * 19 + [2 * k for k in range(1, 8)]
    numels.append((geo.GATHER_CTAS_PER_SM * sm + 1) * geo.GATHER_CHUNK + 3)      # a second grid-stride pass
    misalign.append(0)
    numels += [9 + k % 17 for k in range(321 - len(numels))]                  # 321 items: three launches
    misalign += [(k % 8) * 2 for k in range(321 - len(misalign))]
    return numels, misalign


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_gather_copies_exactly(dtype):
    sm = _sm()
    numels, misalign = _gather_set(sm, dtype, 1)
    RAN.update(("gather", c) for c in geo.gather_cells(numels, misalign, sm))
    assert geo.gather_cells(numels, misalign, sm) == set(geo.GATHER_CELLS)
    for count in (160, 161, 321):
        gs = _Gather(numels[-count:] if count < 321 else numels, misalign[-count:] if count < 321 else misalign, dtype, count)
        assert gs.run() == 0
        gs.verify()
        found = torch.zeros(1, dtype=torch.int32, device="cuda")
        gs.dst.view(torch.int16).fill_(SENT16)
        assert gs.run(checked=_l().SOD_BF16 if dtype == "bfloat16" else _l().SOD_F16, found=found) == 0
        gs.verify()
        assert int(found.item()) == 0


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_gather_checked_flags_each_position_class(dtype):
    sm = _sm()
    l = _l()
    code = l.SOD_BF16 if dtype == "bfloat16" else l.SOD_F16
    numels, misalign = _gather_set(sm, dtype, 2)
    big = numels.index((geo.GATHER_CTAS_PER_SM * sm + 1) * geo.GATHER_CHUNK + 3)
    # (item, element): aligned body, aligned tail, misaligned item, second grid-stride pass, second launch
    where = {"body": (17, 5), "tail": (17, 8192), "misaligned": (20, 3), "second pass": (big, numels[big] - 10),
             "second launch": (300, 4)}
    assert misalign[20] % 16 and misalign[17] == 0 and numels[17] == 8193
    ok_max = 0x7F7F if dtype == "bfloat16" else 0x7BFF
    specials = [0x7F80, 0xFFC1] if dtype == "bfloat16" else [0x7C00, 0xFE01]
    gs = _Gather(numels, misalign, dtype, 7)
    for cls, (k, e) in where.items():
        for bits in specials:
            w = gs.srcs[k].view(torch.int16)
            keep = w[e].clone()
            w[e] = bits - (1 << 16 if bits >= 1 << 15 else 0)
            found = torch.zeros(1, dtype=torch.int32, device="cuda")
            assert gs.run(checked=code, found=found) == 0
            gs.verify()
            assert int(found.item()) == 1, (cls, hex(bits))
            w[e] = keep
            RAN.add(("gather flag", cls))
    # finite extremes are not flagged: the largest finite value, and 0x7C00, finite in bf16 (inf in fp16)
    gs = _Gather(numels, misalign, dtype, 8)
    for k, e in where.values():
        gs.srcs[k].view(torch.int16)[e] = ok_max
        if dtype == "bfloat16":
            gs.srcs[k].view(torch.int16)[e - 1] = 0x7C00
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert gs.run(checked=code, found=found) == 0
    gs.verify()
    assert int(found.item()) == 0
    found.fill_(1)                                            # a preset verdict stays set
    assert gs.run(checked=code, found=found) == 0
    torch.cuda.synchronize()
    assert int(found.item()) == 1


# ---------------------------------------------------------------------------------------------------------------------
# check ranges, nonfinite, merge
# ---------------------------------------------------------------------------------------------------------------------
def _ranges_setup(sm, seed):
    """259 ranges over fp32 and 16-bit buffers: unaligned begins and empty ranges in the first batch, a second batch of
    empty ranges only, then a range of more chunks than the grid; every element between ranges is NaN (bf16 and fp16
    NaN in the 16-bit buffer) and must never be read"""
    lengths, in16 = [], []
    for k in range(128):
        lengths.append([0, 1, 3, 4095, 4096, 4097, 17][k % 7])
        in16.append(k % 2 == 1)
    lengths += [0] * 128
    in16 += [False] * 128
    lengths += [4095, (geo.CHECK_CTAS_PER_SM * sm + 1) * geo.CHECK_CHUNK + 5, 9]
    in16 += [True, False, True]
    begins, off = [], 3
    for x in lengths:
        begins.append(off)
        off += x + 5
    n = off + 8
    g = torch.full((n,), float("nan"), device="cuda")
    h = torch.full((n,), 0x7FC1, dtype=torch.int16, device="cuda")
    for b, x, s in zip(begins, lengths, in16):
        if s:
            h[b:b + x] = 0x3C00
        else:
            g[b:b + x] = 1.5
    return lengths, in16, begins, n, g, h


def _check_call(g, h, n, lengths, in16, begins, f16, found):
    l = _l()
    arr = (l.sod_check_range * len(lengths))()
    for k, (b, x, s) in enumerate(zip(begins, lengths, in16)):
        arr[k] = l.sod_check_range(b, b + x, l.SOD_SEG_GRAD16 if s else 0)
    return L().sod_grad_check_ranges(ptr(g), ptr(h), n, arr, len(lengths), l.SOD_GRAD16_F16 if f16 else 0, ptr(found), sp())


@pytest.mark.parametrize("f16", [False, True])
def test_check_ranges_regimes(f16):
    sm = _sm()
    lengths, in16, begins, n, g, h = _ranges_setup(sm, 0)
    cells = geo.check_cells(lengths, sm)
    assert cells == set(geo.CHECK_CELLS)
    RAN.update(("check", c) for c in cells)
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert _check_call(g, h, n, lengths, in16, begins, f16, found) == 0
    torch.cuda.synchronize()
    assert int(found.item()) == 0                      # nothing outside a range was read
    big = len(lengths) - 2
    where = {"first range": (1, 0), "unaligned 16-bit": (3, 2), "chunk tail": (5, 4096), "second launch": (256, 0),
             "second pass": (big, lengths[big] - 1), "last": (len(lengths) - 1, 8)}
    for cls, (k, e) in where.items():
        assert lengths[k] > e
        for bad in ("inf", "nan"):
            gg, hh = g.clone(), h.clone()
            if in16[k]:
                hh[begins[k] + e] = (0x7C00 if f16 else 0x7F80) if bad == "inf" else (0x7E00 if f16 else 0x7FC0)
            else:
                gg[begins[k] + e] = float(bad)
            found.zero_()
            assert _check_call(gg, hh, n, lengths, in16, begins, f16, found) == 0
            torch.cuda.synchronize()
            assert int(found.item()) == 1, (cls, bad)
        RAN.add(("check flag", cls))


@pytest.mark.parametrize("cell", geo.FLAT_CELLS)
def test_nonfinite_regimes(cell):
    sm = _sm()
    nvec = geo.select("nonfinite", cell, sm)
    n = 4 * nvec
    base = torch.full((n,), 1.0, device="cuda")
    base[0], base[n // 2], base[-1] = -0.0, 1e-45, float(np.finfo(np.float32).max)
    base[1 % n] = -float(np.finfo(np.float32).max)
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert L().sod_grad_nonfinite(ptr(base), n, ptr(found), sp()) == 0
    torch.cuda.synchronize()
    assert int(found.item()) == 0
    stride = geo.flat_grid("nonfinite", nvec, sm) * geo.FLAT_THREADS
    for vec in sorted({0, stride - 1 if stride <= nvec else nvec - 1, nvec - 1, min(stride, nvec - 1)}):
        for lane in (0, 3):
            for bad in (float("inf"), float("-inf"), float("nan")):
                g = base.clone()
                g[4 * vec + lane] = bad
                found.zero_()
                assert L().sod_grad_nonfinite(ptr(g), n, ptr(found), sp()) == 0
                torch.cuda.synchronize()
                assert int(found.item()) == 1, (vec, lane, bad)
    RAN.add(("nonfinite", cell))


@pytest.mark.parametrize("cell", geo.FLAT_CELLS)
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_merge16_regimes(cell, dtype):
    sm = _sm()
    l = _l()
    nvec = geo.select("merge", cell, sm)
    n = 4 * nvec
    rng = np.random.default_rng(_seed("merge", cell, dtype))
    g0 = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    h0 = _f16((rng.standard_normal(n) * np.exp2(rng.integers(-10, 10, n))).astype(np.float32), dtype)
    hb = h0.view(torch.int16).numpy().reshape(nvec, 4)
    # per float4: all zero, a zero low uint32 half, a zero high half, a lone −0, random
    kinds = rng.integers(0, 5, nvec)
    hb[kinds == 0] = 0
    hb[kinds == 1, :2] = 0
    hb[kinds == 2, 2:] = 0
    hb[kinds == 3] = 0
    hb[kinds == 3, 1] = -32768
    g0[4 * np.flatnonzero(kinds == 0)] = np.nan                # h = 0 there: g is left alone, NaN included
    hv = h0.float().numpy()
    want = np.where(np.repeat(_bits16(h0).reshape(-1, 4).any(axis=1), 4), g0 + hv, g0).astype(np.float32)
    g, h = torch.from_numpy(g0.copy()).cuda(), h0.cuda()
    if dtype == "bfloat16":
        assert L().sod_grad_merge_bf16(ptr(g), ptr(h), n, sp()) == 0
    else:
        assert L().sod_grad_merge16(ptr(g), ptr(h), n, l.SOD_GRAD16_F16, sp()) == 0
    torch.cuda.synchronize()
    _assert_same(g.cpu().numpy(), want, "merged gradient")
    assert not _bits16(h).any()
    RAN.add(("merge", cell))


# ---------------------------------------------------------------------------------------------------------------------
# refusals: nothing written, nothing advanced
# ---------------------------------------------------------------------------------------------------------------------
class _Snap:
    def __init__(self, *ts):
        self.ts = [t for t in ts if t is not None]
        self.before = [t.clone() for t in self.ts]

    def unchanged(self):
        torch.cuda.synchronize()
        return all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(self.ts, self.before))


def test_step_entries_refuse_before_any_launch():
    l = _l()
    n = 4 * 700
    p, v, m, g = (torch.randn(n + 4, device="cuda")[:n] for _ in range(4))
    h = torch.randn(n, device="cuda").to(torch.bfloat16)
    sh = torch.full((n,), SENT16, dtype=torch.int16, device="cuda")
    steps = torch.tensor([3, 4] + [0] * 15, dtype=torch.int32, device="cuda")
    sc = torch.zeros(l.SOD_LOSS_SCALER_WORDS, dtype=torch.int32)
    sc.view(torch.float32)[1] = 1024.0
    sc[3] = 1
    sc = sc.cuda()
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    odd = torch.zeros(n + 8, device="cuda")[1:n + 1]                 # 4 bytes off 16
    good_sgd = [dict(begin=0, end=n // 2, lr=0.1, wd=0.0, mu=0.9, flags=0), dict(begin=n // 2, end=n, lr=0.1, wd=0.0, mu=0.9, flags=0)]
    good_adam = [dict(begin=0, end=n // 2, lr=1e-3, wd=0.0, beta1=0.9, beta2=0.999, eps=1e-8, flags=0),
                 dict(begin=n // 2, end=n, lr=1e-3, wd=0.0, beta1=0.9, beta2=0.999, eps=1e-8, flags=0)]
    bad_tables = {
        "unsorted": lambda t: [t[1], t[0]], "end > n": lambda t: [t[0], dict(t[1], end=n + 4)],
        "begin < 0": lambda t: [dict(t[0], begin=-4), t[1]], "end < begin": lambda t: [dict(t[0], end=0, begin=8), t[1]],
        "unaligned": lambda t: [dict(t[0], end=n // 2 - 2), dict(t[1], begin=n // 2 - 2)],
    }
    snap = _Snap(p, v, m, g, h, sh, steps, sc, found)

    def call(entry, rule_segs, nseg=None, **over):
        a = dict(p=ptr(p), v=ptr(v), m=ptr(m), g=ptr(g), h=ptr(h), sh=ptr(sh), n=n, steps=ptr(steps), sc=ptr(sc),
                 found=ptr(found))
        a.update(over)
        rule = "adam" if "adam" in entry else "sgd"
        arr = _seg_array(rule, rule_segs, True) if rule_segs is not None else None
        ns = len(rule_segs or []) if nseg is None else nseg
        arrp = C.cast(arr, C.POINTER(l.sod_adam_segment if rule == "adam" else l.sod_sgd_segment)) if arr is not None else None
        if entry == "sod_sgd_momentum":
            return L().sod_sgd_momentum(a["p"], a["v"], a["g"], a["h"], a["sh"], a["n"], arrp, ns, None, 1.0, a["found"], 1, sp())
        if entry == "sod_sgd_momentum_scaler":
            return L().sod_sgd_momentum_scaler(a["p"], a["v"], a["g"], a["h"], a["sh"], a["n"], arrp, ns, None, a["sc"], 1, sp())
        if entry == "sod_adam":
            return L().sod_adam(a["p"], a["m"], a["v"], a["g"], a["h"], a["sh"], a["n"], arrp, ns, None, a["steps"], 1.0,
                                a["found"], 1, sp())
        return L().sod_adam_scaler(a["p"], a["m"], a["v"], a["g"], a["h"], a["sh"], a["n"], arrp, ns, None, a["steps"], a["sc"],
                                   1, sp())

    for entry in ("sod_sgd_momentum", "sod_sgd_momentum_scaler", "sod_adam", "sod_adam_scaler"):
        good = good_adam if "adam" in entry else good_sgd
        cases = [(-1, dict(p=None)), (-1, dict(g=None)), (-1, dict(v=None)), (-1, dict(n=0)), (-1, dict(n=-4)),
                 (-2, dict(n=n - 2)), (-2, dict(p=ptr(odd))), (-2, dict(g=ptr(odd))), (-2, dict(v=ptr(odd))),
                 (-2, dict(h=ptr(h) + 2)), (-2, dict(sh=ptr(sh) + 2))]
        if "adam" in entry:
            cases += [(-1, dict(m=None)), (-1, dict(steps=None)), (-2, dict(m=ptr(odd)))]
        if "scaler" in entry:
            cases.append((-1, dict(sc=None)))
        for want, over in cases:
            assert call(entry, good, **over) == want, (entry, over)
        for name, f in bad_tables.items():
            assert call(entry, f(good)) == (-2 if name == "unaligned" else -1), (entry, name)
        assert call(entry, good, nseg=-1) == -1 and call(entry, good, nseg=17) == -1 and call(entry, None, nseg=2) == -1
        if "adam" in entry:
            for bad in (dict(beta1=1.0), dict(beta2=-0.1), dict(eps=-1e-8), dict(beta1=float("nan")), dict(flags=l.SOD_SEG_NESTEROV)):
                assert call(entry, [good[0], dict(good[1], **bad)]) == -1, (entry, bad)
        assert snap.unchanged(), entry


def test_gradient_entries_refuse_before_any_launch():
    """every refusal of the six gradient entries leaves every output, found_inf included, byte-identical — also when
    item 161 or range 129 is the invalid one (the first batch used to be launched before it was seen)"""
    l = _l()
    gs = _Gather([37] * 170, [0] * 170, "bfloat16", 3)
    found = torch.zeros(1, dtype=torch.int32, device="cuda")
    snap = _Snap(gs.dst, found)
    t = gs.total
    gcases = [dict(bad=(160, "src", None)), dict(bad=(160, "numel", 0)), dict(bad=(160, "dst_offset", -8)),
              dict(bad=(160, "dst_offset", gs.offs[160] + 4)), dict(bad=(160, "dst_offset", t - 8)),
              dict(bad=(0, "numel", -1)), dict(bad=(169, "src", None))]
    for c in gcases:
        for checked in (None, l.SOD_BF16, l.SOD_F16):
            rc = gs.run(checked=checked, found=found, **c)
            assert rc == (-2 if c["bad"][2] == gs.offs[160] + 4 else -1), (c, checked)
    arr = gs.items()
    assert L().sod_grad_gather16(arr, -1, ptr(gs.dst), t, sp()) == -1
    assert L().sod_grad_gather16(None, 3, ptr(gs.dst), t, sp()) == -1
    assert L().sod_grad_gather16(arr, 3, None, t, sp()) == -1
    assert L().sod_grad_gather16(arr, 3, ptr(gs.dst), 0, sp()) == -1
    assert L().sod_grad_gather16(arr, 3, ptr(gs.dst) + 2, t - 8, sp()) == -2
    assert L().sod_grad_gather16_checked(arr, 3, ptr(gs.dst), t, l.SOD_F32, ptr(found), sp()) == -1
    assert L().sod_grad_gather16_checked(arr, 3, ptr(gs.dst), t, l.SOD_BF16, None, sp()) == -1
    assert snap.unchanged()
    # range check: range 129 invalid after 128 ranges whose values would set found_inf
    n = 4 * 600
    g = torch.full((n,), float("inf"), device="cuda")
    h = torch.full((n,), 0x7C00, dtype=torch.int16, device="cuda")
    snap = _Snap(g, h, found)

    def ranges(bad):
        arr = (l.sod_check_range * 140)()
        for k in range(140):
            arr[k] = l.sod_check_range(k, k + 3, l.SOD_SEG_GRAD16 if k % 2 else 0)
        arr[128] = l.sod_check_range(*bad)
        return arr
    for bad, gp, hp in [((5, n + 1, 0), g, h), ((-1, 4, 0), g, h), ((9, 8, 0), g, h), ((4, 8, 0), None, h),
                        ((4, 8, l.SOD_SEG_GRAD16), g, None)]:
        rc = L().sod_grad_check_ranges(ptr(gp), ptr(hp), n, ranges(bad), 140, 0, ptr(found), sp())
        assert rc == -1, bad
    arr = ranges((4, 8, 0))
    assert L().sod_grad_check_ranges(ptr(g), ptr(h), n, arr, 140, 0, None, sp()) == -1
    assert L().sod_grad_check_ranges(ptr(g), ptr(h), 0, arr, 140, 0, ptr(found), sp()) == -1
    assert L().sod_grad_check_ranges(ptr(g), ptr(h), n, arr, -1, 0, ptr(found), sp()) == -1
    assert L().sod_grad_check_ranges(ptr(g), ptr(h), n, None, 3, 0, ptr(found), sp()) == -1
    # nonfinite and the merges
    odd = torch.zeros(n + 8, device="cuda")[1:n + 1]
    assert L().sod_grad_nonfinite(None, n, ptr(found), sp()) == -1
    assert L().sod_grad_nonfinite(ptr(g), n, None, sp()) == -1
    assert L().sod_grad_nonfinite(ptr(g), 0, ptr(found), sp()) == -1
    assert L().sod_grad_nonfinite(ptr(g), n - 1, ptr(found), sp()) == -2
    assert L().sod_grad_nonfinite(ptr(odd), n, ptr(found), sp()) == -2
    for merge in (lambda a, b, k: L().sod_grad_merge_bf16(a, b, k, sp()),
                  lambda a, b, k: L().sod_grad_merge16(a, b, k, l.SOD_GRAD16_F16, sp())):
        assert merge(None, ptr(h), n) == -1 and merge(ptr(g), None, n) == -1 and merge(ptr(g), ptr(h), 0) == -1
        assert merge(ptr(g), ptr(h), n - 2) == -2 and merge(ptr(odd), ptr(h), n) == -2 and merge(ptr(g), ptr(h) + 2, n) == -2
    assert snap.unchanged()


# ---------------------------------------------------------------------------------------------------------------------
def test_every_cell_ran():
    need = {("step", c) for c in geo.STEP_CELLS} | {("edge", e) for e in geo.EDGE_CLASSES}
    need |= {("shape", s) for s in ("float4", "empty", "gap", "frozen", "ends at n", "16 segments", "nseg 0")}
    need |= {("step", r, g, m) for r in RULES for g in G16 for m in MODES}
    need |= {("combo", r, a, b) for r in RULES for a in (False, True) for b in (False, True)}
    need |= {("tier", t) for t in ("random", "special", "ties")}
    need |= {("gather", c) for c in geo.GATHER_CELLS} | {("check", c) for c in geo.CHECK_CELLS}
    need |= {("gather flag", c) for c in ("body", "tail", "misaligned", "second pass", "second launch")}
    need |= {("check flag", c) for c in ("first range", "unaligned 16-bit", "chunk tail", "second launch", "second pass", "last")}
    need |= {("nonfinite", c) for c in geo.FLAT_CELLS} | {("merge", c) for c in geo.FLAT_CELLS}
    missing = sorted(need - RAN, key=repr)
    assert not missing, missing
