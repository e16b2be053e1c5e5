"""The resampling kernels of csrc/resample.cu, csrc/maxpool.cu and csrc/nearest.cu in every launch regime of this GPU,
element by element against float64 (oracle/resample.py), the nearest ×2 kernels bit for bit (the forward against torch,
the backward against the fixed-order restatement of tests/_nearest.py), and `sod_colsum` bit for bit against an fp32
replay of its summation order.

Which threads make a second pass, which stay idle and which run the colsum tail is decided at launch time from the SM
count.  oracle/resample_geometry.py picks, for the device the test runs on, the smallest shape that puts each of the
eight grid-stride kernels (bilinear ×2, 2×2 average pool, 3×3/2 max pool, nearest ×2; forward and backward) in each wave
regime (a partial wave below the 16·#SMs cap, one full pass, a full pass plus a ragged one, two or more passes ragged
and exact), and the row counts that give `sod_colsum` every L = C/8 from 1 to 256, a grid below and at its cap, every
tail residue q mod 4, idle threads and a single row.  The shapes res50 passes to each kernel at 256², 320² and 384²
(bs 16), and the twelve nearest up-sample shapes of aim_res50 at 320² and 352² (bs 16; at 320² the 64-channel 80² maps
are 819 200 packets, more than one pass of a 132-SM H100's 540 672 threads), are recorded by wrapping the library calls
of one training iteration, and are run too.  Each kernel runs on its own: the backward
kernels get their dy (and the max-pool's window positions) from the test, not from the forward kernel.

Inputs come in three tiers.
* Exact: integers in [−64, 64] ([−8, 8] for colsum beyond 2¹⁸ rows).  All weights are multiples of 1/16, so every fp32
  intermediate is exact and each output must equal the float64 result rounded once to its dtype, whatever its size:
  any wrong index, weight, tap or tail shows.
* Random N(0, 1).  Up-sample: one ulp of the output dtype plus 2⁻²⁰ of the same weighted sum over |values| (the
  fp32 rounding of the 4-term forward, ≤ 16-term backward).  Average pool: one ulp plus 2⁻²² of the mean of |x| in every
  dtype (four 2-byte values whose exponents lie far apart do not sum exactly in fp32, and the fp32 sum then rounds a
  second time to the dtype: measured on an H100, 1 of 4.3 M random fp16 means is half an ulp off the correctly rounded
  one); the backward dy/4 is exact.  Max pool:
  the forward and its window positions equal the oracle's; the backward is within one ulp plus 2⁻²²·Σ|dy|.  fp32
  arithmetic on fp32 subnormals rounds to 2⁻¹⁴⁹, so fp32 adds that absolute error per operation.  Colsum equals the
  replay bit for bit (rounded once for 2-byte dtypes).
* Special values: ±inf and NaN at the first and last row, column and channel, and on window tie positions; the dtype's
  largest finite value M, where the up-sample's fused add must overflow exactly where the float64 sum rounds past M;
  subnormals, which must not be flushed.  Where the oracle's result in the dtype is not finite the kernel must give
  the same (NaN where NaN, the same infinity); elsewhere the random-tier bound holds.  The average pool sums its four
  inputs in fp32 before the quarter, as torch's kernel does, so its windows keep that sum finite (M only in fp16, where
  4M fits fp32).  The nearest kernels are compared by bits in every tier, NaN by class (its payload is the device's).

Refusals: null pointers, 2-byte misalignment, n/h/w ≤ 0, C % 8, colsum C = 24 and 4096, a short workspace and an
unknown dtype code each return their code and leave a sentinel-filled output untouched.
"""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from _nearest import upsample2x_nearest_bwd

from oracle import resample as ors
from oracle import resample_geometry as geo

pytestmark = pytest.mark.gpu

TORCH_DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}
MANT = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}
EMIN = {torch.float32: -126, torch.bfloat16: -126, torch.float16: -14}
SOD_EINVAL, SOD_EALIGN, SOD_EWORKSPACE, SOD_EUNSUPPORTED = -1, -2, -3, -4
TIERS = ("exact", "random", "special")
RAN: dict = {}              # case id → regime cells it reached on this device


def _sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def ulp(ref, dtype):
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** EMIN[dtype])))
    return torch.exp2(e - MANT[dtype])


def _sub(dtype):
    """the smallest subnormal of dtype"""
    return 2.0 ** (EMIN[dtype] - MANT[dtype])


# ---- direct calls of the C ABI ---------------------------------------------------------------------------------------
def _lib():
    from distributed_sod_project_b200 import _lib
    return _lib


def _cl(shape, dtype):
    return torch.empty(shape, dtype=dtype, device="cuda", memory_format=torch.channels_last)


def _run(name, *args):
    L = _lib()
    rc = getattr(L.lib(), name)(*args)
    L.check(rc, name)
    torch.cuda.synchronize()


def up_fwd(x, add=None):
    n, c, h, w = x.shape
    y = _cl((n, c, 2 * h, 2 * w), x.dtype)
    _run("sod_upsample2x_bilinear_fwd", x.data_ptr(), None if add is None else add.data_ptr(), y.data_ptr(), n, h, w, c,
         _lib().dtype_code(x.dtype), _lib().stream_ptr())
    return y


def up_bwd(dy):
    n, c, h2, w2 = dy.shape
    dx = _cl((n, c, h2 // 2, w2 // 2), dy.dtype)
    _run("sod_upsample2x_bilinear_bwd", dy.data_ptr(), dx.data_ptr(), n, h2 // 2, w2 // 2, c, _lib().dtype_code(dy.dtype),
         _lib().stream_ptr())
    return dx


def avg_fwd(x):
    n, c, h, w = x.shape
    y = _cl((n, c, h // 2, w // 2), x.dtype)
    _run("sod_avgpool2x2_fwd", x.data_ptr(), y.data_ptr(), n, h // 2, w // 2, c, _lib().dtype_code(x.dtype), _lib().stream_ptr())
    return y


def avg_bwd(dy):
    n, c, ho, wo = dy.shape
    dx = _cl((n, c, 2 * ho, 2 * wo), dy.dtype)
    _run("sod_avgpool2x2_bwd", dy.data_ptr(), dx.data_ptr(), n, ho, wo, c, _lib().dtype_code(dy.dtype), _lib().stream_ptr())
    return dx


def max_fwd(x):
    n, c, h, w = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    y = _cl((n, c, ho, wo), x.dtype)
    arg = torch.empty((n, ho, wo, c), dtype=torch.uint8, device="cuda")
    _run("sod_maxpool3x3s2_fwd", x.data_ptr(), y.data_ptr(), arg.data_ptr(), n, h, w, c, _lib().dtype_code(x.dtype),
         _lib().stream_ptr())
    return y, arg


def max_bwd(dy, arg, h, w):
    n, c = dy.shape[:2]
    dx = _cl((n, c, h, w), dy.dtype)
    _run("sod_maxpool3x3s2_bwd", dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), n, h, w, c, _lib().dtype_code(dy.dtype),
         _lib().stream_ptr())
    return dx


def near_fwd(x):
    n, c, h, w = x.shape
    y = _cl((n, c, 2 * h, 2 * w), x.dtype)
    _run("sod_upsample2x_nearest_fwd", x.data_ptr(), y.data_ptr(), n, h, w, c, _lib().dtype_code(x.dtype), _lib().stream_ptr())
    return y


def near_bwd(dy):
    n, c, h2, w2 = dy.shape
    dx = _cl((n, c, h2 // 2, w2 // 2), dy.dtype)
    _run("sod_upsample2x_nearest_bwd", dy.data_ptr(), dx.data_ptr(), n, h2 // 2, w2 // 2, c, _lib().dtype_code(dy.dtype),
         _lib().stream_ptr())
    return dx


_WS = {}


def _workspace():
    if "ws" not in _WS:
        _WS["ws"] = torch.zeros(int(_lib().lib().sod_colsum_workspace_bytes()), dtype=torch.uint8, device="cuda")
    return _WS["ws"]


def colsum(x2d):
    rows, c = x2d.shape
    out = torch.empty(c, dtype=x2d.dtype, device="cuda")
    ws = _workspace()
    _run("sod_colsum", x2d.data_ptr(), out.data_ptr(), rows, c, _lib().dtype_code(x2d.dtype), ws.data_ptr(), ws.numel(),
         _lib().stream_ptr())
    return out


# ---- inputs ------------------------------------------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def make(shape, dtype, tier, seed, role="x"):
    """a channels-last tensor of `tier`; `role` picks where the special tier puts its values ("x": the op's input,
    "add": the up-sample's fused addend, "dy": a gradient)"""
    g = _gen(seed)
    n, c, h, w = shape
    if tier == "exact":
        hi = 8 if n * h * w > 1 << 18 else 64
        t = torch.randint(-hi, hi + 1, shape, generator=g, device="cuda").float()
    else:
        t = torch.randn(shape, generator=g, device="cuda")
    if tier == "special":
        inf, nan = float("inf"), float("nan")
        big = torch.finfo(dtype).max
        t[0, 0, 0, 0] = inf                                  # first row, column, channel
        t[n - 1, c - 1, h - 1, w - 1] = -inf                 # last row, column, channel
        t[0, c - 1, 0, w - 1] = nan
        t[n - 1, 0, h - 1, 0] = inf
        t[0, 1, h // 2, w // 2] = -inf
        if h > 2 and w > 2:
            t[n - 1, 1, 1, 1] = nan                          # a position inside up to four 3×3 windows
        # channel 2: M, which overflows in the up-sample's fused add (M + M) and in the backward's weight sum (4M);
        # channel 3: the largest power of two P ≤ M, cancelled by the addend (P − P); channel 4: P + (M − P) = M exactly,
        # the largest finite sum (M/8 as a gradient: 4·M/8 stays finite)
        p2 = 2.0 ** math.floor(math.log2(big))
        t[:, 2] = big
        t[:, 3] = p2 if role != "add" else -p2
        t[:, 4] = {"x": p2, "add": big - p2, "dy": big / 8}[role]
        # channel 5: subnormals (integer multiples of the smallest one)
        t[:, 5] = torch.randint(-64, 65, (n, h, w), generator=g, device="cuda").float() * _sub(dtype)
        # channel 6: ties in every window, with −inf filling one sample
        t[:, 6] = torch.randint(-2, 3, (n, h, w), generator=g, device="cuda").float()
        t[n - 1, 6] = -inf
    return t.to(dtype).contiguous(memory_format=torch.channels_last)


def _avg_safe(x):
    """average-pool input of the special tier with every window's fp32 sum finite: M only in fp16, otherwise M in one of
    the four inputs of a window and small values beside it"""
    if x.dtype == torch.float16:
        return x
    x = x.clone()
    big = torch.finfo(x.dtype).max
    for ch in (2, 3, 4):
        x[:, ch] = torch.where(x[:, ch].float().abs() >= big / 2, torch.zeros((), device="cuda", dtype=x.dtype), x[:, ch])
        x[:, ch, 0::2, 0::2] = big if ch != 4 else -big
    return x.contiguous(memory_format=torch.channels_last)


# ---- comparison --------------------------------------------------------------------------------------------------------
def assert_matches(got, ref, tol, dtype, what):
    """non-finite where ref rounded to dtype is (NaN where NaN, the same infinity), within tol of ref elsewhere;
    tol=None: equal to ref rounded to dtype"""
    got = got.double()
    want = ref.to(dtype).double()
    fin = want.isfinite()
    nf = ~fin
    same = (got[nf] == want[nf]) | (got[nf].isnan() & want[nf].isnan())
    assert bool(same.all()), (f"{what}: {int((~same).sum())} non-finite results differ, first got "
                              f"{float(got[nf][~same][0])} want {float(want[nf][~same][0])}")
    if tol is None:
        bad = fin & (got != want)
    else:
        bad = fin & ~((got - ref).abs() <= tol)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements off, first at {i}: got {float(got[tuple(i)])!r}, "
                             f"float64 {float(ref[tuple(i)])!r}" + ("" if tol is None else f", bound {float(tol[tuple(i)]):.3g}"))


def assert_same_bits(got, want, what):
    """bit for bit, NaN by class (a NaN's payload is the device's)"""
    bits = {4: torch.int32, 2: torch.int16}[got.element_size()]
    g, w = got.contiguous(), want.contiguous()
    nan = w.isnan()
    assert torch.equal(g.isnan(), nan), f"{what}: NaN at other positions ({int((g.isnan() != nan).sum())})"
    bad = (g.view(bits) != w.view(bits)) & ~nan
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ, first at {i}: got "
                             f"{float(g[tuple(i)])!r}, want {float(w[tuple(i)])!r}")


def _fp32_floor(dtype, ops):
    """the absolute rounding of `ops` fp32 operations on subnormal fp32 values"""
    return ops * 2.0 ** -149 if dtype == torch.float32 else 0.0


def check_kernel(kernel, shape, dtype, tier, seed):
    n, c, h, w = shape
    exact = tier == "exact"
    if kernel == "upsample_fwd":
        x = make(shape, dtype, tier, seed)
        add = None if exact and seed % 2 else make((n, c, 2 * h, 2 * w), dtype, tier, seed + 1, "add")
        y = up_fwd(x, add)
        ref = ors.upsample2x(x.double(), None if add is None else add.double())
        tol = None
        if not exact:
            mag = ors.upsample2x(x.double().abs(), None if add is None else add.double().abs())
            tol = ulp(ref, dtype) + 2.0 ** -20 * mag.nan_to_num(posinf=0.0) + _fp32_floor(dtype, 8)
        assert_matches(y, ref, tol, dtype, f"{kernel} {tier}")
    elif kernel == "upsample_bwd":
        dy = make((n, c, 2 * h, 2 * w), dtype, tier, seed, "dy")
        dx = up_bwd(dy)
        ref = ors.upsample2x_bwd(dy.double())
        tol = None if exact else (ulp(ref, dtype) + 2.0 ** -20 * ors.upsample2x_bwd(dy.double().abs()).nan_to_num(posinf=0.0)
                                  + _fp32_floor(dtype, 32))
        assert_matches(dx, ref, tol, dtype, f"{kernel} {tier}")
    elif kernel == "avgpool_fwd":
        x = make(shape, dtype, tier, seed)
        if tier == "special":
            x = _avg_safe(x)
        y = avg_fwd(x)
        ref = ors.avgpool2x2(x.double())
        tol = None
        if not exact:
            tol = ulp(ref, dtype) + 2.0 ** -22 * ors.avgpool2x2(x.double().abs()).nan_to_num(posinf=0.0) + _fp32_floor(dtype, 4)
        assert_matches(y, ref, tol, dtype, f"{kernel} {tier}")
    elif kernel == "avgpool_bwd":
        dy = make((n, c, h // 2, w // 2), dtype, tier, seed, "dy")
        dx = avg_bwd(dy)
        assert_matches(dx, ors.avgpool2x2_bwd(dy.double()), None, dtype, f"{kernel} {tier}")
    elif kernel == "maxpool_fwd":
        x = make(shape, dtype, tier, seed)
        y, arg = max_fwd(x)
        ref, aref = ors.maxpool_fwd(x.double().permute(0, 2, 3, 1))
        assert_matches(y, ref.permute(0, 3, 1, 2), None, dtype, f"{kernel} {tier}")
        bad = arg.long() != aref
        assert not bool(bad.any()), f"{kernel} {tier}: {int(bad.sum())} window positions differ from the oracle's"
    elif kernel == "maxpool_bwd":
        x = make(shape, dtype, tier, seed)
        _, aref = ors.maxpool_fwd(x.double().permute(0, 2, 3, 1))
        ho, wo = aref.shape[1:3]
        dy = make((n, c, ho, wo), dtype, tier, seed + 1, "dy")
        dx = max_bwd(dy, aref.to(torch.uint8).contiguous(), h, w)
        d64 = dy.double().permute(0, 2, 3, 1)
        ref = ors.maxpool_bwd(d64, aref, h, w).permute(0, 3, 1, 2)
        tol = None if exact else (ulp(ref, dtype) + 2.0 ** -22 * ors.maxpool_bwd(d64.abs(), aref, h, w).permute(0, 3, 1, 2)
                                  .nan_to_num(posinf=0.0) + _fp32_floor(dtype, 4))
        assert_matches(dx, ref, tol, dtype, f"{kernel} {tier}")
    elif kernel == "nearest_fwd":
        x = make(shape, dtype, tier, seed)
        assert_same_bits(near_fwd(x), F.interpolate(x, scale_factor=2, mode="nearest"), f"{kernel} {tier}")
    elif kernel == "nearest_bwd":
        dy = make((n, c, 2 * h, 2 * w), dtype, tier, seed, "dy")
        assert_same_bits(near_bwd(dy), upsample2x_nearest_bwd(dy), f"{kernel} {tier}")
    else:
        raise KeyError(kernel)


# ---- the eight grid-stride kernels in every wave regime ----------------------------------------------------------------
WAVE_CASES = [(k, d, wv) for k in geo.GRID_STRIDE_KERNELS for d in geo.DTYPES for wv in geo.WAVES]


@pytest.mark.parametrize("kernel, dtype, wave", WAVE_CASES, ids=[f"{k}-{d}-{w}" for k, d, w in WAVE_CASES])
def test_wave_regime(kernel, dtype, wave):
    sm = _sm()
    shape = geo.select(kernel, wave, sm)
    dt = TORCH_DT[dtype]
    for j, tier in enumerate(TIERS):
        check_kernel(kernel, shape, dt, tier, seed=zlib.crc32(f"{kernel}-{dtype}-{wave}-{j}".encode()))
    RAN[f"{kernel}-{dtype}-{wave}"] = {(kernel, dtype, geo.classify(geo.packets(kernel, shape), sm))}


# ---- small and degenerate shapes (one CTA; H or W equal to 1) -----------------------------------------------------------
SMALL = [(1, 8, 1, 1), (3, 8, 1, 5), (2, 16, 7, 1), (2, 32, 5, 7), (1, 128, 2, 9), (2, 8, 3, 3)]


@pytest.mark.parametrize("dtype", geo.DTYPES)
@pytest.mark.parametrize("kernel", geo.GRID_STRIDE_KERNELS)
def test_small_and_degenerate_shapes(kernel, dtype):
    for i, (n, c, h, w) in enumerate(SMALL):
        shape = (n, c, 2 * h, 2 * w) if kernel.startswith("avgpool") else (n, c, h, w)
        for j, tier in enumerate(TIERS):
            check_kernel(kernel, shape, TORCH_DT[dtype], tier, seed=100 * i + j)


def test_upsample_border_infinities_stay_infinite():
    """±inf in input row or column 0 reaches output row / column 0 as ±inf: the tap of weight 0 there is not multiplied
    (0·inf would be NaN)"""
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        x = torch.ones((1, 8, 3, 4), dtype=dtype, device="cuda").contiguous(memory_format=torch.channels_last)
        x[0, 0, 0, 0] = float("inf")                      # corner
        x[0, 1, 0, 2] = float("-inf")                     # row 0
        x[0, 2, 1, 0] = float("inf")                      # column 0
        y = up_fwd(x)
        want = ors.upsample2x(x.double())
        got = y.double()
        for ch, pts in ((0, [(0, 0), (0, 1), (1, 0), (1, 1)]), (1, [(0, 3), (0, 4), (0, 5), (1, 4)]), (2, [(2, 0), (3, 0), (2, 1)])):
            for p in pts:
                assert float(got[0, ch][p]) == float(want[0, ch][p]), (str(dtype), ch, p, got[0, ch].tolist())
        assert_matches(y, want, None, dtype, "border")


# ---- the shapes res50 and aim_res50 pass to each kernel ----------------------------------------------------------------
_RES50: dict = {}


def _res50_shapes(size, model="res50"):
    """{kernel: sorted forward-input shapes} of one bs-16 `model` training iteration at size², recorded at the C ABI;
    "nearest_calls": the number of nearest forward launches"""
    if (model, size) in _RES50:
        return _RES50[(model, size)]
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.synthetic import synth_batch
    real = resample._lib
    calls = []

    class _Lib:
        def __init__(self, h):
            self._h = h

        def __getattr__(self, name):
            fn = getattr(self._h, name)

            def wrapped(*a):
                calls.append((name, a))
                return fn(*a)
            return wrapped

    class _Rec:
        def __getattr__(self, name):
            return getattr(real, name)

        def lib(self):
            return _Lib(real.lib())

    tr = Trainer(model_name=model, dtype=torch.bfloat16, channels_last=True, use_graph=False)
    x, m = synth_batch(7, 16, size)
    resample._lib = _Rec()
    try:
        tr.step(x.cuda(), m.cuda())
        torch.cuda.synchronize()
    finally:
        resample._lib = real
    del tr
    shapes = {}
    for name, a in calls:
        if name == "sod_upsample2x_bilinear_fwd":
            k, s = "upsample_fwd", (a[3], a[6], a[4], a[5])
        elif name == "sod_upsample2x_bilinear_bwd":
            k, s = "upsample_bwd", (a[2], a[5], a[3], a[4])
        elif name in ("sod_avgpool2x2_fwd", "sod_avgpool2x2_bwd"):
            k, s = ("avgpool_fwd" if name.endswith("fwd") else "avgpool_bwd"), (a[2], a[5], 2 * a[3], 2 * a[4])
        elif name == "sod_maxpool3x3s2_fwd":
            k, s = "maxpool_fwd", (a[3], a[6], a[4], a[5])
        elif name == "sod_maxpool3x3s2_bwd":
            k, s = "maxpool_bwd", (a[3], a[6], a[4], a[5])
        elif name == "sod_colsum":
            k, s = "colsum", (a[2], a[3])
        elif name in ("sod_upsample2x_nearest_fwd", "sod_upsample2x_nearest_bwd"):
            k, s = ("nearest_fwd" if name.endswith("fwd") else "nearest_bwd"), (a[2], a[5], a[3], a[4])
        else:
            continue
        shapes.setdefault(k, set()).add(s)
    out = {k: sorted(v) for k, v in shapes.items()}
    out["nearest_calls"] = sum(name == "sod_upsample2x_nearest_fwd" for name, _ in calls)
    _RES50[(model, size)] = out
    return out


@pytest.mark.parametrize("size", [256, 320, 384])
def test_res50_shapes(size):
    shapes = dict(_res50_shapes(size))
    assert shapes.pop("nearest_calls") == 0                                  # res50 has no nearest up-sample
    assert set(shapes) == set(geo.KERNELS) | {"colsum"}, sorted(shapes)
    for kernel in geo.KERNELS:
        for i, shape in enumerate(shapes[kernel]):
            for dtype in geo.DTYPES:
                for j, tier in enumerate(("exact", "random")):
                    check_kernel(kernel, shape, TORCH_DT[dtype], tier, seed=size + 10 * i + j)
    for rows, c in shapes["colsum"]:
        for dtype in geo.DTYPES:
            for tier in ("exact", "random"):
                check_colsum(rows, c, TORCH_DT[dtype], tier, seed=rows + c)


@pytest.mark.parametrize("size", [320, 352])
def test_aim_res50_nearest_shapes(size):
    """the twelve nearest up-samples of one bs-16 aim_res50 iteration (64 channels at S/4 … S/32, 1024 at S/32), forward
    and backward, in every dtype and tier; at 320² the largest run the grid-stride loop twice on a 132-SM H100"""
    shapes = _res50_shapes(size, "aim_res50")
    assert shapes["nearest_calls"] == 12
    q = size // 4
    want = sorted({(16, 64, q >> k, q >> k) for k in range(4)} | {(16, 1024, q // 8, q // 8)})
    assert shapes["nearest_fwd"] == shapes["nearest_bwd"] == want, shapes["nearest_fwd"]
    for kernel in ("nearest_fwd", "nearest_bwd"):
        for i, shape in enumerate(shapes[kernel]):
            for dtype in geo.DTYPES:
                for j, tier in enumerate(TIERS):
                    check_kernel(kernel, shape, TORCH_DT[dtype], tier, seed=size + 10 * i + j)


# ---- sod_colsum ----------------------------------------------------------------------------------------------------------
def check_colsum(rows, c, dtype, tier, seed):
    import numpy as np
    g = _gen(seed)
    if tier == "exact":
        hi = 8 if rows > 1 << 18 else 64
        x = torch.randint(-hi, hi + 1, (rows, c), generator=g, device="cuda").float()
    else:
        x = torch.randn((rows, c), generator=g, device="cuda")
    if tier == "special":
        big = torch.finfo(dtype).max
        x[0, 0] = float("inf")
        x[rows - 1, c - 1] = float("-inf")
        x[rows // 2, min(1, c - 1)] = float("nan")
        if c >= 8:
            x[:, 2] = big                                     # overflows the fp32 chain (or the final rounding)
            x[:, 3] = torch.randint(-64, 65, (rows,), generator=g, device="cuda").float() * _sub(dtype)
    x = x.to(dtype)
    got = colsum(x)
    with np.errstate(over="ignore", invalid="ignore"):
        want = torch.from_numpy(geo.colsum_replay(x.float().cpu().numpy(), _sm())).cuda().to(dtype)
    assert_matches(got, want.double(), None, dtype, f"colsum {rows}x{c} {tier}")
    if tier == "exact":
        assert torch.equal(got, x.double().sum(0).to(dtype)), "integer column sums must be exact"
    assert torch.equal(colsum(x).view(torch.uint8), got.view(torch.uint8)), "two launches differ"


COLSUM_CASES = [(d, j) for d in geo.DTYPES for j in range(len(geo.COLSUM_SPECS))]


@pytest.mark.parametrize("dtype, spec", COLSUM_CASES, ids=[f"{d}-s{j}" for d, j in COLSUM_CASES])
def test_colsum_regime(dtype, spec):
    sm = _sm()
    want = geo.COLSUM_SPECS[spec]
    rows = geo.select_colsum(want, sm)
    assert rows is not None, f"{want} unreachable on {sm} SMs"
    c = 8 * want["L"]
    for j, tier in enumerate(TIERS):
        check_colsum(rows, c, TORCH_DT[dtype], tier, seed=1000 * spec + j)
    RAN[f"colsum-{dtype}-s{spec}"] = {(f"colsum<{dtype}>",) + cell for cell in geo.colsum_cells(geo.colsum_launch(rows, c, sm))}


def test_every_regime_cell_ran_on_this_device():
    """every (kernel, dtype, wave) and every colsum (dtype, axis value) cell was reached by a passing case"""
    if not RAN:
        pytest.skip("the regime cases did not run in this session")
    want_cases = [f"{k}-{d}-{w}" for k, d, w in WAVE_CASES] + [f"colsum-{d}-s{j}" for d, j in COLSUM_CASES]
    missing_cases = [c for c in want_cases if c not in RAN]
    assert not missing_cases, f"{len(missing_cases)} regime cases did not pass: {missing_cases[:5]}"
    required = {(k, d, w) for k, d, w in WAVE_CASES} | {(f"colsum<{d}>",) + cell for d in geo.DTYPES
                                                         for cell in geo.required_colsum_cells()}
    missing = required - set().union(*RAN.values())
    assert not missing, sorted(missing, key=str)


# ---- refusals ------------------------------------------------------------------------------------------------------------
SENTINEL = 0x5A


def _sentinel(nbytes):
    return torch.full((nbytes + 64,), SENTINEL, dtype=torch.uint8, device="cuda")


def _refuse(fn, args, code, outs, what):
    rc = fn(*args)
    torch.cuda.synchronize()
    assert rc == code, f"{what}: returned {rc}, expected {code}"
    for o in outs:
        assert bool((o == SENTINEL).all()), f"{what}: the output was written"


@pytest.mark.parametrize("entry", ["up_fwd", "up_bwd", "avg_fwd", "avg_bwd", "max_fwd", "max_bwd", "near_fwd", "near_bwd"])
def test_grid_stride_entries_refuse_bad_arguments(entry):
    L = _lib()
    lib, st, f32 = L.lib(), L.stream_ptr(), L.SOD_F32
    n, h, w, c = 2, 6, 4, 16
    src = torch.zeros(n * 4 * h * w * c + 64, dtype=torch.float32, device="cuda")
    out = _sentinel(n * 4 * h * w * c * 4)
    arg = _sentinel(n * h * w * c)
    s, o, a = src.data_ptr(), out.data_ptr(), arg.data_ptr()
    if entry == "up_fwd":
        fn = lib.sod_upsample2x_bilinear_fwd

        def call(p=(s, s, o), dims=(n, h, w, c), dt=f32):
            return (*p, *dims, dt, st)
        ptrs, optional = [0, 2], [1]
    elif entry == "max_fwd":
        fn = lib.sod_maxpool3x3s2_fwd

        def call(p=(s, o, a), dims=(n, h, w, c), dt=f32):
            return (*p, *dims, dt, st)
        ptrs, optional = [0, 1, 2], []
    elif entry == "max_bwd":
        fn = lib.sod_maxpool3x3s2_bwd

        def call(p=(s, a, o), dims=(n, h, w, c), dt=f32):
            return (*p, *dims, dt, st)
        ptrs, optional = [0, 1, 2], []
    else:
        fn = {"up_bwd": lib.sod_upsample2x_bilinear_bwd, "avg_fwd": lib.sod_avgpool2x2_fwd,
              "avg_bwd": lib.sod_avgpool2x2_bwd, "near_fwd": lib.sod_upsample2x_nearest_fwd,
              "near_bwd": lib.sod_upsample2x_nearest_bwd}[entry]

        def call(p=(s, o), dims=(n, h, w, c), dt=f32):
            return (*p, *dims, dt, st)
        ptrs, optional = [0, 1], []
    outs = (out, arg)
    base = list(call()[:len(ptrs) + len(optional)])
    for i in ptrs:                                                   # null pointers
        p = list(base)
        p[i] = None
        _refuse(fn, call(tuple(p)), SOD_EINVAL, outs, f"{entry} null pointer {i}")
    for i in ptrs + optional:                                        # 2-byte misalignment
        p = list(base)
        p[i] = p[i] + 2
        _refuse(fn, call(tuple(p)), SOD_EALIGN, outs, f"{entry} misaligned pointer {i}")
    for k in range(3):                                               # n, h, w ≤ 0
        for bad in (0, -1):
            d = [n, h, w, c]
            d[k] = bad
            _refuse(fn, call(dims=tuple(d)), SOD_EINVAL, outs, f"{entry} dim {k} = {bad}")
    _refuse(fn, call(dims=(n, h, w, 0)), SOD_EINVAL, outs, f"{entry} c = 0")
    for bad_c in (4, 12, 20):
        _refuse(fn, call(dims=(n, h, w, bad_c)), SOD_EUNSUPPORTED, outs, f"{entry} c = {bad_c}")
    for bad_dt in (3, -1, 99):
        _refuse(fn, call(dt=bad_dt), SOD_EINVAL, outs, f"{entry} dtype {bad_dt}")


def test_colsum_refuses_bad_arguments():
    L = _lib()
    lib, st, f32 = L.lib(), L.stream_ptr(), L.SOD_F32
    rows, c = 100, 64
    x = torch.zeros(rows * 4096 + 64, dtype=torch.float32, device="cuda")
    out = _sentinel(4096 * 4)
    ws = torch.zeros(int(lib.sod_colsum_workspace_bytes()) + 64, dtype=torch.uint8, device="cuda")
    nws = int(lib.sod_colsum_workspace_bytes())
    X, O, W = x.data_ptr(), out.data_ptr(), ws.data_ptr()

    def call(xp=X, op=O, wp=W, r=rows, cc=c, dt=f32, nb=nws):
        return (xp, op, r, cc, dt, wp, nb, st)
    fn, outs = lib.sod_colsum, (out,)
    _refuse(fn, call(xp=None), SOD_EINVAL, outs, "x null")
    _refuse(fn, call(op=None), SOD_EINVAL, outs, "out null")
    _refuse(fn, call(wp=None), SOD_EINVAL, outs, "workspace null")
    _refuse(fn, call(r=0), SOD_EINVAL, outs, "rows 0")
    _refuse(fn, call(r=-5), SOD_EINVAL, outs, "rows < 0")
    _refuse(fn, call(cc=0), SOD_EINVAL, outs, "c 0")
    for bad_c in (12, 24, 4096):                                      # C % 8, L not a power of two, C > 2048
        _refuse(fn, call(cc=bad_c), SOD_EUNSUPPORTED, outs, f"c = {bad_c}")
    _refuse(fn, call(xp=X + 2), SOD_EALIGN, outs, "x misaligned")
    _refuse(fn, call(wp=W + 2), SOD_EALIGN, outs, "workspace misaligned")
    _refuse(fn, call(nb=nws - 1), SOD_EWORKSPACE, outs, "short workspace")
    for bad_dt in (3, 99):
        _refuse(fn, call(dt=bad_dt), SOD_EINVAL, outs, f"dtype {bad_dt}")
    # the refusals left the ticket alone: a real sum with this workspace is still right
    x2 = torch.arange(rows * c, dtype=torch.float32, device="cuda").reshape(rows, c) % 7
    assert L.lib().sod_colsum(x2.data_ptr(), O, rows, c, f32, W, nws, st) == 0
    torch.cuda.synchronize()
    assert torch.equal(out[:c * 4].view(torch.float32), x2.double().sum(0).float())
