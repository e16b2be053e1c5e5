"""The data-side kernels — pre-processing, quantize and the saliency head / histogram (csrc/pipeline.cu), the Pillow
resize (csrc/resize.cu) and the training augmentation (csrc/augment.cu) — in every launch regime of this GPU, against
exact and float64 oracles, through the C ABI.

oracle/data_geometry.py picks, for the device the test runs on, the shapes that reach each regime cell: every wave of
the grid-stride pre-processing and quantize loops (a partial wave, one pass, a pass plus a ragged one, two or more passes
ragged and exact), the head kernel's idle threads and thousands of strides per thread, the histogram's 1 … 64 CTAs per
image (capped, and one CTA for a whole large image among tiny ones), the resize's 1 … 128 row-CTAs per image with every
pass structure, and the augmentation's multi-row tiles and one-row tiles of S ≥ 1024.  Every output is filled with a
sentinel before each launch, so an element a launch skips shows.  The last test asserts that every cell was reached.

Bounds.
* Pre-processing, identity path (what evaluation uses): `(u/255 − mean)/std` in IEEE fp32 is what torch's CPU
  ToTensor + Normalize computes for every byte (`oracle.pipeline.normalise_table`), so fp32 must be equal bit for bit
  and bf16 / fp16 equal to that value rounded once.
* Pre-processing, bilinear path: the source coordinate max(s·(o + ½) − ½, 0) is rounded once to fp32 (an FMA, as
  torch's CPU interpolate computes it), which fixes the taps i0, i1 and λ exactly (`oracle.pipeline.bilinear_taps`).
  With exact λ, the float64 value is r = (1−λy)((1−λx)v00 + λx v01) + λy((1−λx)v10 + λx v11) over the fp32 tap values
  v.  The kernel rounds 1 − λ once per axis (an error ≤ 2⁻²⁵, times at most M = max|v| for the pair of taps it weights)
  and then evaluates the expression with two multiplications and two additions on every path from a tap to the result,
  fused or not, so |kernel − r| ≤ γ₄·Σ w|v| + 2⁻²⁴·M ≤ 5·2⁻²⁴·Σ w|v| + 2⁻²⁴·M (γ₄ = 4u/(1 − 4u), u = 2⁻²⁴).  For
  ImageNet normalisation that is below 1.2e-6; a λ off by the twice-rounded coordinate moves the value by up to ≈7e-5.
  The step-edge images (values 0 and 1, constant along one axis) make every output an exact function of λ, so there
  the kernel must equal the oracle bit for bit, at rows where rounding twice gives another λ.  bf16 / fp16 must equal
  the kernel's own fp32 output rounded once.  The mask must equal nearest's min(⌊fp32(o·s)⌋, n − 1) and torch's.
* Quantize: `mul(255).byte()` exactly, at every fp32 k/255 and both its neighbours; with sigmoid, torch CUDA's
  `sigmoid().mul(255).byte()` exactly, and off ⌊255·σ(x)⌋ (float64) only where 255·σ(x) is within 4 fp32 ulps of an
  integer; 2-byte inputs as their fp32 value.  Out of range the kernel clamps: below 0 and −inf give 0, above 1 and
  +inf give 255, NaN gives 0 (PTX's float-to-integer conversion of NaN; the contract recorded here).
* Head and histogram: exactly an oracle written from the reference's formulas (binarise g/(max + 1e-8) > 0.5 in
  float64, centre of mass from np.nonzero with Python round, quadrants by slicing); then `SaliencyMetrics` against
  `oracle.metrics.TotalMetric` at the tolerances of tests/test_gpu_pipeline.py.  Where the reference's S-measure is
  NaN (an empty quadrant, or a one-pixel one) the product's must be finite: the documented deviation.
* Resize and augmentation: Pillow (and torchvision's ColorJitter) byte for byte.
"""
import ctypes as C
import itertools
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

from oracle import data_geometry as geo
from oracle import metrics as om
from oracle import pipeline as opipe

pytestmark = pytest.mark.gpu

TORCH_DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}
DTYPES = tuple(TORCH_DT)
RAN: dict = {}              # case id → regime cells it reached on this device
U = 2.0 ** -24
SENTINEL = 0x5A


def _sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _lib():
    from distributed_sod_project_b200 import _lib
    return _lib


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _seed(*key):
    return zlib.crc32(repr(key).encode())


def _record(case, kernel, cells):
    RAN.setdefault(case, set()).update((kernel,) + c for c in cells)


# ---- pre-processing -------------------------------------------------------------------------------------------------
def preprocess(img, mask, flip, dtype, ho, wo, mean=opipe.MEAN, std=opipe.STD):
    """the C ABI on sentinel-filled outputs (NaN image, −1 mask) → (image [n, ho, wo, 3], mask [n, ho, wo] or None)"""
    L = _lib()
    n, hs, ws, _ = img.shape
    out = torch.full((n, ho, wo, 3), float("nan"), dtype=dtype, device="cuda")
    mout = torch.full((n, 1, ho, wo), -1.0, device="cuda") if mask is not None else None
    rc = L.lib().sod_preprocess_batch(img.data_ptr(), None if mask is None else mask.data_ptr(),
                                      None if flip is None else flip.data_ptr(), out.data_ptr(), L.dtype_code(dtype),
                                      None if mout is None else mout.data_ptr(), n, hs, ws, ho, wo,
                                      (C.c_float * 3)(*mean), (C.c_float * 3)(*std), L.stream_ptr())
    L.check(rc, "sod_preprocess_batch")
    torch.cuda.synchronize()
    return out, None if mout is None else mout[:, 0]


def _flipped(x, flip):
    if flip is None:
        return x
    x = x.clone()
    f = flip.bool()
    x[f] = x[f].flip(2)
    return x


def prep_oracle(img, flip, ho, wo, table):
    """→ (float64 value [n, ho, wo, 3], bound or None where the value is exact)"""
    src = _flipped(img, flip).long()
    v = torch.stack([table[c][src[..., c]] for c in range(3)], -1).double()
    n, hs, ws, _ = img.shape
    if (hs, ws) == (ho, wo):
        return v, None
    y0, y1, ly = (torch.from_numpy(a).cuda() for a in opipe.bilinear_taps(hs, ho))
    x0, x1, lx = (torch.from_numpy(a).cuda() for a in opipe.bilinear_taps(ws, wo))
    ly, lx = ly[None, :, None, None], lx[None, None, :, None]
    hy, hx = 1 - ly, 1 - lx
    r0, r1 = v[:, y0], v[:, y1]
    v00, v01, v10, v11 = r0[:, :, x0], r0[:, :, x1], r1[:, :, x0], r1[:, :, x1]
    ref = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11)
    a00, a01, a10, a11 = v00.abs(), v01.abs(), v10.abs(), v11.abs()
    mag = hy * (hx * a00 + lx * a01) + ly * (hx * a10 + lx * a11)
    m = torch.maximum(torch.maximum(a00, a01), torch.maximum(a10, a11))
    return ref, 5 * U * mag + U * m


_TABLES = {}


def _table(mean=opipe.MEAN, std=opipe.STD):
    key = (mean, std)
    if key not in _TABLES:
        _TABLES[key] = opipe.normalise_table(mean, std).cuda()
    return _TABLES[key]


def check_preprocess(img, mask, flip, ho, wo, what):
    n, hs, ws, _ = img.shape
    want, tol = prep_oracle(img, flip, ho, wo, _table())
    x32, m32 = preprocess(img, mask, flip, torch.float32, ho, wo)
    if tol is None:
        assert torch.equal(x32, want.float()), f"{what}: identity path not bit-exact"
    else:
        bad = ~((x32.double() - want).abs() <= tol)
        if bool(bad.any()):
            i = bad.nonzero()[0].tolist()
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} off, first at {i}: got {float(x32[tuple(i)])!r} "
                                 f"float64 {float(want[tuple(i)])!r} bound {float(tol[tuple(i)]):.3g}")
    for dt in (torch.bfloat16, torch.float16):
        x16, m16 = preprocess(img, mask, flip, dt, ho, wo)
        assert torch.equal(x16, x32.to(dt)), f"{what}: {dt} is not the fp32 output rounded once"
        if mask is not None:
            assert torch.equal(m16, m32)
    if mask is not None:
        msrc = _flipped(mask, flip).long()
        iy = torch.from_numpy(opipe.nearest_index(hs, ho)).cuda()
        ix = torch.from_numpy(opipe.nearest_index(ws, wo)).cuda()
        mtab = (torch.arange(256, dtype=torch.float32) / 255).cuda()
        assert torch.equal(m32, mtab[msrc[:, iy][:, :, ix]]), f"{what}: mask differs from floor(fp32(o·s))"
        # (the table holds the IEEE quotients: torch's CUDA division by a scalar multiplies by its reciprocal)
        near = F.interpolate(mtab[msrc][:, None], size=(ho, wo), mode="nearest")[:, 0]
        assert torch.equal(m32, near), f"{what}: mask differs from torch nearest"


def _image(n, h, w, seed):
    """random bytes with a saturated band (0 / 255) across the top third"""
    g = _gen(seed)
    img = torch.randint(0, 256, (n, h, w, 3), generator=g, device="cuda", dtype=torch.uint8)
    band = max(h // 3, 1) if h > 2 else 0
    img[:, :band] = torch.where(img[:, :band] > 127, 255, 0).to(torch.uint8)
    mask = torch.randint(0, 256, (n, h, w), generator=g, device="cuda", dtype=torch.uint8)
    flip = (torch.arange(n, device="cuda") % 2).to(torch.uint8)
    return img, mask, flip


PREP_CASES = [(w, m) for w in geo.WAVES for m in geo.PREP_MODES]


@pytest.mark.parametrize("wave, mode", PREP_CASES, ids=[f"{w}-{m}" for w, m in PREP_CASES])
def test_preprocess_regime(wave, mode):
    sm = _sm()
    shape = geo.select("preprocess", ("wave", wave, mode), sm)
    n, hs, ws, ho, wo = shape
    img, mask, flip = _image(n, hs, ws, _seed("prep", wave, mode))
    check_preprocess(img, mask, flip, ho, wo, f"{shape} mask+flip")
    check_preprocess(img, None, None, ho, wo, f"{shape} plain")
    _record(f"prep-{wave}-{mode}", "preprocess", geo.cells("preprocess", shape, sm))


@pytest.mark.parametrize("shape", [(1, 1, 1, 5, 7), (3, 5, 7, 1, 1), (2, 1, 1, 1, 1), (2, 1, 9, 4, 1), (2, 9, 1, 1, 4),
                                   (4, 37, 53, 64, 64), (5, 64, 64, 48, 80), (3, 320, 320, 224, 224)])
def test_preprocess_small_and_one_pixel_shapes(shape):
    n, hs, ws, ho, wo = shape
    img, mask, flip = _image(n, hs, ws, _seed("prep-small", shape))
    check_preprocess(img, mask, flip, ho, wo, f"{shape}")
    _record(f"prep-small-{shape}", "preprocess", geo.cells("preprocess", shape, _sm()))


@pytest.mark.parametrize("size", [None, 256, 288, 352, 384])
def test_preprocess_production_geometries(size):
    """320² at bs 16 to every multi-scale training size, and the evaluation identity path"""
    img, mask, flip = _image(16, 320, 320, _seed("prep-prod", size))
    s = size or 320
    check_preprocess(img, mask, flip, s, s, f"320 -> {s}")
    check_preprocess(img, None, None, s, s, f"320 -> {s} plain")


# (n_in, n_out, output rows where one rounding of s·(o + ½) − ½ and two roundings give different λ)
TWO_ROUNDING_ROWS = ((320, 224, (1, 22, 179)), (320, 288, (14, 115, 230)), (256, 384, (3, 12, 48, 192)),
                     (384, 416, (17, 277)))


@pytest.mark.parametrize("n_in, n_out, rows", TWO_ROUNDING_ROWS)
def test_preprocess_bilinear_coordinate_is_rounded_once(n_in, n_out, rows):
    """step edges: source rows i1(o) of the listed rows hold 1, the rest 0 (mean 0, std 1), constant along the other
    axis, so every output is fp32((1 − λ)·a + λ·b) with a, b ∈ {0, 1}, exactly; torch CPU agrees at the listed rows"""
    i0, i1, lam = opipe.bilinear_taps(n_in, n_out)
    _, _, lam2 = opipe.bilinear_taps(n_in, n_out, fused=False)
    assert all(lam[o] != lam2[o] for o in rows)
    hot = np.zeros(n_in, bool)
    hot[[i1[o] for o in rows]] = True
    assert not any(hot[i0[o]] for o in rows)
    a, b = hot[i0].astype(np.float64), hot[i1].astype(np.float64)
    hy = (1 - lam).astype(np.float32).astype(np.float64)
    want = torch.from_numpy((hy * a + lam * b).astype(np.float32))
    for axis in (0, 1):
        u = torch.from_numpy(hot.astype(np.uint8) * 255)
        plane = u[:, None].expand(n_in, 8) if axis == 0 else u[None, :].expand(8, n_in)
        img = plane[None, :, :, None].expand(1, *plane.shape, 3).contiguous().cuda()
        ho, wo = (n_out, 8) if axis == 0 else (8, n_out)
        for dt in DTYPES:
            x, _ = preprocess(img, None, None, TORCH_DT[dt], ho, wo, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0))
            x = x.float().cpu()
            got = x[0, :, 0, 0] if axis == 0 else x[0, 0, :, 0]
            assert bool((x == (got[:, None, None] if axis == 0 else got[None, :, None])).all())
            assert torch.equal(got, want.to(TORCH_DT[dt]).float()), (axis, dt, (got != want).nonzero().flatten().tolist())
        t = F.interpolate(img.permute(0, 3, 1, 2).float().cpu() / 255, size=(ho, wo), mode="bilinear", align_corners=False)
        tl = t[0, 0, :, 0] if axis == 0 else t[0, 0, 0, :]
        for o in rows:
            assert float(tl[o]) == float(want[o]) == lam[o], (axis, o)


# ---- quantize ---------------------------------------------------------------------------------------------------------
def quantize(x, sigmoid):
    L = _lib()
    out = torch.full(x.shape, SENTINEL, dtype=torch.uint8, device="cuda")
    rc = L.lib().sod_saliency_quantize(x.data_ptr(), L.dtype_code(x.dtype), out.data_ptr(), x.numel(), int(sigmoid),
                                       L.stream_ptr())
    L.check(rc, "sod_saliency_quantize")
    torch.cuda.synchronize()
    return out


def _quant_specials(sigmoid):
    inf, nan = float("inf"), float("nan")
    if not sigmoid:
        k = (torch.arange(256, dtype=torch.float64) / 255).float()
        near = torch.cat([k, torch.nextafter(k, torch.tensor(2.0)), torch.nextafter(k, torch.tensor(-1.0))])
        return torch.cat([near, torch.tensor([0.0, -0.0, 1.0, -1.0, 2.0, 1.0000001, -1e-45, 1e-45, inf, -inf, nan, 1e30, -1e30])])
    p = (torch.arange(1, 255, dtype=torch.float64) / 255)
    logit = torch.log(p / (1 - p)).float()                             # 255·σ(x) lands next to every integer
    near = torch.cat([logit, torch.nextafter(logit, torch.tensor(inf)), torch.nextafter(logit, torch.tensor(-inf))])
    return torch.cat([near, torch.tensor([0.0, -0.0, 1e-45, -1e-45, 88.0, -88.0, 104.0, -104.0, 1e30, -1e30, inf, -inf, nan])])


def quant_oracle(x, sigmoid):
    """the kernel's contract in float64: clamp(fp32(255·x), 0, 255) truncated, NaN → 0 (no sigmoid)"""
    t = (x.double() * 255).float().double()                            # x·255 is exact in float64: one fp32 rounding
    t = torch.nan_to_num(t, nan=0.0).clamp(0, 255)
    return t.floor().to(torch.uint8)


def check_quantize(total, dtype, sigmoid, seed, what):
    g = _gen(seed)
    if sigmoid:
        x = torch.randn(total, generator=g, device="cuda") * 8
    else:
        x = torch.rand(total, generator=g, device="cuda")
    sp = _quant_specials(sigmoid).cuda()
    k = min(sp.numel(), total)
    x[:k] = sp[:k]
    x[total - k:] = sp[sp.numel() - k:]                                 # the same values in the last pass too
    x = x.to(TORCH_DT[dtype])
    got = quantize(x, sigmoid)
    xf = x.float()
    assert torch.equal(got, quantize(xf, sigmoid)), f"{what}: {dtype} input is not its fp32 value"
    nan = xf.isnan()
    assert bool((got[nan] == 0).all()), f"{what}: NaN does not give 0"
    if not sigmoid:
        assert torch.equal(got, quant_oracle(xf, False)), f"{what}: differs from clamp(fp32(255 x)) truncated"
        inr = (xf >= 0) & (xf <= 1)
        assert torch.equal(got[inr], xf[inr].mul(255).byte()), f"{what}: differs from mul(255).byte()"
        assert bool((got[xf > 1] == 255).all()) and bool((got[xf < 0] == 0).all())
        return
    want = xf.sigmoid().mul(255).byte()
    assert torch.equal(got[~nan], want[~nan]), f"{what}: differs from torch sigmoid().mul(255).byte() at " \
                                                f"{(got != want)[~nan].nonzero().flatten()[:5].tolist()}"
    t = torch.sigmoid(xf.double()) * 255
    k64 = t.floor()
    off = (~nan) & (got.double() != k64)
    ulp = torch.exp2(torch.floor(torch.log2(t.clamp_min(2.0 ** -126))) - 23)
    near_int = (t - t.round()).abs() <= 4 * ulp
    assert bool((near_int[off]).all()) and bool(((got.double() - k64).abs()[off] <= 1).all()), \
        f"{what}: {int((off & ~near_int).sum())} results off floor(255 σ(x)) away from an integer"


QUANT_CASES = [(w, d, s) for w in geo.WAVES for d in DTYPES for s in (False, True)]


@pytest.mark.parametrize("wave, dtype, sigmoid", QUANT_CASES, ids=[f"{w}-{d}-{'sig' if s else 'lin'}" for w, d, s in QUANT_CASES])
def test_quantize_regime(wave, dtype, sigmoid):
    sm = _sm()
    (total,) = geo.select("quantize", ("wave", wave), sm)
    check_quantize(total, dtype, sigmoid, _seed("quant", wave, dtype, sigmoid), f"quantize {total} {dtype}")
    _record(f"quant-{wave}-{dtype}-{sigmoid}", "quantize", geo.cells("quantize", (total,), sm))


def test_quantize_tiny():
    for total in (1, 2, 255, 256):
        for sigmoid in (False, True):
            check_quantize(total, "float32", sigmoid, total, f"quantize {total}")


# ---- saliency head and histogram ---------------------------------------------------------------------------------------
def metric_oracle(p8, g8):
    """(head int64[8], split (cy, cx), hist int64[4, 2, 256]) from the reference's formulas, written independently of the
    kernels: float64 binarisation, np.nonzero centre of mass with Python round, quadrants by slicing"""
    h, w = p8.shape
    gmax = int(g8.max())
    gb = g8 / (gmax + 1e-8) > 0.5
    ys, xs = np.nonzero(gb)
    n_fg = len(ys)
    head = np.array([p8.min(), p8.max(), gmax, 0, n_fg, ys.sum(), xs.sum(), 0], dtype=np.int64)
    # SaliencyMetrics splits an empty ground truth at (1, 1); the reference never forms its quadrants
    cy, cx = (int(round(ys.mean())) + 1, int(round(xs.mean())) + 1) if n_fg else (1, 1)
    k = p8.astype(np.int64) - int(p8.min())
    hist = np.zeros((4, 2, 256), dtype=np.int64)
    for q, (r0, r1, c0, c1) in enumerate(((0, cy, 0, cx), (0, cy, cx, w), (cy, h, 0, cx), (cy, h, cx, w))):
        for b in (0, 1):
            sel = gb[r0:r1, c0:c1] == b
            hist[q, b] = np.bincount(k[r0:r1, c0:c1][sel], minlength=256)
    return head, (cy, cx), hist


def _gt(kind, h, w, rng):
    if kind == "soft2":                                               # 2g == gmax at g = 1
        g = rng.integers(0, 3, (h, w))
        g.flat[0] = 2
    elif kind == "soft254":
        g = rng.choice([0, 126, 127, 128, 254], (h, w))
        g.flat[-1] = 254
    elif kind == "max1":
        g = rng.integers(0, 2, (h, w))
    elif kind == "max255":
        g = rng.integers(0, 256, (h, w))
    elif kind == "empty":
        g = np.zeros((h, w))
    elif kind == "full":
        g = np.full((h, w), 255)
    elif kind in ("row0", "rowN", "col0", "colN"):
        g = np.zeros((h, w))
        {"row0": lambda: g.__setitem__((0, slice(None)), 255), "rowN": lambda: g.__setitem__((h - 1, slice(None)), 255),
         "col0": lambda: g.__setitem__((slice(None), 0), 255), "colN": lambda: g.__setitem__((slice(None), w - 1), 255)}[kind]()
    elif kind == "half":                      # a diagonal of 2 or 4 pixels: centre of mass at .5 or 1.5 on both axes
        g = np.zeros((h, w))
        m = 4 if min(h, w) >= 4 else min(h, w, 2)
        g[np.arange(m), np.arange(m)] = 255
    else:
        raise KeyError(kind)
    return g.astype(np.uint8)


def _pred(kind, h, w, rng):
    if kind in (0, 77, 255):
        return np.full((h, w), kind, np.uint8)
    if kind == "levels":
        return rng.permutation(np.arange(h * w) % 256).reshape(h, w).astype(np.uint8)
    return rng.integers(0, 256, (h, w)).astype(np.uint8)


GT_KINDS = ("soft2", "soft254", "max1", "max255", "empty", "full", "row0", "rowN", "col0", "colN", "half")
PRED_KINDS = (0, 77, 255, "levels", "random")
TINY = ((1, 1), (1, 7), (9, 1), (2, 2), (3, 5), (1, 2), (2, 1), (4, 4))


def _images(sizes, seed):
    rng = np.random.default_rng(seed)
    preds, gts = [], []
    for i, (h, w) in enumerate(sizes):
        preds.append(_pred(PRED_KINDS[i % len(PRED_KINDS)], h, w, rng))
        gts.append(_gt(GT_KINDS[(i // len(PRED_KINDS) + i) % len(GT_KINDS)], h, w, rng))
    return preds, gts


def _ragged(arrays):
    from distributed_sod_project_b200.pipeline import Ragged
    flat = torch.from_numpy(np.concatenate([a.reshape(-1) for a in arrays])).cuda()
    return Ragged(flat, torch.tensor([a.shape[:2] for a in arrays], dtype=torch.int32), 1)


def check_metric_kernels(preds, gts, ragged, what):
    """head and hist exactly against metric_oracle; the split the product derives from the head is the oracle's"""
    from distributed_sod_project_b200.metrics import SaliencyMetrics
    L = _lib()
    lib, s = L.lib(), L.stream_ptr()
    n = len(preds)
    want = [metric_oracle(p, g) for p, g in zip(preds, gts)]
    head = torch.full((n, 8), -7, dtype=torch.int64, device="cuda")
    hist = torch.zeros((n, 4, 2, 256), dtype=torch.int32, device="cuda")
    split = torch.tensor([w[1] for w in want], dtype=torch.int32, device="cuda")
    if ragged:
        p, g = _ragged(preds), _ragged(gts)
        assert lib.sod_saliency_head_ragged(p.data.data_ptr(), g.data.data_ptr(), n, p.off_d.data_ptr(), p.hw_d.data_ptr(),
                                            head.data_ptr(), s) == 0
        torch.cuda.synchronize()
        assert torch.equal(SaliencyMetrics._split(head), split), f"{what}: the product's split is not the oracle's"
        assert lib.sod_saliency_hist_ragged(p.data.data_ptr(), g.data.data_ptr(), n, p.off_d.data_ptr(), p.hw_d.data_ptr(),
                                            head.data_ptr(), split.data_ptr(), hist.data_ptr(), s) == 0
    else:
        h, w = preds[0].shape
        pf, gf = torch.from_numpy(np.stack(preds)).cuda(), torch.from_numpy(np.stack(gts)).cuda()
        assert lib.sod_saliency_head(pf.data_ptr(), gf.data_ptr(), n, h, w, head.data_ptr(), s) == 0
        torch.cuda.synchronize()
        assert torch.equal(SaliencyMetrics._split(head), split), f"{what}: the product's split is not the oracle's"
        assert lib.sod_saliency_hist(pf.data_ptr(), gf.data_ptr(), n, h, w, head.data_ptr(), split.data_ptr(),
                                     hist.data_ptr(), s) == 0
    torch.cuda.synchronize()
    hh, hs = head.cpu().numpy(), hist.cpu().numpy().astype(np.int64)
    for i, (wh, _, whist) in enumerate(want):
        assert np.array_equal(hh[i], wh), f"{what}: image {i} {preds[i].shape} head {hh[i].tolist()} want {wh.tolist()}"
        assert np.array_equal(hs[i], whist), f"{what}: image {i} {preds[i].shape} histogram differs in " \
                                             f"{int((hs[i] != whist).sum())} counters"


def check_metrics_show(preds, gts, what):
    """SaliencyMetrics.update_ragged / show against TotalMetric; images whose reference S-measure is NaN separately"""
    from distributed_sod_project_b200.metrics import SaliencyMetrics
    with np.errstate(all="ignore"):
        sm_ref = [om.smeasure(*om.normalise(p, g)) for p, g in zip(preds, gts)]
    groups = {True: [i for i, v in enumerate(sm_ref) if np.isfinite(v)], False: [i for i, v in enumerate(sm_ref) if not np.isfinite(v)]}
    for finite, idx in groups.items():
        if not idx:
            continue
        cal = SaliencyMetrics(num=len(idx))
        cal.update_ragged(_ragged([preds[i] for i in idx]), _ragged([gts[i] for i in idx]))
        res = cal.show()
        tot = om.TotalMetric(len(idx), with_wfm=False)
        with np.errstate(all="ignore"):
            for i in idx:
                tot.update(*om.normalise(preds[i], gts[i]))
            want = tot.show()
        for k in ("MaxF", "MeanF", "MAE", "EM"):
            assert res[k] == pytest.approx(float(want[k]), rel=1e-10), (what, finite, k)
        if finite:
            assert res["SM"] == pytest.approx(float(want["SM"]), rel=2e-7), (what, k)
        else:
            assert math.isfinite(res["SM"]) and not math.isfinite(float(want["SM"])), (what, res["SM"])


@pytest.mark.parametrize("cell", ["idle", "1", "mid", "cap"])
def test_metric_fixed_entry_regime(cell):
    sm = _sm()
    (hw,) = geo.select("hist_fixed", ("image", cell), sm)
    shapes = [hw, (hw[1], hw[0])] if hw[0] != hw[1] else [hw]
    if cell == "cap":
        shapes.append((700, 1000))                                     # 700k px: each of the 64 CTAs strides 43 times
    for j, (h, w) in enumerate(shapes):
        preds, gts = _images([(h, w)] * len(GT_KINDS), _seed("fixed", cell, j))
        check_metric_kernels(preds, gts, False, f"fixed {h}x{w}")
        _record(f"fixed-{cell}-{j}", "hist_fixed", geo.cells("hist_fixed", [(h, w)], sm))
        _record(f"fixed-{cell}-{j}", "head", geo.cells("head", [(h, w)], sm))


def _ragged_sizes(cell, sm):
    n = len(geo.select("hist_ragged", ("per", cell), sm))
    if cell == "max":
        n = max(n, 8) if geo.hist_ragged_cell(8, sm) == "max" else n
        big = [(2000, 1500), (16, 32), (1, 513)][:n]                   # 3 Mpx: every head thread strides 5,860 times
        return big + [TINY[i % len(TINY)] for i in range(n - len(big))]
    if cell == "mid":
        return [(320, 320), (300, 400), (1, 1), (53, 1)] + [TINY[i % len(TINY)] for i in range(max(n - 4, 0))]
    return [(1000, 700)] + [TINY[i % len(TINY)] for i in range(n - 1)]  # one CTA per image: a large one among tiny ones


@pytest.mark.parametrize("cell", ["max", "mid", "1"])
def test_metric_ragged_entry_regime(cell):
    sm = _sm()
    sizes = _ragged_sizes(cell, sm)
    assert geo.hist_ragged_cell(len(sizes), sm) == cell
    preds, gts = _images(sizes, _seed("ragged", cell))
    check_metric_kernels(preds, gts, True, f"ragged {cell} n={len(sizes)}")
    check_metrics_show(preds, gts, f"ragged {cell}")
    _record(f"ragged-{cell}", "hist_ragged", geo.cells("hist_ragged", sizes, sm))
    _record(f"ragged-{cell}", "head", geo.cells("head", sizes, sm))


# ---- resize ------------------------------------------------------------------------------------------------------------
def _content(rng, h, w, ch):
    """noise over a hard-edged half: every tap and the clipping at 0 and 255 matter"""
    a = rng.integers(0, 256, (h, w) if ch == 1 else (h, w, ch)).astype(np.uint8)
    a[: h // 2] = np.where(a[: h // 2] > 127, 255, 0)
    return a


# every pass structure, 1-pixel axes, ≥ 100× down (bicubic: ~1,200 taps per output pixel) and ≥ 100× up
RESIZE_GEOS = (((57, 83), (57, 83)), ((40, 90), (40, 33)), ((90, 40), (29, 40)), ((37, 53), (64, 41)),
               ((1, 1), (1, 1)), ((1, 1), (5, 3)), ((1, 90), (40, 1)), ((77, 1), (1, 77)), ((2, 2), (1, 1)),
               ((6, 3000), (6, 20)), ((2500, 5), (12, 5)), ((3, 2), (400, 300)), ((1, 4), (150, 4)))
RESIZE_MODES = [(ch, f) for ch in (1, 3) for f in ("bilinear", "bicubic")]


def resize(srcs, dst_hw, ch, filt, short=0):
    """the C ABI on a sentinel-filled destination; `short`: bytes less workspace than the query asks for"""
    from distributed_sod_project_b200.pipeline import Ragged
    L = _lib()
    code = L.SOD_RESIZE_BILINEAR if filt == "bilinear" else L.SOD_RESIZE_BICUBIC
    src = Ragged(torch.from_numpy(np.concatenate([a.reshape(-1) for a in srcs])).cuda(),
                 torch.tensor([a.shape[:2] for a in srcs], dtype=torch.int32), ch)
    dst = Ragged.empty(torch.tensor(dst_hw, dtype=torch.int32), ch, "cuda")
    dst.data.fill_(SENTINEL)
    ws_n = L.lib().sod_resize_u8_workspace_bytes(len(srcs), src.hw.data_ptr(), dst.hw.data_ptr(), ch, code)
    assert ws_n > 0
    ws = torch.full((ws_n,), SENTINEL, dtype=torch.uint8, device="cuda")
    rc = L.lib().sod_resize_u8(src.data.data_ptr(), src.off_d.data_ptr(), src.hw_d.data_ptr(), dst.data.data_ptr(),
                               dst.off_d.data_ptr(), dst.hw_d.data_ptr(), len(srcs), ch, code, ws.data_ptr(), ws_n - short,
                               L.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    return [dst.image(i).cpu().numpy() for i in range(len(srcs))]


def _pillow(a, hw, ch, filt):
    return np.asarray(Image.fromarray(a, "L" if ch == 1 else "RGB").resize((hw[1], hw[0]),
                                                                          Image.BILINEAR if filt == "bilinear" else Image.BICUBIC))


def _resize_batch(cell, sm):
    """(sources' and outputs' sizes) for a batch in row-CTA regime `cell`, cycling through RESIZE_GEOS"""
    n = geo.select("resize", ("per", cell), sm)[0]
    if cell == "max":
        return [[g] for g in RESIZE_GEOS]                              # one launch per geometry, n = 1
    if cell == "mid":
        n = max(n, len(RESIZE_GEOS)) if geo.resize_cell(len(RESIZE_GEOS), sm) == "mid" else n
        return [[RESIZE_GEOS[i % len(RESIZE_GEOS)] for i in range(n)]]
    tiny = (((3, 4), (3, 4)), ((3, 4), (3, 7)), ((5, 2), (2, 2)), ((1, 1), (2, 3)), ((2, 5), (4, 1)))
    return [[((300, 200), (150, 400)), ((640, 8), (1000, 8))] + [tiny[i % len(tiny)] for i in range(n - 2)]]


@pytest.mark.parametrize("ch, filt", RESIZE_MODES, ids=[f"{'L' if c == 1 else 'RGB'}-{f}" for c, f in RESIZE_MODES])
@pytest.mark.parametrize("cell", ["max", "mid", "1"])
def test_resize_regime(cell, ch, filt):
    sm = _sm()
    rng = np.random.default_rng(_seed("resize", cell, ch, filt))
    for batch in _resize_batch(cell, sm):
        srcs = [_content(rng, *s, ch) for s, _ in batch]
        outs = resize(srcs, [d for _, d in batch], ch, filt)
        for i, (a, (s, d)) in enumerate(zip(srcs, batch)):
            assert np.array_equal(outs[i], _pillow(a, d, ch, filt)), (cell, i, s, d)
        assert geo.resize_cell(len(batch), sm) == cell
        _record(f"resize-{cell}-{ch}-{filt}", "resize",
                geo.cells("resize", (len(batch), [geo.resize_passes(*s, *d) for s, d in batch]), sm))


@pytest.mark.parametrize("filt", ["bilinear", "bicubic"])
def test_resize_workspace_contract(filt):
    """at the queried size every image is written; one byte short, the last image keeps its sentinel, the others are
    right and the call still returns 0"""
    rng = np.random.default_rng(7)
    batch = [((37, 53), (64, 41)), ((57, 83), (57, 83)), ((40, 90), (40, 33)), ((90, 40), (29, 40))]
    for ch in (1, 3):
        srcs = [_content(rng, *s, ch) for s, _ in batch]
        want = [_pillow(a, d, ch, filt) for a, (_, d) in zip(srcs, batch)]
        for short in (0, 1):
            outs = resize(srcs, [d for _, d in batch], ch, filt, short=short)
            for i in range(len(batch)):
                if short and i == len(batch) - 1:
                    assert bool((outs[i] == SENTINEL).all()), "the image that does not fit was written"
                else:
                    assert np.array_equal(outs[i], want[i]), (short, i)
    _record(f"resize-ws-{filt}", "resize", {("workspace", "short")})


# ---- augmentation ---------------------------------------------------------------------------------------------------
ANGLES = (0.0, 1e-13, -1e-13, 10.0, -10.0, -0.1, -1e-9, 3.7)             # −0.1 and −1e-9 rotate by 359.9…°
ORDERS = tuple(itertools.permutations(range(3)))


def augment(img, mask, params):
    L = _lib()
    n, s = len(params), params.size
    io = torch.full_like(img, SENTINEL)
    mo = torch.full_like(mask, SENTINEL)
    ws_n = L.lib().sod_augment_u8_workspace_bytes(n)
    ws = torch.empty(ws_n, dtype=torch.uint8, device="cuda")
    rc = L.lib().sod_augment_u8(img.data_ptr(), mask.data_ptr(), io.data_ptr(), mo.data_ptr(), n, s, params.c_array(),
                                ws.data_ptr(), ws_n, L.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    return io.cpu().numpy(), mo.cpu().numpy()


def check_augment(img, mask, params, what):
    from test_gpu_train_disk import _pil_augment
    out, mout = augment(torch.from_numpy(img).cuda(), torch.from_numpy(mask).cuda(), params)
    for i in range(len(params)):
        wi, wm = _pil_augment(Image.fromarray(img[i], "RGB"), Image.fromarray(mask[i], "L"), params.flip[i], params.angle[i],
                              params.order[i], params.factor[i])
        assert np.array_equal(out[i], np.asarray(wi)), (what, i, params.angle[i], params.order[i])
        assert np.array_equal(mout[i], np.asarray(wm)), (what, i, params.angle[i])


def _params(n, s, seed, k0=0):
    from distributed_sod_project_b200.pipeline import draw_augment_params
    p = draw_augment_params(n, s, torch.Generator().manual_seed(seed))
    for i in range(n):
        p.angle[i] = ANGLES[(i + k0) % len(ANGLES)]
        p.order[i] = list(ORDERS[(i + k0) % len(ORDERS)])
        p.flip[i] = bool((i + k0) % 3 == 1)
    return p


@pytest.mark.parametrize("n, s", [(1, 32), (64, 32), (1, 33), (64, 33), (3, 1023), (2, 1024), (2, 1025), (1, 2048), (1, 4096)])
def test_augment_regime(n, s):
    from test_gpu_train_disk import _content as aug_content
    rng = np.random.default_rng(_seed("aug", n, s))
    img, mask = aug_content(rng, n, s)
    reps = 3 if n < 4 and s <= 1025 else 1
    for k in range(reps):
        check_augment(img, mask, _params(n, s, _seed("augp", n, s, k), k0=n * k), f"{n}x{s}")
    _record(f"aug-{n}-{s}", "augment", geo.cells("augment", (n, s), _sm()))


@pytest.mark.parametrize("s", [32, 1024, 2048])
def test_augment_contrast_mean_rounding(s):
    """grey images whose ΣL/S² is exactly k + ½ (int(mean + .5) rounds up) and exactly k, with contrast first"""
    from distributed_sod_project_b200.pipeline import draw_augment_params
    k = 100
    img = np.full((4, s, s, 3), k, np.uint8)
    img[0, : s // 2] = k + 1                                           # mean k + ½
    img[1, :, : s // 2] = k - 1
    img[1, :, s // 2:] = k + 2                                         # mean k + ½
    img[3, ::2] = k - 3
    img[3, 1::2] = k + 3                                               # mean k
    mask = np.zeros((4, s, s), np.uint8)
    p = draw_augment_params(4, s, torch.Generator().manual_seed(s))
    for i in range(4):
        p.angle[i], p.flip[i] = 0.0, bool(i % 2)
        p.order[i] = [1, 0, 2] if i < 3 else [1, 2, 0]
        p.factor[i] = [1.0, float(np.float32(1.1 if i != 1 else 0.9)), 1.0]
    assert [int(img[i, ..., 0].astype(np.int64).sum()) * 2 for i in range(2)] == [(2 * k + 1) * s * s] * 2
    check_augment(img, mask, p, f"contrast mean {s}")


# ---- every cell --------------------------------------------------------------------------------------------------------
def test_every_regime_cell_ran_on_this_device():
    """every cell of oracle.data_geometry.required, for every kernel, was reached by a passing case"""
    if not RAN:
        pytest.skip("the regime cases did not run in this session")
    sm = _sm()
    got = set().union(*RAN.values())
    required = {(k,) + c for k in geo.KERNELS for c in geo.required(k, sm)} | {("resize", "workspace", "short")}
    missing = required - got
    assert not missing, sorted(missing, key=str)
