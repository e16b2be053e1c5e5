"""The nearest ×2 kernels of csrc/nearest.cu (`sod_upsample2x_nearest_fwd` / `_bwd`, LightAIM's up-sampling) on the
GPU: the forward bit for bit against torch, the backward bit for bit against the fixed-order restatement of
tests/_nearest.py and, in 16 bit, within one rounding of the float64 sum; infinities, NaN, −0 and sums past the largest
finite value through the backward; reruns and CUDA-graph replay bit-identical; every refusal code.  Every launch regime
of both kernels is in tests/test_gpu_resample_regimes.py."""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

from _nearest import upsample2x_nearest_bwd, upsample2x_nearest_bwd64

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
SOD_EINVAL, SOD_EALIGN, SOD_EUNSUPPORTED = -1, -2, -4


@pytest.fixture(autouse=True)
def _enabled(monkeypatch):
    from distributed_sod_project_b200 import resample
    monkeypatch.setattr(resample, "ENABLED", True)


def _neck_shapes(s, n=2):
    """the twelve up-sample inputs of one aim_res50 forward at input side s, as (n, c, h, w)"""
    q = s // 4
    return ([(n, 64, q, q)] * 2 + [(n, 64, q, q), (n, 64, q // 2, q // 2), (n, 64, q // 2, q // 2)]
            + [(n, 64, q // 2, q // 2), (n, 64, q // 4, q // 4), (n, 64, q // 4, q // 4)]
            + [(n, 64, q // 4, q // 4), (n, 64, q // 8, q // 8), (n, 64, q // 8, q // 8)] + [(n, 1024, q // 8, q // 8)])


_GRID = [(n, c, h, w) for c in (8, 64, 1024) for (n, h, w) in ((1, 1, 1), (2, 4, 6), (3, 5, 7), (1, 9, 11), (2, 10, 3))]
SHAPES = sorted(set(_GRID + [sh for s in (64, 320, 352) for sh in _neck_shapes(s)]))


def _x(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, device="cuda", generator=g).to(dtype).contiguous(memory_format=torch.channels_last)


def _fwd_bwd(x, dy):
    from distributed_sod_project_b200 import resample
    xr = x.detach().requires_grad_(True)
    y = resample.upsample2x_nearest(xr)
    assert y is not None and y.dtype == x.dtype and y.is_contiguous(memory_format=torch.channels_last)
    (dx,) = torch.autograd.grad(y, xr, dy)
    return y.detach(), dx


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_nearest_matches_torch_and_the_fixed_order_oracle(shape, dtype):
    x = _x(shape, dtype, sum(shape))
    dy = _x((shape[0], shape[1], 2 * shape[2], 2 * shape[3]), dtype, sum(shape) + 1)
    y, dx = _fwd_bwd(x, dy)
    bits = torch.int32 if dtype == torch.float32 else torch.int16
    ref = F.interpolate(x.float(), scale_factor=2, mode="nearest").to(dtype)
    assert torch.equal(y.contiguous().view(bits), ref.contiguous().view(bits))
    oracle = upsample2x_nearest_bwd(dy.cpu()).cuda()
    assert torch.equal(dx.contiguous().view(bits), oracle.contiguous().view(bits))
    if dtype != torch.float32:
        exact = upsample2x_nearest_bwd64(dy)
        ulp = torch.finfo(dtype).eps * exact.abs().clamp_min(torch.finfo(dtype).tiny)
        assert bool(((dx.double() - exact).abs() <= ulp).all())


def _classes(t):
    """per element: 0 finite, 1 NaN, 2 +inf, 3 −inf"""
    return t.isnan().int() + 2 * t.isposinf().int() + 3 * t.isneginf().int()


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_backward_special_values(dtype):
    """±inf, NaN and −0 in dy; four taps of the largest finite value M (their sum overflows the dtype: in fp32 for fp32
    and bf16, in the final rounding for fp16, where 4M fits fp32), four of M/4 (exactly M), ±M alternating (exactly 0);
    in fp16 four taps summing to 65536 (past 65504: inf) and to 65512 (below the 65520 midpoint: 65504).  The backward
    equals the fixed-order oracle bit for bit (NaN by class) and torch's own nearest backward class for class (NaN,
    +inf, −inf, finite)."""
    n, c, h, w = 2, 16, 5, 6
    big = torch.finfo(dtype).max
    inf, nan = float("inf"), float("nan")
    dy = _x((n, c, 2 * h, 2 * w), torch.float32, 21)
    dy[0, 0, 0, 0] = inf                                   # one +inf tap, first window
    dy[0, 1, 0, 0], dy[0, 1, 1, 1] = inf, -inf             # +inf + −inf: NaN
    dy[0, 2, 2, 3] = nan
    dy[n - 1, 3, 2 * h - 1, 2 * w - 1] = -inf              # last window, last channel-group row
    dy[:, 4] = -0.0                                        # (((0 + −0) + −0) + −0) + −0 = +0
    dy[:, 5], dy[:, 5, 0::2, :] = 0.0, -0.0                 # −0 and +0 taps
    dy[:, 6] = big
    dy[:, 7] = big / 4
    dy[:, 8, :, 0::2], dy[:, 8, :, 1::2] = big, -big       # ((0 + M) − M) + M) − M, never past M
    if dtype == torch.float16:
        dy[:, 9] = 16384.0
        dy[:, 10] = 16376.0
        dy[:, 10, 1::2, 1::2] = 16384.0
    dy = dy.to(dtype).contiguous(memory_format=torch.channels_last)
    assert bool(dy[:, 4].signbit().all())
    x = torch.zeros((n, c, h, w), dtype=dtype, device="cuda").contiguous(memory_format=torch.channels_last)
    _, dx = _fwd_bwd(x, dy)
    oracle = upsample2x_nearest_bwd(dy.cpu()).cuda()
    bits = torch.int32 if dtype == torch.float32 else torch.int16
    got, want = dx.contiguous(), oracle.contiguous()
    nan_at = want.isnan()
    assert torch.equal(got.isnan(), nan_at)
    assert torch.equal(got.view(bits)[~nan_at], want.view(bits)[~nan_at])
    # the cases land where they should: NaN, ±inf, +0 and M
    assert bool(got[0, 1, 0, 0].isnan()) and bool(got[0, 2, 1, 1].isnan())
    assert float(got[0, 0, 0, 0]) == inf and float(got[n - 1, 3, h - 1, w - 1]) == -inf
    assert bool((got[:, 4:6] == 0).all()) and not bool(got[:, 4].signbit().any())
    assert bool(got[:, 6].isposinf().all()) and bool((got[:, 7] == big).all()) and bool((got[:, 8] == 0).all())
    if dtype == torch.float16:
        assert bool(got[:, 9].isposinf().all()) and bool((got[:, 10] == 65504.0).all())
    xr = x.detach().requires_grad_(True)
    (ref,) = torch.autograd.grad(F.interpolate(xr, scale_factor=2, mode="nearest"), xr, dy)
    assert torch.equal(_classes(got), _classes(ref))


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_reruns_and_graph_replay_are_bit_identical(dtype):
    from distributed_sod_project_b200 import resample
    x = _x((4, 64, 40, 40), dtype, 3)
    dy = _x((4, 64, 80, 80), dtype, 4)
    y0, dx0 = _fwd_bwd(x, dy)
    for _ in range(3):
        y1, dx1 = _fwd_bwd(x, dy)
        assert torch.equal(y1, y0) and torch.equal(dx1, dx0)
    sx, sdy = x.clone(), dy.clone()
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _fwd_bwd(sx, sdy)
    torch.cuda.current_stream().wait_stream(side)
    with torch.cuda.graph(g):
        xr = sx.detach().requires_grad_(True)
        gy = resample.upsample2x_nearest(xr)
        (gdx,) = torch.autograd.grad(gy, xr, sdy)
    sx.copy_(_x(sx.shape, dtype, 9))
    sdy.copy_(_x(sdy.shape, dtype, 10))
    g.replay()
    sx.copy_(x)
    sdy.copy_(dy)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(gy, y0) and torch.equal(gdx, dx0)


@pytest.mark.parametrize("entry", ["sod_upsample2x_nearest_fwd", "sod_upsample2x_nearest_bwd"])
def test_refusal_codes(entry):
    """null pointers, non-positive sizes and an unknown dtype → SOD_EINVAL, a misaligned pointer → SOD_EALIGN, C % 8 != 0
    → SOD_EUNSUPPORTED; a refused call writes nothing"""
    from distributed_sod_project_b200 import _lib
    lib, s = _lib.lib(), _lib.stream_ptr()
    a = torch.ones(4096, dtype=torch.float32, device="cuda")
    b = torch.full((4096,), 7.0, dtype=torch.float32, device="cuda")
    f = getattr(lib, entry)
    fp32 = _lib.dtype_code(torch.float32)
    refused = [((None, b.data_ptr(), 1, 2, 2, 8, fp32), SOD_EINVAL), ((a.data_ptr(), None, 1, 2, 2, 8, fp32), SOD_EINVAL),
               ((a.data_ptr(), b.data_ptr(), 1, 2, 2, 8, 99), SOD_EINVAL),
               ((a.data_ptr() + 4, b.data_ptr(), 1, 2, 2, 8, fp32), SOD_EALIGN),
               ((a.data_ptr(), b.data_ptr() + 8, 1, 2, 2, 8, fp32), SOD_EALIGN),
               ((a.data_ptr(), b.data_ptr(), 1, 2, 2, 12, fp32), SOD_EUNSUPPORTED),
               ((a.data_ptr(), b.data_ptr(), 1, 2, 2, 4, fp32), SOD_EUNSUPPORTED)]
    refused += [((a.data_ptr(), b.data_ptr(), *dims, fp32), SOD_EINVAL)
                for dims in ((0, 2, 2, 8), (1, 0, 2, 8), (1, 2, -1, 8), (1, 2, 2, 0), (-1, 2, 2, 8))]
    for args, code in refused:
        assert f(*args, s) == code, (args, code)
    torch.cuda.synchronize()
    assert bool((b == 7.0).all())
    assert f(a.data_ptr(), b.data_ptr(), 1, 2, 2, 8, fp32, s) == 0
    torch.cuda.synchronize()
    assert bool((b[:32] == (1.0 if entry.endswith("fwd") else 4.0)).all())


def test_seam_falls_back_exactly_where_the_kernels_do_not_cover():
    """`blocks.nearest2x` runs the kernel when `resample._ok` holds and F.interpolate otherwise (C % 8 != 0, fp64, CPU),
    with the same values"""
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.network.blocks import nearest2x
    calls = []
    orig = resample._UpNearest2x.forward

    def fwd(ctx, x):
        calls.append(tuple(x.shape))
        return orig(ctx, x)

    resample._UpNearest2x.forward = staticmethod(fwd)
    try:
        for x, covered in ((_x((2, 16, 3, 5), torch.float32, 1), True), (_x((2, 12, 3, 5), torch.float32, 2), False),
                           (_x((2, 16, 3, 5), torch.float32, 3).double(), False), (torch.randn(1, 8, 2, 2), False)):
            n0 = len(calls)
            y = nearest2x(x)
            assert (len(calls) > n0) == covered == resample._ok(x)
            assert torch.equal(y, F.interpolate(x, scale_factor=2, mode="nearest"))
    finally:
        resample._UpNearest2x.forward = staticmethod(orig)
