"""`sod_maxpool2x2s2_fwd` / `_bwd` (csrc/maxpool.cu, VGG16-BN's MaxPool2d(2, 2)) bit for bit against torch.

The forward's values and window positions must equal `F.max_pool2d(x, 2, 2, return_indices=True)` (its flat input
indices converted to kh·2 + kw, or to 4 where torch's index lies outside the window: a window with nothing above −inf
other than the first keeps torch's initial index, the plane's first element), and the backward must equal torch's autograd backward bit for bit, −0 gradients
included (torch copies dy into a zeroed dx where windows do not overlap, so a −0 dy stays −0).  Covered: every wave regime of the
grid-stride loops on this GPU (one packet, a partial wave below the 16·#SMs cap, exactly the cap, two passes and a
ragged tail), fp32 / bf16 / fp16, C ∈ {8, 64, 128, 256, 512}, even and odd H and W down to 2 and 3 (floor mode drops
the last row / column; their dx must be 0), the four pools of VGG16-BN at bs 16 and 256², 320², 384², and special
values: zero ties (after a ReLU), windows of −inf, a NaN at each window position, ±inf.  Refused calls leave their
outputs untouched, and a rerun gives the same bits.
"""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

from oracle import resample_geometry as geo

pytestmark = pytest.mark.gpu

DTYPES = (torch.float32, torch.bfloat16, torch.float16)
INT_VIEW = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}
SOD_EINVAL, SOD_EALIGN, SOD_EUNSUPPORTED = -1, -2, -4


def _lib():
    from distributed_sod_project_b200 import _lib
    return _lib


def _sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _bits(t):
    return t.contiguous().view(INT_VIEW[t.dtype])


def _kernel_fwd(x):
    n, c, h, w = x.shape
    y = torch.empty((n, c, h // 2, w // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    arg = torch.empty(y.numel(), dtype=torch.uint8, device=x.device)
    rc = _lib().lib().sod_maxpool2x2s2_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), n, h, w, c, _lib().dtype_code(x.dtype),
                                           _lib().stream_ptr())
    assert rc == 0, rc
    return y, arg.view(n, h // 2, w // 2, c).permute(0, 3, 1, 2)


def _kernel_bwd(dy, arg, h, w):
    n, c = dy.shape[:2]
    dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
    rows = arg.permute(0, 2, 3, 1).contiguous()                       # [n, ho, wo, c], the kernel's layout
    rc = _lib().lib().sod_maxpool2x2s2_bwd(dy.data_ptr(), rows.data_ptr(), dx.data_ptr(), n, h, w, c,
                                           _lib().dtype_code(dy.dtype), _lib().stream_ptr())
    assert rc == 0, rc
    return dx


def _torch(x, dy):
    """torch's forward (values, window positions) and autograd backward on the same channels-last tensors"""
    xr = x.detach().clone().requires_grad_(True)
    y, idx = F.max_pool2d(xr, 2, 2, return_indices=True)
    y.backward(dy)
    w = x.shape[3]
    ho, wo = y.shape[2:]
    oh = torch.arange(ho, device=x.device).view(1, 1, ho, 1)
    ow = torch.arange(wo, device=x.device).view(1, 1, 1, wo)
    kh, kw = idx // w - 2 * oh, idx % w - 2 * ow
    inside = (kh >= 0) & (kh < 2) & (kw >= 0) & (kw < 2)        # torch's index of an all −inf window is the plane's first
    pos = torch.where(inside, kh * 2 + kw, 4)
    return y.detach(), pos.to(torch.uint8), xr.grad


def _dy(shape, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn(shape, generator=g, device="cuda").to(dtype)
    dy[..., ::5, ::3] = -0.0                                         # −0 gradients stay −0 in torch's backward
    return dy.contiguous(memory_format=torch.channels_last)


def _check(x, seed=0):
    n, c, h, w = x.shape
    dy = _dy((n, c, h // 2, w // 2), x.dtype, seed)
    y, arg = _kernel_fwd(x)
    ry, rpos, rdx = _torch(x, dy)
    assert torch.equal(_bits(y), _bits(ry)), "forward values"
    assert torch.equal(arg, rpos), "window positions"
    dx = _kernel_bwd(dy, arg, h, w)
    bad = (_bits(dx) != _bits(rdx)).nonzero()
    assert not len(bad), f"backward: {len(bad)} elements differ, first {bad[0].tolist()}: " \
                         f"{dx[tuple(bad[0])].item()!r} vs torch {rdx[tuple(bad[0])].item()!r}"
    if h % 2 or w % 2:
        assert not _bits(dx)[:, :, 2 * (h // 2):, :].any() and not _bits(dx)[:, :, :, 2 * (w // 2):].any()
    return y, arg, dx


def _randn(shape, dtype, seed, relu=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, generator=g, device="cuda")
    if relu:
        x = x.clamp_min(0)
    return x.to(dtype).contiguous(memory_format=torch.channels_last)


# -- wave regimes ------------------------------------------------------------------------------------------------------
def _regime_shapes():
    """(name, shape) with C = 8; the forward writes n·⌊h/2⌋·⌊w/2⌋ packets, the backward n·h·w"""
    sm = _sm()
    return [("one packet", (1, 8, 2, 2)), ("one packet odd", (1, 8, 3, 3)), ("below cap", (3, 8, 37, 45)),
            ("fwd at cap", (sm, 8, 128, 129)), ("bwd at cap", (sm, 8, 64, 64)), ("fwd cap + tail", (sm + 1, 8, 128, 128)),
            ("two passes + tail", (2 * sm + 1, 8, 129, 128))]


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_every_wave_regime(dtype):
    sm = _sm()
    fwd, bwd = set(), set()
    for i, (name, shape) in enumerate(_regime_shapes()):
        n, c, h, w = shape
        fwd.add(geo.classify(n * (h // 2) * (w // 2) * (c // 8), sm))
        bwd.add(geo.classify(n * h * w * (c // 8), sm))
        _check(_randn(shape, dtype, i), seed=i)
    assert {"partial", "1", "1+ragged", ">=2 ragged"} <= fwd and {"partial", "1", ">=2 ragged"} <= bwd, (fwd, bwd)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("c", [8, 64, 128, 256, 512])
def test_channels_and_odd_sizes(dtype, c):
    for i, (h, w) in enumerate([(2, 2), (3, 3), (2, 3), (3, 2), (4, 6), (5, 7), (16, 17), (31, 30)]):
        _check(_randn((2, c, h, w), dtype, 100 * c + i, relu=i % 2 == 0), seed=i)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("size", [256, 320, 384])
def test_vgg16_pool_shapes(dtype, size):
    """the inputs of the four pools of VGG16-BN at bs 16 (after a ReLU: many zero ties)"""
    for i, (c, s) in enumerate([(64, size), (128, size // 2), (256, size // 4), (512, size // 8)]):
        _check(_randn((16, c, s, s), dtype, size + i, relu=True), seed=i)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_special_values(dtype):
    """zero ties in every window, all −inf windows, NaN at each of the four positions (alone and two NaNs), ±inf"""
    n, c, h, w = 2, 16, 6, 8
    x = torch.zeros((n, c, h, w), device="cuda")
    x[0, 1] = float("-inf")
    x[0, 2, 2:4, 2:4] = float("-inf")
    for k in range(4):
        x[1, k, k // 2, 2 + k % 2] = float("nan")                  # NaN at window position k, rest 0
        x[1, 4 + k, 2 + k // 2, 4 + k % 2] = float("nan")
        x[1, 4 + k, 2 + (k + 1) % 4 // 2, 4 + (k + 1) % 4 % 2] = float("nan")   # two NaNs: the later one wins
    x[0, 3, 0, 0], x[0, 3, 1, 1] = float("inf"), float("inf")
    x[0, 4] = float("-inf")
    x[0, 4, 1, 1] = float("inf")
    x[0, 5, ::2, ::2] = -1.0
    x[0, 6] = torch.arange(h * w, device="cuda").view(h, w) % 3 - 1.0      # ties of 1s and 0s
    x = x.to(dtype).contiguous(memory_format=torch.channels_last)
    y, arg, _ = _check(x, seed=7)
    assert bool(torch.isnan(y[1, :8]).any()) and bool((y[0, 1] == float("-inf")).all())
    assert int(arg[0, 1, 0, 0]) == 0 and bool((arg[0, 1].flatten()[1:] == 4).all()) and int(arg[0, 2, 1, 1]) == 4


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_refusals_leave_outputs_untouched_and_reruns_are_identical(dtype):
    lib, code = _lib().lib(), _lib().dtype_code(dtype)
    x = _randn((2, 16, 8, 8), dtype, 3)
    y = torch.full((2 * 16 * 16 + 8,), 7.0, device="cuda").to(dtype)
    arg = torch.full((2 * 16 * 16 + 16,), 0xAB, dtype=torch.uint8, device="cuda")
    dx = torch.full((2 * 16 * 64 + 8,), 5.0, device="cuda").to(dtype)
    ys, argc, dxs = y.clone(), arg.clone(), dx.clone()
    es = y.element_size()
    cases = [
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr(), None, 2, 8, 8, 16), SOD_EINVAL),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr() + es, y.data_ptr(), arg.data_ptr(), 2, 8, 8, 16), SOD_EALIGN),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr() + es, arg.data_ptr(), 2, 8, 8, 16), SOD_EALIGN),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr(), arg.data_ptr() + 8, 2, 8, 8, 16), SOD_EALIGN),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr(), arg.data_ptr(), 2, 1, 8, 16), SOD_EUNSUPPORTED),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr(), arg.data_ptr(), 2, 8, 1, 16), SOD_EUNSUPPORTED),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr(), arg.data_ptr(), 2, 8, 8, 12), SOD_EUNSUPPORTED),
        (lib.sod_maxpool2x2s2_fwd, (x.data_ptr(), y.data_ptr(), arg.data_ptr(), 0, 8, 8, 16), SOD_EINVAL),
        (lib.sod_maxpool2x2s2_bwd, (y.data_ptr(), arg.data_ptr(), dx.data_ptr() + es, 2, 8, 8, 16), SOD_EALIGN),
        (lib.sod_maxpool2x2s2_bwd, (y.data_ptr(), arg.data_ptr(), dx.data_ptr(), 2, 8, 1, 16), SOD_EUNSUPPORTED),
        (lib.sod_maxpool2x2s2_bwd, (y.data_ptr(), arg.data_ptr(), dx.data_ptr(), 2, 8, 8, 20), SOD_EUNSUPPORTED),
        (lib.sod_maxpool2x2s2_bwd, (y.data_ptr(), None, dx.data_ptr(), 2, 8, 8, 16), SOD_EINVAL),
    ]
    for fn, args, want in cases:
        assert fn(*args, code, _lib().stream_ptr()) == want, (fn, args)
    assert lib.sod_maxpool2x2s2_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), 2, 8, 8, 16, 9, None) == SOD_EINVAL
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(ys)) and torch.equal(arg, argc) and torch.equal(_bits(dx), _bits(dxs))
    a = _check(x, seed=1)
    b = _check(x, seed=1)
    assert all(torch.equal(_bits(u) if u.is_floating_point() else u, _bits(v) if v.is_floating_point() else v)
               for u, v in zip(a, b))


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_seam_autograd_matches_torch(dtype):
    """`resample.maxpool2x2s2` (what `_VGGPool` calls) against nn.MaxPool2d(2, 2) through autograd, and None outside the
    kernel's cover (CPU, C % 8, H or W < 2, switched off); a `_VGGPool` asked for indices keeps torch's op"""
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.network.blocks import _VGGPool
    old = resample.ENABLED, resample.MAXPOOL_ENABLED
    resample.ENABLED = resample.MAXPOOL_ENABLED = True
    try:
        x = _randn((4, 64, 33, 40), dtype, 11, relu=True)
        dy = _dy((4, 64, 16, 20), dtype, 12)
        a = x.clone().requires_grad_(True)
        y = _VGGPool(2, 2)(a)
        assert y.grad_fn is not None and type(y.grad_fn).__name__ == "_MaxPool2x2s2Backward"
        y.backward(dy)
        ry, _, rdx = _torch(x, dy)
        assert torch.equal(_bits(y.detach()), _bits(ry)) and torch.equal(_bits(a.grad), _bits(rdx))
        assert y.is_contiguous(memory_format=torch.channels_last)
        assert resample.maxpool2x2s2(x.cpu()) is None
        assert resample.maxpool2x2s2(_randn((1, 12, 8, 8), dtype, 1)) is None
        assert resample.maxpool2x2s2(_randn((1, 8, 1, 8), dtype, 1)) is None
        ty, tidx = F.max_pool2d(x, 2, 2, return_indices=True)      # return_indices: torch's op and its tuple
        got = _VGGPool(2, 2, return_indices=True)(x)
        assert isinstance(got, tuple) and torch.equal(got[1], tidx) and torch.equal(_bits(got[0]), _bits(ty))
        resample.MAXPOOL_ENABLED = False
        assert resample.maxpool2x2s2(x) is None
    finally:
        resample.ENABLED, resample.MAXPOOL_ENABLED = old
