"""The 32-group 3×3 convolution kernels (csrc/gconv.cu) against float64 `conv2d(groups=32)` and its gradients.

Error bound, per element, against float64 on the same (already rounded) inputs:
    |out − out64| ≤ 2^-p·|out64|  +  2·(K + 1)·u·Σ|a·b|
* 2^-p: one rounding of the output to its dtype (p = 24 fp32, 8 bf16, 11 fp16; dŴ is fp32 in every dtype);
* u = 2^-24, K = the reduction length (9·cpg for fwd and dgrad, N·Ho·Wo for wgrad) and Σ|a·b| = the same convolution
  on |x|, |Ŵ|, |dy|: a sum of K fp32 terms is off by at most K·u·Σ|terms|, the products are exact in fp32 for 16-bit
  inputs (8 + 8 and 11 + 11 significand bits) and off by u for fp32 inputs (the +1).  The factor 2 allows the tensor
  cores' accumulation, which truncates instead of rounding to nearest (at most 2u per addition).
The float64 reference runs on the GPU (cuDNN in double precision), so the capped-split shapes stay affordable.
"""
from __future__ import annotations

import pytest
import torch
import torch.nn.functional as F

from oracle import gconv_geometry as geo

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
P = {torch.float32: 24, torch.bfloat16: 8, torch.float16: 11}
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
CL = torch.channels_last

# (cpg, stride, side of the input at a 1×1 image) of the sixteen convolutions, per distinct shape
MODEL = ((4, 1, 4), (8, 2, 4), (8, 1, 8), (16, 2, 8), (16, 1, 16), (32, 2, 16), (32, 1, 32))


def _lib():
    from distributed_sod_project_b200 import _lib
    return _lib


def _tensors(n, h, w, cpg, stride, dtype, seed):
    c = 32 * cpg
    g = torch.Generator(device="cuda").manual_seed(seed)
    ho, wo = geo.out_size(h, stride), geo.out_size(w, stride)
    x = torch.randn(n, c, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL)
    wh = (torch.randn(c, cpg, 3, 3, device="cuda", generator=g) / (3 * cpg ** 0.5)).to(dtype).contiguous(memory_format=CL)
    dy = torch.randn(n, c, ho, wo, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL)
    return x, wh, dy


def run_kernels(x, wh, dy, stride):
    """(y, dx, dŴ) of the three C entries"""
    L = _lib()
    lib, code, G, st = L.lib(), L.dtype_code(x.dtype), L.SOD_GCONV_GROUPS, L.stream_ptr()
    n, c, h, w = x.shape
    y, dx = torch.empty_like(dy), torch.empty_like(x)
    dw = torch.empty(wh.shape, dtype=torch.float32, device="cuda", memory_format=CL)
    ws = torch.zeros(int(lib.sod_gconv3x3_wgrad_workspace_bytes(n, h, w, c, G, stride)), dtype=torch.uint8,
                     device="cuda")
    L.check(lib.sod_gconv3x3_fwd(x.data_ptr(), wh.data_ptr(), y.data_ptr(), code, n, h, w, c, G, stride, st))
    L.check(lib.sod_gconv3x3_dgrad(dy.data_ptr(), wh.data_ptr(), dx.data_ptr(), code, n, h, w, c, G, stride, st))
    L.check(lib.sod_gconv3x3_wgrad(x.data_ptr(), dy.data_ptr(), dw.data_ptr(), code, n, h, w, c, G, stride,
                                   ws.data_ptr(), ws.numel(), st))
    torch.cuda.synchronize()
    return y, dx, dw


def references(x, wh, dy, stride):
    """float64 (y, dx, dŴ) and the same maps on magnitudes"""
    out = []
    for f in (lambda t: t.double(), lambda t: t.double().abs()):
        x64, w64, d64 = f(x), f(wh), f(dy)
        out.append((F.conv2d(x64, w64, None, stride, 1, 1, 32),
                    torch.nn.grad.conv2d_input(x.shape, w64, d64, stride, 1, 1, 32),
                    torch.nn.grad.conv2d_weight(x64, wh.shape, d64, stride, 1, 1, 32)))
    return out


def check(n, h, w, cpg, stride, dtype, seed=0):
    x, wh, dy = _tensors(n, h, w, cpg, stride, dtype, seed)
    got = run_kernels(x, wh, dy, stride)
    (ref, mag) = references(x, wh, dy, stride)
    k_len = (9 * cpg, 9 * cpg, dy.shape[0] * dy.shape[2] * dy.shape[3])
    prec = (P[dtype], P[dtype], 24)
    for name, g, r, m, k, p in zip(("y", "dx", "dw"), got, ref, mag, k_len, prec):
        assert g.is_contiguous(memory_format=CL)
        err = (g.double() - r).abs()
        bound = 2.0 ** -p * r.abs() + 2 * (k + 1) * U * m
        worst = (err - bound).max().item()
        assert worst <= 0, f"{name}: {n}x{h}x{w} cpg {cpg} stride {stride} {dtype}: error exceeds its bound by {worst}"
    return got


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("cpg", geo.CPG)
def test_every_regime(cpg, stride, dtype):
    """every (wgrad split, last chunk, last m-tile, last CTA) cell of oracle/gconv_geometry.py, with 1×1 and 2×2 maps,
    odd and non-square sizes"""
    for n, h, w, c, s, _ in geo.regime_cases():
        if (c, s) == (cpg, stride):
            check(n, h, w, cpg, stride, dtype, seed=n + h + w)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("size", [64, 320, 352])
def test_model_shapes(size, dtype):
    """the sixteen convolutions' shapes at 64² (down to 2×2 maps), the 320² bench size and 352² (11², 22² maps)"""
    for cpg, stride, k in MODEL:
        side = size // k
        check(2, side, side, cpg, stride, dtype, seed=size + cpg + stride)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=str)
def test_bench_batch_layer1(dtype):
    """N = 16 at the bench size: wgrad reduces 102 400 pixels in the capped split"""
    check(16, 80, 80, 4, 1, dtype)


def test_n1_maps():
    for cpg in geo.CPG:
        for side in (1, 2, 3):
            for stride in (1, 2):
                check(1, side, side, cpg, stride, torch.bfloat16)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_second_call_is_bit_identical(dtype):
    x, wh, dy = _tensors(4, 40, 40, 8, 1, dtype, 3)
    a, b = run_kernels(x, wh, dy, 1), run_kernels(x, wh, dy, 1)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_refusals_launch_nothing():
    L = _lib()
    lib, G, st = L.lib(), L.SOD_GCONV_GROUPS, L.stream_ptr()
    x, wh, dy = _tensors(1, 8, 8, 8, 1, torch.bfloat16, 4)
    y = torch.full_like(dy, 7.0)
    dw = torch.full(wh.shape, 7.0, device="cuda")
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    bf = L.SOD_BF16
    fwd = lambda xp, wp, yp, dt, n, c, g, s: lib.sod_gconv3x3_fwd(xp, wp, yp, dt, n, 8, 8, c, g, s, st)  # noqa: E731
    xp, wp, yp = x.data_ptr(), wh.data_ptr(), y.data_ptr()
    assert fwd(None, wp, yp, bf, 1, 256, G, 1) == -1
    assert fwd(xp, wp, yp, 7, 1, 256, G, 1) == -1
    assert fwd(xp, wp, yp, bf, 0, 256, G, 1) == -1
    assert fwd(xp, wp, yp, bf, 1, 250, G, 1) == -1                # C not a multiple of the groups
    assert fwd(xp, wp, yp, bf, 1, 256, 16, 1) == -4                # 16 groups
    assert fwd(xp, wp, yp, bf, 1, 64, G, 1) == -4                  # 2 channels per group
    assert fwd(xp, wp, yp, bf, 1, 2048, G, 1) == -4                # 64 channels per group
    assert fwd(xp, wp, yp, bf, 1, 256, G, 3) == -4
    assert fwd(xp + 2, wp, yp, bf, 1, 256, G, 1) == -2
    assert lib.sod_gconv3x3_dgrad(dy.data_ptr(), wp + 2, yp, bf, 1, 8, 8, 256, G, 1, st) == -2
    assert lib.sod_gconv3x3_wgrad(xp, dy.data_ptr(), dw.data_ptr(), bf, 1, 8, 8, 256, G, 1, ws.data_ptr(), 16, st) == -3
    assert lib.sod_gconv3x3_wgrad(xp, dy.data_ptr(), dw.data_ptr(), bf, 1, 8, 8, 256, G, 1, None, ws.numel(), st) == -1
    assert lib.sod_gconv3x3_wgrad_workspace_bytes(1, 8, 8, 256, 16, 1) == 0
    torch.cuda.synchronize()
    assert bool((y == 7).all()) and bool((dw == 7).all()) and bool((ws == 0).all())


@pytest.mark.parametrize("channels_last", [True, False])
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_seam_gradients_reach_the_master_weight(dtype, channels_last):
    """FusedWSConv2d on a grouped convolution: y, dx and the fp32 master weight's gradient against float64 autograd of
    the reference's WS expression and conv2d — dŴ leaves the wgrad kernel in the order sod_ws_bwd reads, with a
    channels-last master and with an NCHW one (Trainer(channels_last=False))"""
    from distributed_sod_project_b200.network.blocks import WSConv2d
    from distributed_sod_project_b200.wsgn import FusedWSConv2d
    torch.manual_seed(5)
    ref = WSConv2d(256, 256, 3, 2, 1, groups=32, bias=False).cuda()
    mod = FusedWSConv2d(256, 256, 3, 2, 1, groups=32, bias=False).cuda()
    mod.weight = torch.nn.Parameter(ref.weight.detach().clone())
    if channels_last:
        mod = mod.to(memory_format=CL)
    x = torch.randn(2, 256, 13, 12, device="cuda").to(dtype)
    xin = (x.contiguous(memory_format=CL) if channels_last else x.clone()).requires_grad_(True)
    with torch.autocast("cuda", dtype=dtype, enabled=dtype != torch.float32):
        y = mod(xin)
    assert y.dtype == dtype
    dy = torch.randn(y.shape, device="cuda").to(dtype)
    y.backward(dy)
    w64 = ref.weight.detach().double().requires_grad_(True)
    x64 = x.double().requires_grad_(True)
    y64 = F.conv2d(x64, WSConv2d.standardized_weight(type("P", (), {"weight": w64, "eps": 1e-5})()), None, 2, 1, 1, 32)
    y64.backward(dy.double())
    tol = {torch.float32: 1e-5, torch.bfloat16: 3e-2, torch.float16: 4e-3}[dtype]
    for got, want in ((y, y64), (xin.grad, x64.grad), (mod.weight.grad, w64.grad)):
        scale = want.abs().max().item()
        assert (got.double() - want).abs().max().item() <= tol * scale
    assert mod.weight.grad.dtype == torch.float32


def test_seam_refuses_uncovered_grouped_geometry():
    from distributed_sod_project_b200 import _lib as L
    from distributed_sod_project_b200.wsgn import FusedWSConv2d
    x = torch.randn(1, 64, 8, 8, device="cuda")
    for kw in (dict(groups=16), dict(groups=32, dilation=2, padding=2), dict(groups=32, bias=True)):
        m = FusedWSConv2d(64, 64, 3, 1, kw.pop("padding", 1), **kw).cuda()
        with pytest.raises(L.SodError):
            m(x)
