"""GroupNorm(32) and weight-standardisation kernels (csrc/wsgn.cu) against the fp64 oracle (oracle/wsgn.py).

Error bound (GroupNorm), per element, against float64 on the same (rounded) inputs:
    |out − out64| ≤ 2^-p·|out64|  +  8·D·u·scale
* 2^-p: one rounding of the output dtype (p = 24 fp32, 8 bf16, 11 fp16);
* u = 2^-24 and D = the longest chain of fp32 additions the value went through in the reduction tree of
  oracle/wsgn_geometry.py: rows per thread (rc / R) + row phases R + channels per group + CTAs per sample S (+ N for
  dγ/dβ) — every fp32 sum of D terms is off by at most D·u times the sum of the magnitudes;
* scale: the magnitude the sums carried — forward |γ|·(1 + |x̂| + |μ|·rstd) + |β| + |residual| (the |μ|·rstd term is the
  large-mean case: the shifted sums lose |μ|·u per term); dx: rstd·(|γ·dz| + mean|γ·dz| + |x̂|·mean|γ·dz·x̂|)·(1 + |μ|·rstd);
  dγ: Σ|dz|·(1 + |x̂|)·(1 + |μ|·rstd) (x̂ carries the statistics' error), dβ: Σ|dz|, over the batch.
Weight standardisation: Ŵ within one output rounding plus 8·(K/256 + 16)·u·(1 + |ŵ|); dW within 8·(K/256 + 16)·u times
the magnitude of its three terms, |g|/s + mean|g|/s + |v|·Σ|g·v|/(s²·(K−1)·σ).
"""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from oracle import wsgn as ow
from oracle import wsgn_geometry as geo

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
P = {torch.float32: 24, torch.bfloat16: 8, torch.float16: 11}
DTYPES = [torch.float32, torch.bfloat16, torch.float16]
EPILOGUES = [(False, False), (True, False), (True, True), (False, True)]


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(n, c, h, w, dtype, mean=0.0, std=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, c, h, w, generator=g, dtype=torch.float64) * std + mean).to(dtype)
    gamma = (torch.rand(c, generator=g) + 0.5)
    beta = torch.randn(c, generator=g) * 0.5
    res = torch.randn(n, c, h, w, generator=g, dtype=torch.float64).to(dtype)
    dy = torch.randn(n, c, h, w, generator=g, dtype=torch.float64).to(dtype)
    return x, gamma, beta, res, dy


def _cl(t):
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _depth(n, h, w, c, sms, batch=False):
    gm = geo.make_geom(n, h * w, c, sms)
    return (gm.rc + gm.R - 1) // gm.R + gm.R + c // 32 + gm.S + (n if batch else 0) + 8


def run_gn(x, gamma, beta, res, dy, relu):
    """forward + backward through the module seam; returns numpy fp64 of (y, dx, dres, dγ, dβ)"""
    from distributed_sod_project_b200 import wsgn
    xc = _cl(x).requires_grad_(True)
    rc = _cl(res).requires_grad_(True) if res is not None else None
    gm = gamma.cuda().requires_grad_(True)
    bt = beta.cuda().requires_grad_(True)
    y = wsgn.group_norm(xc, gm, bt, 1e-5, residual=rc, relu=relu)
    y.backward(_cl(dy))
    f = lambda t: None if t is None else t.detach().double().cpu().numpy()  # noqa: E731
    return f(y), f(xc.grad), f(rc.grad) if rc is not None else None, f(gm.grad), f(bt.grad)


def check_gn(n, c, h, w, dtype, relu, with_res, sms, mean=0.0, std=1.0, outlier=0.0):
    x, gamma, beta, res, dy = _inputs(n, c, h, w, dtype, mean, std, seed=n * 7 + c + h)
    if outlier:
        x[:, :, 0, 0] = (x[:, :, 0, 0].double() + outlier).to(dtype)     # the first row of every sample
    res = res if with_res else None
    y, dx, dres, dg, db = run_gn(x, gamma, beta, res, dy, relu)
    x64, g64, b64 = x.double().numpy(), gamma.double().numpy(), beta.double().numpy()
    r64 = None if res is None else res.double().numpy()
    o = ow.group_norm_forward(x64, g64, b64, r64, relu)
    p = 2.0 ** -P[dtype]
    D = _depth(n, h, w, c, sms)
    mu = np.repeat(o["mean"], c // 32, axis=1)[:, :, None, None]
    rs = np.repeat(o["rstd"], c // 32, axis=1)[:, :, None, None]
    big = 1.0 + np.abs(mu) * rs
    gg, bb = np.abs(g64)[None, :, None, None], np.abs(b64)[None, :, None, None]
    scale = gg * (1 + np.abs(o["xhat"])) * big + bb + (0 if r64 is None else np.abs(r64))
    err = np.abs(y - o["y"])
    bound = p * np.abs(o["y"]) + 8 * D * U * scale
    assert (err <= bound).all(), f"y: worst {np.max(err / bound):.2f}x the bound"
    # backward against the oracle with the kernel's own ReLU mask (a |y| below one rounding may fall either side of 0)
    dz = dy.double().numpy() * ((y > 0) if relu else 1.0)
    b = ow.group_norm_backward(dz, x64, g64, b64, None, False)
    gdz = np.abs(dz * g64[None, :, None, None])
    m1 = np.repeat(gdz.reshape(n, 32, -1).mean(axis=2), c // 32, axis=1)[:, :, None, None]
    m2 = np.repeat((gdz * np.abs(o["xhat"])).reshape(n, 32, -1).mean(axis=2), c // 32, axis=1)[:, :, None, None]
    dscale = rs * (gdz + m1 + np.abs(o["xhat"]) * m2) * big
    err = np.abs(dx - b["dx"])
    bound = p * np.abs(b["dx"]) + 8 * D * U * dscale
    assert (err <= bound).all(), f"dx: worst {np.max(err / bound):.2f}x the bound"
    if with_res:
        np.testing.assert_array_equal(dres, dz)
    Db = _depth(n, h, w, c, sms, batch=True)
    for got, want, mag in ((dg, b["dgamma"], (np.abs(dz) * (1 + np.abs(o["xhat"])) * big).sum(axis=(0, 2, 3))),
                           (db, b["dbeta"], np.abs(dz).sum(axis=(0, 2, 3)))):
        assert (np.abs(got - want) <= U * np.abs(want) + 8 * Db * U * mag).all()


def test_every_launch_regime(sms):
    """the regime cells of the geometry model on this SM count, every dtype, every epilogue"""
    cases = geo.regime_cases(sms)
    assert len({c[-1] for c in cases}) >= 8
    for n, h, w, c, cell in cases:
        assert torch.cuda.is_available()
        from distributed_sod_project_b200 import _lib
        assert _lib.lib().sod_groupnorm_splits(n, h * w, c, 32) == geo.make_geom(n, h * w, c, sms).S, cell
        for dtype in DTYPES:
            for relu, res in EPILOGUES:
                check_gn(n, c, h, w, dtype, relu, res, sms)


# the backbone's GroupNorm layers at the smallest and largest inputs and batch sizes: C 64 … 2048, N 1 … 16, 64² … 384²
MODEL_SHAPES = [(16, 64, 32, 32), (16, 256, 16, 16), (16, 512, 8, 8), (16, 1024, 4, 4), (16, 2048, 2, 2),
                (1, 64, 192, 192), (1, 128, 96, 96), (1, 256, 96, 96), (1, 512, 48, 48), (1, 1024, 24, 24),
                (1, 2048, 12, 12), (4, 64, 80, 80)]


@pytest.mark.parametrize("shape", MODEL_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_model_shapes(shape, dtype, sms):
    n, c, h, w = shape
    for relu, res in EPILOGUES[:3]:
        check_gn(n, c, h, w, dtype, relu, res, sms)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("shape", [(2, 64, 40, 40), (4, 2048, 3, 3)], ids=lambda s: "x".join(map(str, s)))
def test_statistics_survive_a_large_mean(shape, dtype, sms):
    """mean / std = 10³: the shifted sums and the (mean, M2) merges keep the variance"""
    n, c, h, w = shape
    check_gn(n, c, h, w, dtype, True, True, sms, mean=1000.0, std=1.0)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("shape", [(2, 64, 160, 160), (16, 256, 20, 20), (2, 2048, 10, 10)],
                         ids=lambda s: "x".join(map(str, s)))
def test_statistics_survive_an_outlying_first_row(shape, dtype, sms):
    """row 0 of every sample, whose values are the statistics' shift (csrc/wsgn.cu), 10σ above a mean of 10³ — a border
    pixel of a convolution's output, say: the variance loses about u·10² relatively, inside the bound"""
    n, c, h, w = shape
    check_gn(n, c, h, w, dtype, True, True, sms, mean=1000.0, std=1.0, outlier=10.0)


# C = 32: one channel per group, 64 row phases per pass — the narrowest width the kernels take (not in the backbone)
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("shape", [(1, 32, 1, 1), (1, 32, 7, 9), (3, 32, 40, 40), (16, 32, 64, 64)],
                         ids=lambda s: "x".join(map(str, s)))
def test_narrowest_width(shape, dtype, sms):
    n, c, h, w = shape
    for relu, res in EPILOGUES:
        check_gn(n, c, h, w, dtype, relu, res, sms)


def test_same_call_is_bit_identical(sms):
    x, gamma, beta, res, dy = _inputs(8, 256, 40, 40, torch.bfloat16)
    a = run_gn(x, gamma, beta, res, dy, True)
    b = run_gn(x, gamma, beta, res, dy, True)
    for u, v in zip(a, b):
        np.testing.assert_array_equal(u, v)


def test_c_abi_refusals():
    from distributed_sod_project_b200 import _lib, wsgn
    h = _lib.lib()
    x = torch.zeros(2 * 64 * 64 + 64, dtype=torch.float32, device="cuda")
    st = torch.zeros(2 * 32 * 2, device="cuda")
    gb = torch.ones(64, device="cuda")
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    eps = ctypes.c_float(1e-5)
    p = x.data_ptr()

    def fwd(c=64, dtype=0, xp=p, groups=32, wsb=ws.numel(), wsp=ws.data_ptr(), n=2):
        return h.sod_groupnorm_fwd(xp, None, p, dtype, gb.data_ptr(), gb.data_ptr(), st.data_ptr(), n, 16, c, groups, eps,
                                   1, wsp, wsb, None)

    def bwd(c=64, dtype=0, xp=p, groups=32, wsb=ws.numel()):
        return h.sod_groupnorm_bwd(p, xp, p, p, None, dtype, gb.data_ptr(), st.data_ptr(), gb.data_ptr(), gb.data_ptr(),
                                   2, 16, c, groups, 1, ws.data_ptr(), wsb, 0, None)

    assert fwd(c=48) == -1 and bwd(c=48) == -1                     # C % G != 0
    assert fwd(c=96) == -4 and bwd(c=96) == -4                     # C/8 not a power of two
    assert fwd(c=4096) == -4 and fwd(groups=16) == -4
    assert fwd(dtype=7) == -1 and bwd(dtype=7) == -1               # unsupported dtype
    assert fwd(xp=p + 4) == -2 and bwd(xp=p + 4) == -2             # misaligned
    assert fwd(wsp=ws.data_ptr() + 8) == -2
    assert fwd(wsb=16) == -3 and bwd(wsb=16) == -3                 # workspace
    assert fwd(n=0) == -1 and fwd(xp=None) == -1
    assert h.sod_groupnorm_workspace_bytes(2, 16, 96, 32) == 0
    w = torch.zeros(65, device="cuda")
    assert h.sod_ws_fwd(w.data_ptr(), w.data_ptr(), 0, 8, 1, eps, None) == -1          # K = 1
    assert h.sod_ws_fwd(w.data_ptr() + 2, w.data_ptr(), 0, 8, 8, eps, None) == -2      # misaligned
    assert h.sod_ws_fwd(w.data_ptr(), w.data_ptr(), 5, 8, 8, eps, None) == -1          # dtype
    assert h.sod_ws_bwd(w.data_ptr(), w.data_ptr() + 2, 0, w.data_ptr(), 8, 8, eps, 0, None) == -2
    assert h.sod_ws_bwd(w.data_ptr(), w.data_ptr(), 0, None, 8, 8, eps, 0, None) == -1
    torch.cuda.synchronize()
    # the module seam: CPU tensors and uncovered shapes raise, naming the shape
    with pytest.raises(_lib.SodError):
        wsgn.GroupNorm32(32, 64)(torch.zeros(1, 64, 2, 2))
    with pytest.raises(_lib.SodError, match=r"C=96"):
        wsgn.GroupNorm32(32, 96).cuda()(torch.zeros(1, 96, 2, 2, device="cuda"))
    with pytest.raises(_lib.SodError):
        wsgn.FusedWSConv2d(8, 8, 3, bias=False)(torch.zeros(1, 8, 4, 4))


def _ws_shapes():
    from distributed_sod_project_b200 import network
    m = network.wsgn_res50()
    seen = {}
    for mod in m.modules():
        if isinstance(mod, network.blocks.WSConv2d):
            seen.setdefault(tuple(mod.weight.shape), mod.weight.detach().clone())
    return seen


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_weight_standardisation_every_filter_shape(dtype):
    from distributed_sod_project_b200 import wsgn
    shapes = _ws_shapes()
    assert len(shapes) == 20
    g = torch.Generator().manual_seed(3)
    for shape, w in shapes.items():
        for cl in (False, True):
            wc = w.cuda().contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format)
            wc.requires_grad_(True)
            what = wsgn.standardize_weight(wc, dtype)
            assert what.dtype == dtype and what.stride() == wc.stride()
            up = torch.randn(shape, generator=g).to(dtype)
            what.backward(up.cuda())
            K = w[0].numel()
            D = K // 256 + 16
            w64 = w.double().numpy()
            ref = ow.ws_forward(w64)
            got = what.detach().double().cpu().numpy()
            bound = 2.0 ** -P[dtype] * np.abs(ref) + 8 * D * U * (1 + np.abs(ref))
            assert (np.abs(got - ref) <= bound).all(), (shape, cl)
            g64 = up.double().numpy()
            dref = ow.ws_backward(w64, g64)
            v = (w64.reshape(shape[0], -1) - w64.reshape(shape[0], -1).mean(axis=1, keepdims=True))
            sig = v.std(axis=1, ddof=1, keepdims=True)
            s = sig + 1e-5
            ga = np.abs(g64.reshape(shape[0], -1))
            mag = ga / s + ga.mean(axis=1, keepdims=True) / s + np.abs(v) * (ga * np.abs(v)).sum(axis=1, keepdims=True) / (
                s * s * (K - 1) * sig)
            dgot = wc.grad.double().cpu().numpy().reshape(shape[0], -1)
            assert (np.abs(dgot - dref.reshape(shape[0], -1)) <= 8 * D * U * mag).all(), (shape, cl)


def test_ws_backward_adds_into_a_bound_fp32_grad():
    from distributed_sod_project_b200 import _lib, wsgn
    w = torch.randn(64, 64, 3, 3, device="cuda").requires_grad_(True)
    w.grad = torch.full_like(w, 0.5)
    before = _lib.grad_writes
    what = wsgn.standardize_weight(w, torch.bfloat16)
    up = torch.randn_like(what)
    what.backward(up)
    assert _lib.grad_writes == before + 1
    w2 = w.detach().clone().requires_grad_(True)
    wsgn.standardize_weight(w2, torch.bfloat16).backward(up)
    torch.testing.assert_close(w.grad, w2.grad + 0.5, rtol=0, atol=1e-6)
