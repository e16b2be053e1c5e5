"""Parity of the SyncBN kernels (world 1 here; world 2 in test_gpu_multi.py) with the fp64 oracle and with
torch's own batch_norm autograd."""

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import syncbn as obn

pytestmark = pytest.mark.gpu

SHAPES = [  # N, C, H, W  — the channel counts of the TestModel's 84 BN layers, plus ragged row counts
    (2, 32, 5, 7), (16, 64, 80, 80), (4, 64, 33, 31), (2, 128, 9, 9), (16, 256, 20, 20), (3, 512, 7, 5),
    (16, 1024, 20, 20), (2, 2048, 2, 2), (16, 2048, 10, 10), (1, 64, 1, 1), (16, 32, 160, 160),
]


def _mk(shape, dtype, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    t = (torch.randn(shape, generator=g) * scale + shift).to(dtype)
    return t.cuda().contiguous(memory_format=torch.channels_last)


def _bn(c):
    from distributed_sod_project_b200.syncbn import SyncBatchNorm
    bn = SyncBatchNorm(c).cuda()
    with torch.no_grad():
        bn.weight.copy_(torch.linspace(0.5, 1.5, c)); bn.bias.copy_(torch.linspace(-0.3, 0.3, c))
    return bn


def _tol(dtype):
    return dict(rtol=2e-2, atol=2e-2) if dtype != torch.float32 else dict(rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("variant", ["plain", "relu", "pre_relu", "res_relu", "all"])
def test_forward_backward_vs_oracle(shape, dtype, variant):
    n, c, h, w = shape
    x = _mk(shape, dtype, 1, 1.5, 0.3).requires_grad_(True)
    pre = _mk(shape, dtype, 2).requires_grad_(True) if variant in ("pre_relu", "all") else None
    res = _mk(shape, dtype, 3).requires_grad_(True) if variant in ("res_relu", "all") else None
    relu = variant != "plain"
    bn = _bn(c)
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    y = bn.fused_forward(x, pre_add=pre, residual=res, relu=relu)
    dy = _mk(shape, dtype, 4)
    y.backward(dy)
    torch.cuda.synchronize()

    f64 = lambda t: None if t is None else t.detach().float().cpu().numpy().astype(np.float64)  # noqa: E731
    ref = obn.syncbn_forward([f64(x)], f64(bn.weight), f64(bn.bias), f64(rm0), f64(rv0),
                             pre_adds=None if pre is None else [f64(pre)],
                             residuals=None if res is None else [f64(res)], relu=relu)
    tol = _tol(dtype)
    np.testing.assert_allclose(f64(y), ref["ys"][0], **tol)
    if n * h * w > 1:
        np.testing.assert_allclose(f64(bn.running_mean), ref["running_mean"], rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(f64(bn.running_var), ref["running_var"], rtol=1e-3, atol=1e-5)
    # backward: the oracle masks with ITS y; use the kernel's y so a value sitting exactly on 0 cannot flip
    rb = obn.syncbn_backward([f64(dy)], ref["zs"], [f64(y)], ref["mean"], ref["invstd"], f64(bn.weight), relu=relu)
    btol = 3e-2 if dtype != torch.float32 else 2e-4
    if n * h * w == 1:
        # degenerate: one value per channel ⇒ var = 0, invstd = 1/sqrt(eps) ≈ 316 amplifies rounding; dz is 0 exactly
        assert np.abs(f64(x.grad)).max() < 1e-3
        return
    gscale = max(np.abs(rb["dzs"][0]).max(), 1e-6)
    assert np.abs(f64(x.grad) - rb["dzs"][0]).max() / gscale < btol
    if pre is not None:
        assert torch.equal(pre.grad, x.grad)
    if res is not None:
        assert np.abs(f64(res.grad) - rb["dresiduals"][0]).max() <= 1e-6 + 1e-2 * (dtype != torch.float32)
    rows = n * h * w
    np.testing.assert_allclose(f64(bn.weight.grad), rb["dgammas"][0], rtol=btol, atol=btol * max(1.0, rows ** 0.5))
    np.testing.assert_allclose(f64(bn.bias.grad), rb["dbetas"][0], rtol=btol, atol=btol * max(1.0, rows ** 0.5))
    assert int(bn.num_batches_tracked) == 1
    assert y.is_contiguous(memory_format=torch.channels_last) and y.dtype == dtype


@pytest.mark.parametrize("shape", [(16, 64, 80, 80), (2, 2048, 2, 2), (5, 256, 13, 11)])
def test_matches_torch_batch_norm_fp32(shape):
    """independent cross-check: torch's BatchNorm2d (train mode) + ReLU with autograd"""
    n, c, h, w = shape
    x1 = _mk(shape, torch.float32, 7, 2.0, -0.5).requires_grad_(True)
    x2 = x1.detach().clone().requires_grad_(True)
    bn = _bn(c)
    tbn = nn.BatchNorm2d(c).cuda()
    tbn.load_state_dict(bn.state_dict())
    dy = _mk(shape, torch.float32, 8)
    bn.fused_forward(x1, relu=True).backward(dy)
    F.relu(tbn(x2)).backward(dy)
    assert torch.allclose(x1.grad, x2.grad, rtol=1e-3, atol=1e-4)
    assert torch.allclose(bn.weight.grad, tbn.weight.grad, rtol=1e-3, atol=1e-3)
    assert torch.allclose(bn.running_var, tbn.running_var, rtol=1e-4, atol=1e-6)


def test_eval_mode_and_nchw_input():
    bn = _bn(64)
    with torch.no_grad():
        bn.running_mean.normal_(); bn.running_var.uniform_(0.5, 2.0)
    bn.eval()
    x = torch.randn(3, 64, 11, 9, device="cuda")                       # plain NCHW: converted on entry
    y = bn(x)
    ref = F.batch_norm(x, bn.running_mean, bn.running_var, bn.weight, bias=bn.bias, training=False, eps=bn.eps)
    assert torch.allclose(y, ref, rtol=1e-5, atol=1e-5)
    assert int(bn.num_batches_tracked) == 0


def test_convert_shares_parameters_and_rejects_cpu():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.syncbn import SyncBatchNorm, convert_syncbn_model
    net = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(), nn.Sequential(nn.BatchNorm2d(8)))
    w = net[1].weight
    out = convert_syncbn_model(net)
    assert out is net and isinstance(net[1], SyncBatchNorm) and isinstance(net[3][0], SyncBatchNorm)
    assert net[1].weight is w                                            # Q2: optimizer built earlier keeps γ/β
    with pytest.raises(_lib.SodError):
        net[1](torch.zeros(1, 8, 2, 2))


def test_repeated_calls_are_deterministic():
    bn = _bn(256)
    x = _mk((16, 256, 20, 20), torch.bfloat16, 11)
    ys = [bn.fused_forward(x, relu=True).clone() for _ in range(5)]
    assert all(torch.equal(ys[0], y) for y in ys[1:])


def test_param_grads_accumulate_into_bound_grad():
    """with γ/β .grad pre-bound (FusedSGD's flat buffer) the kernel adds into them and autograd receives None"""
    bn = _bn(64)
    x = _mk((4, 64, 9, 9), torch.float32, 21).requires_grad_(True)
    dy = _mk((4, 64, 9, 9), torch.float32, 22)
    bn.fused_forward(x, relu=True).backward(dy)
    want_w, want_b = bn.weight.grad.clone(), bn.bias.grad.clone()
    bn2 = _bn(64)
    bn2.weight.grad = torch.full_like(bn2.weight, 0.5)
    bn2.bias.grad = torch.full_like(bn2.bias, -0.25)
    wptr = bn2.weight.grad.data_ptr()
    x2 = x.detach().clone().requires_grad_(True)
    bn2.fused_forward(x2, relu=True).backward(dy)
    assert bn2.weight.grad.data_ptr() == wptr
    assert torch.allclose(bn2.weight.grad, want_w + 0.5, rtol=1e-5, atol=1e-5)
    assert torch.allclose(bn2.bias.grad, want_b - 0.25, rtol=1e-5, atol=1e-5)
    assert torch.allclose(x2.grad, x.grad)


@pytest.mark.parametrize("shape", [(4, 64, 9, 9), (2, 32, 20, 20), (2, 512, 5, 5)])
@pytest.mark.parametrize("dtype,bdtype", [(torch.float32, torch.float32), (torch.bfloat16, torch.bfloat16)])
@pytest.mark.parametrize("two", [False, True])
def test_folded_conv_bias(shape, dtype, bdtype, two):
    """z = x (+pre) + b1 (+b2) inside the kernel; backward hands back Σ_rows dz as the bias gradient"""
    n, c, h, w = shape
    x = _mk(shape, dtype, 31, 1.5, 0.2).requires_grad_(True)
    pre = _mk(shape, dtype, 32).requires_grad_(True) if two else None
    g = torch.Generator().manual_seed(33)
    b1 = torch.randn(c, generator=g).to(bdtype).cuda().requires_grad_(True)
    b2 = torch.randn(c, generator=g).to(bdtype).cuda().requires_grad_(True) if two else None
    if two:      # second bias: gradient accumulated into a pre-bound .grad, first one returned through autograd
        b2.grad = torch.full_like(b2, 0.5)
    bn = _bn(c)
    y = bn.fused_forward(x, pre_add=pre, relu=True, conv_bias=(b1, b2))
    dy = _mk(shape, dtype, 34)
    y.backward(dy)
    torch.cuda.synchronize()
    f64 = lambda t: t.detach().float().cpu().numpy().astype(np.float64)  # noqa: E731
    btot = f64(b1) + (f64(b2) if two else 0.0)
    xin = f64(x) + btot[None, :, None, None]
    ref = obn.syncbn_forward([xin], f64(bn.weight), f64(bn.bias), np.zeros(c), np.ones(c),
                             pre_adds=[f64(pre)] if two else None, relu=True)
    tol = _tol(dtype)
    np.testing.assert_allclose(f64(y), ref["ys"][0], **tol)
    np.testing.assert_allclose(f64(bn.running_mean), ref["running_mean"], rtol=1e-3, atol=2e-3 if dtype != torch.float32 else 1e-5)
    rb = obn.syncbn_backward([f64(dy)], ref["zs"], [f64(y)], ref["mean"], ref["invstd"], f64(bn.weight), relu=True)
    gscale = max(np.abs(rb["dzs"][0]).max(), 1e-6)
    btol = 3e-2 if dtype != torch.float32 else 3e-4
    assert np.abs(f64(x.grad) - rb["dzs"][0]).max() / gscale < btol
    want_db = rb["dzs"][0].sum(axis=(0, 2, 3))          # ≈ 0 at world 1: BN output does not depend on the bias
    scale = np.abs(rb["dzs"][0]).sum(axis=(0, 2, 3)).max()
    assert np.abs(f64(b1.grad) - want_db).max() <= (2e-2 if dtype != torch.float32 else 1e-4) * scale + 1e-6
    if two:
        assert np.abs(f64(b2.grad) - 0.5 - want_db).max() <= (2e-2 if dtype != torch.float32 else 1e-4) * scale + 8e-3
        assert torch.equal(pre.grad, x.grad)


@pytest.mark.parametrize("shape", [(16, 64, 80, 80), (4, 64, 33, 31), (16, 256, 20, 20), (2, 2048, 2, 2), (16, 32, 160, 160)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("with_pre,with_cb", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("hints", [False, True])
def test_bwd_mask_from_x_agrees_with_mask_from_y(shape, dtype, with_pre, with_cb, hints, monkeypatch):
    """SOD_BN_BWD_MASK_FROM_X re-derives the ReLU mask from x: against the y-mask variant on the same inputs the result
    may differ only by the summation order of the statistics (different strip geometry)."""
    from distributed_sod_project_b200 import syncbn
    n, c, h, w = shape
    x = _mk(shape, dtype, 1, 1.5, 0.3).requires_grad_(True)
    pre = _mk(shape, dtype, 2) if with_pre else None
    cb = (torch.linspace(-0.5, 0.5, c, device="cuda").to(dtype).requires_grad_(True), None) if with_cb else (None, None)
    bn = _bn(c)
    y = bn.fused_forward(x, pre_add=pre, relu=True, conv_bias=cb)
    _, _, _, _, mean, invstd = y.grad_fn.saved_tensors
    dy = _mk(shape, dtype, 4)
    out = {}
    for flag in (False, True):
        monkeypatch.setattr(syncbn, "MASK_FROM_X", flag)       # restored to the session's setting when the test ends
        monkeypatch.setattr(syncbn, "L2_HINTS", hints and flag)
        dcb = (torch.zeros_like(cb[0]), None) if with_cb else (None, None)
        dz, _, dg, db = syncbn.raw_backward(dy, x.detach(), pre, y.detach(), bn.weight.detach(), mean, invstd, True, False,
                                            conv_bias=tuple(None if t is None else t.detach() for t in cb),
                                            dconv_bias=dcb, bias=bn.bias.detach())
        torch.cuda.synchronize()
        out[flag] = (dz.float(), dg, db, None if dcb[0] is None else dcb[0].float())
    scale = float(out[False][0].abs().max())
    tol = 2e-5 if dtype == torch.float32 else 1e-2
    assert float((out[False][0] - out[True][0]).abs().max()) <= tol * scale
    rows = n * h * w
    for a, b in zip(out[False][1:], out[True][1:]):
        if a is not None:
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-4 * rows ** 0.5 if dtype == torch.float32 else 2e-2 * rows ** 0.5)


@pytest.mark.parametrize("mean,std", [(100.0, 0.1), (-50.0, 1e-2), (1000.0, 1.0), (0.0, 1.0)])
@pytest.mark.parametrize("shape", [(16, 64, 80, 80), (4, 256, 20, 20), (16, 32, 160, 160), (2, 2048, 2, 2)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_forward_statistics_survive_a_large_mean(mean, std, shape, with_bias):
    """|mean| ≫ std (a post-residual channel): E[x²] − E[x]² in fp32 would lose the variance ((mean/std)² · 2⁻²⁴ is
    6 % at 100/0.1 and > 100 % at 50/0.01).  The kernel accumulates deviations from a sample row and merges per-strip
    (mean, M2) pairs — the scheme apex / torch SyncBN use — so the statistics must agree with the fp64 oracle.
    Tolerances: invstd 2e-3 relative (limited by the fp32 input's own spacing at |x| ≈ |mean|), y 2e-2 absolute at the
    two extreme settings (x·scale and the shift are ≈ |mean|/std ≈ 5·10³ and cancel in fp32: one ulp there is 5·10⁻⁴,
    and the fp32 mean itself is only known to ulp(|mean|)/std)."""
    n, c, h, w = shape
    x = _mk(shape, torch.float32, 11, std, mean)
    bn = _bn(c)
    cb = (torch.linspace(-3, 3, c).cuda() * (1 + abs(mean))) if with_bias else None     # a huge folded conv bias changes nothing
    y = bn.fused_forward(x, relu=False, conv_bias=(cb, None))
    torch.cuda.synchronize()
    x64 = x.detach().cpu().numpy().astype(np.float64)
    if cb is not None:
        x64 = x64 + cb.cpu().numpy().astype(np.float64)[None, :, None, None]
    ref = obn.syncbn_forward([x64], bn.weight.detach().cpu().numpy().astype(np.float64),
                             bn.bias.detach().cpu().numpy().astype(np.float64), np.zeros(c), np.ones(c), relu=False)
    # the statistics the kernel saved for the backward (mean, invstd) are the direct evidence
    saved = y.grad_fn.saved_tensors
    got_invstd = saved[5].double().cpu().numpy()
    np.testing.assert_allclose(got_invstd, ref["invstd"], rtol=2e-3)
    np.testing.assert_allclose(saved[4].double().cpu().numpy(), ref["mean"], rtol=1e-6, atol=1e-6 * max(1.0, abs(mean)))
    # running_var = 0.9 + 0.1 * unbiased variance is stored in fp32: its own spacing near 0.9 (6e-8) limits what can be read back
    var_ref = 1.0 / ref["invstd"] ** 2
    got_rv = (bn.running_var.double().cpu().numpy() - 0.9) / 0.1
    rows = n * h * w
    np.testing.assert_allclose(got_rv * (rows - 1) / rows, var_ref - 1e-5, rtol=4e-3, atol=7e-7)
    got_mean = bn.running_mean.double().cpu().numpy() / 0.1
    np.testing.assert_allclose(got_mean, ref["mean"], rtol=1e-6, atol=1e-6 * max(1.0, abs(mean)))
    extreme = abs(mean) / std > 500
    np.testing.assert_allclose(y.detach().double().cpu().numpy(), ref["ys"][0], rtol=0, atol=(4e-2 if with_bias else 2e-2) if extreme else 2e-3)
