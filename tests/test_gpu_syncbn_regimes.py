"""SyncBN kernels in every ring regime of this GPU, in fp32, bf16 and fp16, at rounding-level tolerances.

Which branches a launch takes (chunks per strip against the stage count, a short last strip, a partial last chunk, one /
a few / a grid-filling number of strips, the channel count) is decided at launch time from the device.  The covering set
of oracle/syncbn_geometry.py gives every kernel instance every value of every regime axis, with shapes chosen for the
SM count and shared memory of the device the test runs on; each launch's strip count is read back from the kernels'
debug stamps, so a change of the host geometry that moved a case out of its regime fails here instead of silently
testing something else.

Reference: the fp64 formulas of oracle/syncbn.py (test_fp64_reference_matches_the_oracle pins the two together),
evaluated on the GPU on the inputs as rounded to the I/O dtype.  Tolerances:

* fp32 outputs (saved mean / invstd, running statistics, dγ, dβ, fp32 conv-bias gradients), for every I/O dtype: they
  are accumulated in fp32 from inputs the I/O dtype holds exactly, so 1e-5 relative; a sum over `rows` terms of random
  sign is held to 1e-5 · √rows · rms(term).  num_batches_tracked is exact; in eval the running statistics are untouched.
* y, dz (and a conv-bias gradient kept in T): one ulp of T at |ref| (the final rounding is half of it; the other half
  covers a value next to a rounding boundary) plus the fp32 slack of the kernel's arithmetic: 2⁻¹⁹ of the magnitudes
  that enter the fused multiply-adds (|z·scale|, |shift| parts, |residual|; |A·dy|, |B|·(|z| + |mean|), |A·mean_dy|)
  plus the error of the two fp32 column means of the backward (2⁻¹⁸ of their absolute means, times their weight).
  2⁻¹⁹ is ~16 fp32 ulps, 2⁻¹¹ of a bf16 ulp.
* dres is the masked dy bit for bit; the ReLU mask is the kernel's own y.  An element may be positive in one of the
  kernel's y and the reference's y but not in the other only where the exact y is within the tolerance above of 0.
* fp16 gradients are those of a 2¹⁶-scaled mean loss (dy ≈ 2¹⁶ / numel), so small tensors see large values and large
  ones see fp16 subnormals.
"""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import syncbn as obn
from oracle import syncbn_geometry as geo

pytestmark = pytest.mark.gpu

TORCH_DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}
MANT = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}
EMIN = {torch.float32: -126, torch.bfloat16: -126, torch.float16: -14}
CASES = geo.covering_cases()
# a few regime cases that are also run with the cooperative and the programmatic-dependent launch
LAUNCH_MODE_CASES = [
    next(c.id for c in CASES if c.kind == "fwd" and c.dtype == "float32" and c.spec == 0),                    # grid-filling
    next(c.id for c in CASES if c.kind == "fwd" and c.dtype == "bfloat16" and c.res and c.pre and c.spec == 3),
    next(c.id for c in CASES if c.kind == "bwd" and c.dtype == "float16" and c.xmask and c.nbias and c.spec == 0),
    next(c.id for c in CASES if c.kind == "bwd" and c.dtype == "bfloat16" and c.res and c.pre and c.spec == 5),
]
RAN: dict = {}              # case id → cells of the regime table it reached on this device
EPS, MOMENTUM = 1e-5, 0.1
STAMP_BYTES = geo.K_MAX_GRID * 64


@pytest.fixture
def sbn(monkeypatch):
    """the syncbn module with the debug stamps on and every switch at its default, restored afterwards"""
    from distributed_sod_project_b200 import syncbn
    monkeypatch.setattr(syncbn, "DEBUG_FLAGS", 4)          # SOD_DEBUG_TIMING: per-CTA start stamps
    monkeypatch.setattr(syncbn, "LAUNCH_MODE", "plain")
    monkeypatch.setattr(syncbn, "MASK_FROM_X", True)
    monkeypatch.setattr(syncbn, "L2_HINTS", True)
    return syncbn


def _device():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.shared_memory_per_block_optin


def ulp(ref, dtype):
    """spacing of `dtype` at |ref| (fp64 tensor), subnormal spacing below the smallest normal"""
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** EMIN[dtype])))
    return torch.exp2(e - MANT[dtype])


class Stamps:
    """the kernels' SOD_DEBUG_TIMING area: slot 0 of CTA b is its start time, so the number of non-zero slots is the grid"""

    def __init__(self, syncbn, C):
        from distributed_sod_project_b200 import _lib
        self.ws = syncbn._dev_state(torch.device("cuda", torch.cuda.current_device()))["ws"]
        self.off = int(_lib.lib().sod_syncbn_workspace_bytes(1, C))
        assert self.off % 8 == 0 and self.off + STAMP_BYTES <= self.ws.numel()

    def zero(self):
        self.ws[self.off:self.off + STAMP_BYTES].zero_()

    def ctas(self):
        torch.cuda.synchronize()
        return int((self.ws[self.off:self.off + STAMP_BYTES].view(torch.int64).view(geo.K_MAX_GRID, 8)[:, 0] != 0).sum())


def rows_of(t):
    """[N, C, H, W] channels-last → [rows, C] float64"""
    return t.detach().permute(0, 2, 3, 1).reshape(-1, t.shape[1]).double()


def ref_forward(z, gamma, beta, res=None, relu=False, rm=None, rv=None, training=True):
    """oracle/syncbn.py syncbn_forward on [rows, C] fp64 (world 1); eval: the running statistics instead"""
    if training:
        mean = z.mean(0)
        var = ((z - mean) ** 2).mean(0)
    else:
        mean, var = rm, rv
    invstd = 1.0 / torch.sqrt(var + EPS)
    y = (z - mean) * (invstd * gamma) + beta
    if res is not None:
        y = y + res
    if relu:
        y = y.clamp_min(0.0)
    return y, mean, var, invstd


def ref_backward(dy_m, z, mean, invstd, gamma):
    """oracle/syncbn.py syncbn_backward on [rows, C] fp64, dy already masked"""
    mean_dy = dy_m.mean(0)
    mean_dy_xmu = (dy_m * (z - mean)).mean(0)
    dz = (dy_m - mean_dy - (z - mean) * invstd * invstd * mean_dy_xmu) * invstd * gamma
    return dz, (dy_m * (z - mean) * invstd).sum(0), dy_m.sum(0), mean_dy, mean_dy_xmu


def assert_sum_close(got, ref, terms, what, extra=0.0):
    """an fp32 column sum over `rows` terms: 1e-5 relative, 1e-5 · √rows · rms(term) absolute (+ `extra`)"""
    rows = terms.shape[0]
    tol = 1e-5 * ref.abs() + 1e-5 * rows ** 0.5 * terms.pow(2).mean(0).sqrt() + extra + 1e-30
    err = (got.double() - ref).abs()
    assert bool((err <= tol).all()), f"{what}: worst {float((err / tol).max()):.3g}x the tolerance"


def assert_within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = err > tol
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} elements off, worst "
                                 f"{float((err / tol).max()):.3g}x the tolerance (got {float(got.double()[bad][0])}, "
                                 f"ref {float(ref[bad][0])})")


def make_inputs(case, shape, dtype):
    n, c, h, w = shape
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(case.id.encode()))
    mk = lambda scale, shift=0.0: (torch.randn(shape, generator=gen, device="cuda") * scale + shift).to(dtype) \
        .contiguous(memory_format=torch.channels_last)  # noqa: E731
    dscale = 2.0 ** 16 / (n * c * h * w) if dtype == torch.float16 else 1.0
    bdt = torch.float32 if case.bias_fp32 else dtype
    ins = dict(x=mk(1.5, 2.0), pre=mk(0.5) if case.pre else None, res=mk(1.0) if case.res else None, dy=mk(dscale),
               cbs=[(torch.randn(c, generator=gen, device="cuda") * 0.5).to(bdt) for _ in range(case.nbias)])
    return ins


def make_bn(c):
    from distributed_sod_project_b200.syncbn import SyncBatchNorm
    bn = SyncBatchNorm(c, eps=EPS, momentum=MOMENTUM).cuda()
    with torch.no_grad():
        sign = torch.where(torch.arange(c) % 3 == 0, -1.0, 1.0)
        bn.weight.copy_(torch.linspace(0.5, 1.5, c) * sign)
        bn.bias.copy_(torch.linspace(-0.3, 0.3, c))
        bn.running_mean.copy_(torch.linspace(-0.5, 0.5, c))
        bn.running_var.copy_(torch.linspace(0.5, 2.0, c))
    return bn


def run_case(case, sbn, check_geometry=True):
    """one case on this device: the launches, with their grids checked against the model; returns the tensors"""
    sm, smem = _device()
    g = geo.resolve(case, sm, smem)
    assert g is not None, f"{case.id}: regime {geo.SPECS[case.spec]} is unreachable on {sm} SMs / {smem} B"
    shape = geo.shape_of(g)
    dtype = TORCH_DT[case.dtype]
    es = geo.DTYPE_BYTES[case.dtype]
    ins = make_inputs(case, shape, dtype)
    bn = make_bn(g.C)
    stamps = Stamps(sbn, g.C)
    sbn.MASK_FROM_X, sbn.L2_HINTS = case.xmask, case.hint          # the fixture restores both
    out = dict(g=g, shape=shape, dtype=dtype, ins=ins, bn=bn, rm0=bn.running_mean.clone(), rv0=bn.running_var.clone())
    x = ins["x"].clone().requires_grad_(case.kind == "bwd")
    pre = None if ins["pre"] is None else ins["pre"].clone().requires_grad_(case.kind == "bwd")
    res = None if ins["res"] is None else ins["res"].clone().requires_grad_(case.kind == "bwd")
    cbs = [b.clone().requires_grad_(case.kind == "bwd") for b in ins["cbs"]]
    if case.kind == "bwd" and case.nbias == 2:
        cbs[1].grad = torch.full_like(cbs[1], 0.5)         # second bias: accumulated into a bound .grad
    if case.into:
        bn.weight.grad = torch.full_like(bn.weight, 0.5)
        bn.bias.grad = torch.full_like(bn.bias, -0.25)
    conv_bias = tuple(cbs) + (None,) * (2 - len(cbs))
    gf = geo.make_geom(g.rows, g.C, es, *geo.fwd_site(case.pre, case.res), sm, smem)

    stamps.zero()
    y = bn.fused_forward(x, pre_add=pre, residual=res, relu=case.relu, conv_bias=conv_bias)
    if check_geometry:
        assert stamps.ctas() == gf.strips, f"forward grid {stamps.ctas()} != model {gf.strips}"
    out.update(y=y.detach(), mean=y.grad_fn.saved_tensors[4].clone(), invstd=y.grad_fn.saved_tensors[5].clone(),
               rm=bn.running_mean.clone(), rv=bn.running_var.clone(), nbt=int(bn.num_batches_tracked))
    if case.kind == "fwd":
        # eval: running statistics near the data's mean, variances from 1e-4 (where eps matters) to 3
        with torch.no_grad():
            bn.running_mean.copy_(2.0 + torch.linspace(-1, 1, g.C, device="cuda"))
            bn.running_var.copy_(torch.logspace(-4, 0.5, g.C, device="cuda"))
        bn.eval()
        out.update(rm_e=bn.running_mean.clone(), rv_e=bn.running_var.clone())
        stamps.zero()
        with torch.no_grad():
            out["y_eval"] = bn.fused_forward(x, pre_add=pre, residual=res, relu=case.relu, conv_bias=conv_bias)
        if check_geometry:
            assert stamps.ctas() == gf.strips
        assert torch.equal(bn.running_mean, out["rm_e"]) and torch.equal(bn.running_var, out["rv_e"])
        assert int(bn.num_batches_tracked) == out["nbt"]
        return out
    stamps.zero()
    y.backward(ins["dy"])
    if check_geometry:
        assert stamps.ctas() == g.strips, f"backward grid {stamps.ctas()} != model {g.strips}"
    out.update(dz=x.grad, dpre=None if pre is None else pre.grad, dres=None if res is None else res.grad,
               dgamma=bn.weight.grad.clone(), dbeta=bn.bias.grad.clone(), dcbs=[b.grad.clone() for b in cbs])
    return out


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_syncbn_regime_parity(case, sbn):
    sm, _ = _device()
    o = run_case(case, sbn)
    g, dtype, ins = o["g"], o["dtype"], o["ins"]
    gamma, beta = rows_of(o["bn"].weight[None, :, None, None])[0], rows_of(o["bn"].bias[None, :, None, None])[0]
    cb = sum((b.double() for b in ins["cbs"]), torch.zeros(g.C, dtype=torch.float64, device="cuda"))
    zx = rows_of(ins["x"]) + (rows_of(ins["pre"]) if case.pre else 0.0)       # exact (the kernel's fp32 sum is rounded)
    z = zx + cb
    res = rows_of(ins["res"]) if case.res else None
    rows = g.rows

    # ---- forward, training ----------------------------------------------------------------------------------
    y_ref, mean, var, invstd = ref_forward(z, gamma, beta, res, case.relu)
    std = var.sqrt()
    assert_within(o["mean"], mean, 1e-5 * (mean.abs() + std) + 1e-30, "saved mean")
    np.testing.assert_allclose(o["invstd"].double().cpu().numpy(), invstd.cpu().numpy(), rtol=1e-5, err_msg="saved invstd")
    rm_ref = (1 - MOMENTUM) * o["rm0"].double() + MOMENTUM * mean
    rv_ref = (1 - MOMENTUM) * o["rv0"].double() + MOMENTUM * var * (rows / max(rows - 1, 1))
    # plus the fp32 rounding of the momentum update's two products and sum (the old value may be far larger than the result)
    upd = 2.0 ** -22 * ((1 - MOMENTUM) * o["rm0"].double().abs() + MOMENTUM * mean.abs())
    assert_within(o["rm"], rm_ref, 1e-5 * (rm_ref.abs() + MOMENTUM * std) + upd, "running mean")
    assert_within(o["rv"], rv_ref, 1e-5 * rv_ref.abs() + 1e-30, "running var")
    assert o["nbt"] == 1
    sc = (invstd * gamma).abs()
    slack = 2.0 ** -19 * (zx.abs() * sc + (mean.abs() + std + cb.abs()) * sc + beta.abs() + (res.abs() if res is not None else 0.0))
    y = rows_of(o["y"])
    ytol = ulp(y_ref, dtype) + slack
    assert_within(y, y_ref, ytol, "y")
    if case.relu:
        # an element whose exact y is within the kernel's fp32 error of 0 may land on either side; no other may flip
        flips = (y > 0) != (y_ref > 0)
        assert int((flips & (y_ref.abs() > ytol)).sum()) == 0, "ReLU mask flips"
        assert float(flips.double().mean()) < 1e-4

    if case.kind == "fwd":
        # ---- forward, eval: the plain fp64 formula with the running statistics ---------------------------------
        rm_e, rv_e = o["rm_e"].double(), o["rv_e"].double()
        ye_ref, _, _, inv_e = ref_forward(z, gamma, beta, res, case.relu, rm_e, rv_e, training=False)
        sc_e = (inv_e * gamma).abs()
        slack_e = 2.0 ** -19 * (zx.abs() * sc_e + (rm_e.abs() + cb.abs()) * sc_e + beta.abs() + (res.abs() if res is not None else 0.0))
        assert_within(rows_of(o["y_eval"]), ye_ref, ulp(ye_ref, dtype) + slack_e, "eval y")
    else:
        # ---- backward: reference with the kernel's own saved statistics and ReLU mask ----------------------------
        dy = rows_of(ins["dy"])
        dy_m = dy * (y > 0) if case.relu else dy
        kmean, kinv = o["mean"].double(), o["invstd"].double()
        dz_ref, dg_ref, db_ref, mdy, mdx = ref_backward(dy_m, z, kmean, kinv, gamma)
        A = gamma * kinv
        B = -A * kinv * kinv * mdx
        slack = (2.0 ** -19 * ((A * dy_m).abs() + B.abs() * (z.abs() + kmean.abs()) + (A * mdy).abs())
                 + A.abs() * 2.0 ** -18 * dy_m.abs().mean(0)
                 + (A * kinv * kinv).abs() * (z - kmean).abs() * 2.0 ** -18 * (dy_m * (z - kmean)).abs().mean(0))
        assert_within(rows_of(o["dz"]), dz_ref, ulp(dz_ref, dtype) + slack, "dz")
        if case.pre:
            assert torch.equal(o["dpre"], o["dz"])
        if case.res:
            assert torch.equal(rows_of(o["dres"]), dy_m), "dres is the masked dy"
        g0, b0 = (0.5, -0.25) if case.into else (0.0, 0.0)
        # dγ = Σ dy·(z − mean)·invstd: the kernel's fp32 z = x + pre and its mean − bias are rounded; a column of
        # near-constant z (one row: var = 0, invstd = 1/√eps) leaves only that rounding
        z_round = kinv * (2.0 ** -22 * (kmean.abs() + cb.abs()) * db_ref.abs() + 2.0 ** -23 * (dy_m * zx).pow(2).sum(0).sqrt())
        assert_sum_close(o["dgamma"].double() - g0, dg_ref, dy_m * (z - kmean) * kinv, "dgamma", z_round)
        assert_sum_close(o["dbeta"].double() - b0, db_ref, dy_m, "dbeta")
        # Σ dz = A·(Σ dy − rows·mean_dy) + B·Σ(z − mean): ≈ 0 at world 1, so the scale is that of the two terms, not of dz
        cb_terms = (A * dy_m).abs() + (B * (z - kmean)).abs()
        cb_round = B.abs() * 2.0 ** -22 * (kmean.abs() + cb.abs()) * rows
        for i, d in enumerate(o["dcbs"]):
            dcb_ref = dz_ref.sum(0) + (0.5 if i == 1 else 0.0)
            if d.dtype == torch.float32:
                assert_sum_close(d.double(), dcb_ref, cb_terms, f"conv bias {i} gradient", cb_round)
            else:
                tol = ulp(dcb_ref, d.dtype) + 1e-5 * rows ** 0.5 * cb_terms.pow(2).mean(0).sqrt() + cb_round
                assert_within(d, dcb_ref, tol, f"conv bias {i} gradient")
    RAN[case.id] = geo.cells(case, g, sm)


@pytest.mark.parametrize("mode", ["coop", "pdl"])
@pytest.mark.parametrize("case_id", LAUNCH_MODE_CASES)
def test_launch_modes_are_bit_identical(case_id, mode, sbn, monkeypatch):
    """SOD_BN_LAUNCH=coop (cooperative launch) and pdl (programmatic dependent launch) change how the grid is scheduled,
    nothing it computes"""
    case = next(c for c in CASES if c.id == case_id)
    outs = []
    for m in ("plain", mode):
        monkeypatch.setattr(sbn, "LAUNCH_MODE", m)
        outs.append(run_case(case, sbn))
    keys = ("y", "mean", "invstd", "rm", "rv", "y_eval") if case.kind == "fwd" else ("y", "mean", "invstd", "dz", "dres", "dgamma", "dbeta")
    for k in keys:
        a, b = outs[0][k], outs[1][k]
        assert (a is None and b is None) or torch.equal(a, b), k
    if case.kind == "bwd":
        assert all(torch.equal(a, b) for a, b in zip(outs[0]["dcbs"], outs[1]["dcbs"]))


def test_fp64_reference_matches_the_oracle():
    """the GPU fp64 reference above is oracle/syncbn.py's arithmetic"""
    g = torch.Generator().manual_seed(5)
    n, c, h, w = 3, 16, 5, 7
    x, pre, res, dy = (torch.randn((n, c, h, w), generator=g, dtype=torch.float64) for _ in range(4))
    gamma, beta = torch.linspace(0.5, 1.5, c, dtype=torch.float64), torch.linspace(-0.3, 0.3, c, dtype=torch.float64)
    want = obn.syncbn_forward([x.numpy()], gamma.numpy(), beta.numpy(), np.zeros(c), np.ones(c), pre_adds=[pre.numpy()],
                              residuals=[res.numpy()], relu=True)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, c).cuda()  # noqa: E731
    y, mean, var, invstd = ref_forward(rows(x) + rows(pre), gamma.cuda(), beta.cuda(), rows(res), True)
    np.testing.assert_allclose(y.cpu().numpy(), np.moveaxis(want["ys"][0], 1, -1).reshape(-1, c), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(invstd.cpu().numpy(), want["invstd"], rtol=1e-12)
    ymask = np.moveaxis(want["ys"][0], 1, -1).reshape(-1, c) > 0
    wb = obn.syncbn_backward([dy.numpy()], want["zs"], want["ys"], want["mean"], want["invstd"], gamma.numpy(), relu=True)
    dz, dg, db, _, _ = ref_backward(rows(dy) * torch.tensor(ymask, device="cuda"), rows(x) + rows(pre), mean, invstd, gamma.cuda())
    np.testing.assert_allclose(dz.cpu().numpy(), np.moveaxis(wb["dzs"][0], 1, -1).reshape(-1, c), rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(dg.cpu().numpy(), wb["dgammas"][0], rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(db.cpu().numpy(), wb["dbetas"][0], rtol=1e-10, atol=1e-12)


def test_fp16_mask_from_x_matches_the_stored_y(sbn, monkeypatch):
    """fp16 output flushes every fp32 y in (0, 2⁻²⁵] to +0, so torch's relu and the y-mask backward drop the gradient of
    those elements.  The mask-from-x backward re-derives y in fp32 and must round it to fp16 before taking the sign.
    Channels with γ = 2⁻²⁶ put most positive y into that interval (|normalized| ≤ 2) and the rest just above it."""
    shape = (4, 64, 16, 16)
    n, c, h, w = shape
    rows = n * h * w
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(shape, generator=gen, device="cuda").half().contiguous(memory_format=torch.channels_last)
    dy = (torch.randn(shape, generator=gen, device="cuda") * 2.0 ** 10).half().contiguous(memory_format=torch.channels_last)
    bn = make_bn(c)
    tiny = torch.arange(c, device="cuda") % 2 == 0
    with torch.no_grad():
        bn.weight[tiny] = 2.0 ** -26
        bn.bias[tiny] = 0.0
    y = bn.fused_forward(x, relu=True)
    _, _, _, _, mean, invstd = y.grad_fn.saved_tensors
    gamma, beta = rows_of(bn.weight[None, :, None, None])[0], rows_of(bn.bias[None, :, None, None])[0]
    y64 = (rows_of(x) - mean.double()) * (invstd.double() * gamma) + beta
    flushed = (y64 > 0) & (y64 <= 2.0 ** -25)
    assert int(flushed.sum()) > 1000 and float((rows_of(y)[flushed] == 0).double().mean()) > 0.99
    out = {}
    for xmask in (False, True):
        monkeypatch.setattr(sbn, "MASK_FROM_X", xmask)
        out[xmask] = sbn.raw_backward(dy, x.detach(), None, y.detach(), bn.weight.detach(), mean, invstd, True, False,
                                      bias=bn.bias.detach())
    torch.cuda.synchronize()
    dz_y, _, dg_y, db_y = out[False]
    dz_x, _, dg_x, db_x = out[True]
    # same mask ⇒ same results up to the summation order of two strip geometries
    dym = rows_of(dy) * (rows_of(y) > 0)
    assert_sum_close(db_x.double(), db_y.double(), dym, "dbeta, mask from x vs from y")
    assert_sum_close(dg_x.double(), dg_y.double(), dym * (rows_of(x) - mean.double()) * invstd.double(), "dgamma")
    dzy = rows_of(dz_y)
    assert_within(rows_of(dz_x), dzy, ulp(dzy, torch.float16) + 2.0 ** -19 * float(dzy.abs().max()), "dz, mask from x vs from y")
    # torch's relu(batch_norm) autograd on the same fp16 input masks with its own fp16 y: it may differ from the kernel's y
    # only where the two fp32 computations of y straddle a rounding boundary
    xt = x.detach().clone().requires_grad_(True)
    wt, bt = bn.weight.detach().clone().requires_grad_(True), bn.bias.detach().clone().requires_grad_(True)
    F.relu(F.batch_norm(xt, None, None, wt, bt, training=True, eps=EPS)).backward(dy)
    yt = F.relu(F.batch_norm(x, None, None, wt, bt, training=True, eps=EPS)).detach()
    disagree = (rows_of(yt) > 0) != (rows_of(y) > 0)
    assert float(disagree.double().mean()) < 1e-3
    tol = 1e-5 * rows ** 0.5 * dym.pow(2).mean(0).sqrt() + rows_of(dy).abs().mul(disagree).sum(0) + 1e-5 * db_y.double().abs()
    assert bool(((bt.grad.double() - db_x.double()).abs() <= tol).all()), "dbeta against torch's relu(batch_norm)"


@pytest.mark.parametrize("mean,std", [(100.0, 0.1), (1000.0, 1.0)])
@pytest.mark.parametrize("shape", [(16, 64, 80, 80), (4, 256, 20, 20), (2, 2048, 2, 2)])
@pytest.mark.parametrize("relu", [False, True])
def test_backward_survives_a_large_mean(mean, std, shape, relu, sbn):
    """fp32, |mean| ≫ std: dz = A·dy + B·z + D with D ∋ −B·mean, so B·z and B·mean cancel and the result carries the
    rounding of both: ulp(|mean|)·|B| per term.  Held to 4·ulp(|mean|)·|B| plus the fp32 slack of the other terms and of
    the column means (see the module docstring); the reference uses the kernel's saved statistics."""
    n, c, h, w = shape
    gen = torch.Generator(device="cuda").manual_seed(17)
    x = (torch.randn(shape, generator=gen, device="cuda") * std + mean).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    dy = torch.randn(shape, generator=gen, device="cuda").contiguous(memory_format=torch.channels_last)
    bn = make_bn(c)
    y = bn.fused_forward(x, relu=relu)
    _, _, _, _, kmean, kinv = y.grad_fn.saved_tensors
    y.backward(dy)
    torch.cuda.synchronize()
    z = rows_of(x)
    gamma = rows_of(bn.weight[None, :, None, None])[0]
    dy_m = rows_of(dy) * (rows_of(y) > 0) if relu else rows_of(dy)
    kmean, kinv = kmean.double(), kinv.double()
    dz_ref, dg_ref, db_ref, mdy, mdx = ref_backward(dy_m, z, kmean, kinv, gamma)
    A = gamma * kinv
    B = -A * kinv * kinv * mdx
    tol = (4 * ulp(kmean, torch.float32) * B.abs() + ulp(dz_ref, torch.float32)
           + 2.0 ** -19 * ((A * dy_m).abs() + (A * mdy).abs() + B.abs() * (z - kmean).abs())
           + A.abs() * 2.0 ** -18 * dy_m.abs().mean(0)
           + (A * kinv * kinv).abs() * (z - kmean).abs() * 2.0 ** -18 * (dy_m * (z - kmean)).abs().mean(0))
    assert_within(rows_of(x.grad), dz_ref, tol, "dz")
    assert_sum_close(bn.bias.grad.double(), db_ref, dy_m, "dbeta")
    assert_sum_close(bn.weight.grad.double(), dg_ref, dy_m * (z - kmean) * kinv, "dgamma")


def test_every_regime_cell_ran_on_this_device():
    """every cell (kernel instance × regime axis value) of the covering set was reached by a passing case"""
    if not RAN:
        pytest.skip("the regime cases did not run in this session")
    missing_cases = [c.id for c in CASES if c.id not in RAN]
    assert not missing_cases, f"{len(missing_cases)} regime cases did not pass: {missing_cases[:5]}"
    got = set().union(*RAN.values())
    missing = geo.required_cells(got) - got
    assert not missing, sorted(missing)
