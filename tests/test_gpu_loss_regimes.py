"""The fused BCE+CEL kernels in every launch regime of this GPU, for all ten (logits, mask) × kernel instances, element
by element against fp64.

Which kernel runs and which branches its CTAs take (chunks per CTA against the resident limit or the ring's stage count
NS, one / a few / a grid-filling number of CTAs, a last CTA with fewer chunks or a partial last chunk, the scalar tail)
is decided at launch time from the device.  The covering set of oracle/loss_geometry.py gives every instance every value
of every regime axis, with sizes chosen for the SM count and shared memory of the device the test runs on.  For every
case `mode=1` (resident kernel or refusal) must raise exactly when the model says the slice does not fit, which checks
the model against the host code on the device itself; and `mode=2` (always the ring-streamed kernel) must give the same
bits as `mode=0` whenever mode 0 runs the resident kernel: the grid, `per_cta`, the per-thread order, the block
reduction and the fp64 reduction across CTAs are the same in both, so any difference is a slip of the ring or of the
newest-first re-stream.  Two identical launches give identical bytes (no atomics).  Every case has w_bce ≠ w_cel, a
grad_scale (2¹⁶ for fp16 logits, lowered only where the gradient would leave fp16's range), an eps that is either the
default or large enough to move α and β, mean or sum reduction, and a soft (k/255) or binary mask.

Reference: oracle/loss.py's formulas in fp64 (test_fp64_reference_matches_the_oracle pins the two together), on the
inputs as rounded to their dtypes.  u = 2⁻²⁴.  Bounds:

* p = sigmoid(x) and q = 1 − p come from e = __expf(−|x|) (ex2.approx of the fp32 product x·log2e: 2 ulp plus |x|·u
  relative from the rounded argument) and r = __fdividef(1, 1 + e) (2 ulp): ε(x) = (16 + 2|x|)·u relative for each.
* d = p(1 − t) + t·q is CEL's numerator term; the kernel sums d, p, t and the BCE term b = max(x, 0) − x·t + log1pf(e)
  (log1pf: 1 ulp, plus e's error ε(x), times 1.5 for margin; the fp32 product, difference and sum: u·(2|x·t| + 3b))
  along a per-thread chain of 8 per chunk (+1 for the scalar tail), 5 shuffle levels and a 16-warp chain, then in fp64
  across CTAs and a final cast to fp32: an fp32 sum S of K = 8·chunks + 22 steps over terms s_i with errors δ_i is within
  Σδ_i + K·u·Σ|s_i| of the exact one.  Σp·t is reported as (Σp + Σt − Σd)/2, so its error is half the sum of theirs.
  cel = Σd / (Σp + Σt + eps) carries the relative errors of both sums; bce, total follow (plus u for each fp32 cast).
* gradient g = kb·(p − t) + p(1 − p)·(α(1 − 2t) + β), kb = grad_scale·w_bce (/n), α = grad_scale·w_cel/den,
  β = −α·num/den: p's relative error ε(x); p − t and 1 − p are fp32 subtractions, as torch's own sigmoid(x) − t in the
  reference's autograd, so each carries one fp32 ulp of 1 (2⁻²³) absolute besides p's error — relative to a small
  1 − p that is the one loss of precision the gradient keeps, the reference's own; 2⁻²² for kb and its product, u for
  the product p(1 − p); for α and β the rounding to fp32 plus the relative errors of den (α, and twice in β) and of
  num (β) from the bounds above; then u for the product and the final fused add.  Held to one ulp of the output dtype
  at |ref| (half for the final rounding, half for a value next to a rounding boundary) plus that fp32 slack.

In the confident regime (logits agreeing with the mask at |x| of 4–6, 10–12, 14–16, and an all-background mask with
logits ≤ −25, where eps dominates the denominator) the yardstick is the reference's own fp32 error: CEL as
(p − p·t).sum() + (t − p·t).sum() over p.sum() + t.sum() + eps and BCE as F.binary_cross_entropy_with_logits, both in
fp32 with torch on this GPU, measured against fp64.  The kernel must stay within 4× that error plus 2·10⁻⁶ relative.
"""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import loss as oloss
from oracle import loss_geometry as geo

pytestmark = pytest.mark.gpu

TORCH_DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}
MANT = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}
EMIN = {torch.float32: -126, torch.bfloat16: -126, torch.float16: -14}
U = 2.0 ** -24
CASES = geo.covering_cases()
RAN: dict = {}              # case id → cells of the regime table it reached on this device


def _device():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    return p.multi_processor_count, p.shared_memory_per_block_optin


def ulp(ref, dtype):
    """spacing of `dtype` at |ref| (fp64 tensor), subnormal spacing below the smallest normal"""
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** EMIN[dtype])))
    return torch.exp2(e - MANT[dtype])


def same_bits(a, b):
    ity = {4: torch.int32, 2: torch.int16}[a.element_size()]
    return a.dtype == b.dtype and torch.equal(a.contiguous().view(ity), b.contiguous().view(ity))


def run(x, t, **kw):
    from distributed_sod_project_b200.loss import bce_cel_fwd_bwd
    scalars, grad = bce_cel_fwd_bwd(x, t, **kw)
    torch.cuda.synchronize()
    return scalars, grad


def reference(x, t, reduction, w_bce, w_cel, grad_scale, eps):
    """oracle/loss.py bce_cel_fwd_bwd in fp64 on the GPU (q = 1 − p and d = p(1 − t) + t·q formed without cancellation),
    with the per-element quantities the bounds need"""
    x, t = x.double().ravel(), t.double().ravel()
    n = x.numel()
    e = torch.exp(-x.abs())
    p = torch.where(x >= 0, 1.0 / (1.0 + e), e / (1.0 + e))
    q = torch.where(x >= 0, e / (1.0 + e), 1.0 / (1.0 + e))
    b = x.clamp_min(0.0) - x * t + torch.log1p(e)
    d = p * (1.0 - t) + t * q
    sp, st, sd, bs = p.sum(), t.sum(), d.sum(), b.sum()
    den = sp + st + eps
    kb = grad_scale * w_bce * ((1.0 / n) if reduction == "mean" else 1.0)
    alpha = grad_scale * w_cel / den
    beta = -alpha * sd / den
    A = alpha * (1.0 - 2.0 * t) + beta
    grad = kb * (p - t) + p * q * A
    bce = bs / n if reduction == "mean" else bs
    cel = sd / den
    return dict(x=x, t=t, p=p, q=q, b=b, d=d, sp=sp, st=st, sd=sd, bce_sum=bs, den=den, bce=bce, cel=cel,
                total=w_bce * bce + w_cel * cel, kb=kb, alpha=alpha, beta=beta, A=A, grad=grad, n=n,
                reduction=reduction, w_bce=w_bce, w_cel=w_cel)


def eps_p(x):
    """relative error bound of the kernel's p and q at logit x (module docstring)"""
    return (16.0 + 2.0 * x.abs()) * U


def scalar_bounds(r, chunks):
    """absolute error bounds of the kernel's eight scalars (module docstring)"""
    K = (8 * chunks + 22) * U
    x, t, p, d, b = r["x"], r["t"], r["p"], r["d"], r["b"]
    ep = eps_p(x)
    dsp = float((ep * p).sum()) + K * float(r["sp"])
    dst = K * float(r["st"])
    dsd = float(((ep + 3 * U) * d).sum()) + K * float(r["sd"])
    lg = torch.log1p(torch.exp(-x.abs()))
    dbs = float((U * (2 * (x * t).abs() + 3 * b.abs()) + 1.5 * (ep + 2 * U) * lg).sum()) + K * float(b.abs().sum())
    rel_den = (dsp + dst) / float(r["den"])
    rel_num = dsd / max(float(r["sd"]), 1e-300)
    cel = float(r["cel"])
    dcel = cel * (rel_num + rel_den) + U * cel
    dbce = (dbs / r["n"] if r["reduction"] == "mean" else dbs) + U * abs(float(r["bce"]))
    dtotal = r["w_bce"] * dbce + r["w_cel"] * dcel + U * abs(float(r["total"]))
    return dict(rel_den=rel_den, rel_num=rel_num, bounds=[
        dbce, dcel, dtotal, dsp + U * float(r["sp"]), dst + U * float(r["st"]),
        0.5 * (dsp + dst + dsd) + U * abs(float(r["sp"] + r["st"] - r["sd"])) / 2, dbs + U * float(r["bce_sum"]), 0.0])


def grad_slack(r, rel_den, rel_num):
    """the fp32 slack of the kernel's gradient arithmetic (module docstring)"""
    x, t, p, q = r["x"], r["t"], r["p"], r["q"]
    ep = eps_p(x)
    kb, alpha, beta, A = abs(r["kb"]), r["alpha"], r["beta"], r["A"]
    pq = p * q
    one_minus_p = p * (ep * p + 2.0 ** -23)                  # p's error and one ulp of 1 in 1 − p, times p
    bce_part = kb * (ep * p + 2.0 ** -23 + 2.0 ** -22 * (p - t).abs())
    cel_part = ((ep + U) * pq + one_minus_p) * A.abs() + pq * ((alpha * (1.0 - 2.0 * t)).abs() * (2.0 ** -23 + rel_den)
                                                             + beta.abs() * (2.0 ** -23 + rel_num + 2 * rel_den))
    return bce_part + cel_part + 2 * U * (kb * (p - t).abs() + (pq * A).abs())


def assert_within(got, ref, tol, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= tol)                     # NaN fails
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} elements off, worst "
                                 f"{float((err / tol).nan_to_num(float('inf')).max()):.3g}x the tolerance (first at "
                                 f"{int(bad.nonzero()[0])}: got {float(got.double()[bad][0])}, ref {float(ref[bad][0])})")


def check_against_reference(scalars, grad, r, chunks, dtype, what):
    sb = scalar_bounds(r, chunks)
    s = scalars.double().cpu().numpy()
    b = sb["bounds"]
    want = [float(r["bce"]), float(r["cel"]), float(r["total"]), float(r["sp"]), float(r["st"]),
            float((r["sp"] + r["st"] - r["sd"]) / 2), float(r["bce_sum"]), float(np.float32(r["n"]))]
    names = ("bce", "cel", "total", "sum_p", "sum_t", "sum_pt", "bce_sum", "n")
    for i, name in enumerate(names):
        assert abs(s[i] - want[i]) <= b[i], f"{what}: {name} {s[i]!r} vs {want[i]!r} (bound {b[i]:.3g})"
    tol = ulp(r["grad"], dtype) + grad_slack(r, sb["rel_den"], sb["rel_num"])
    assert_within(grad.ravel(), r["grad"], tol, f"{what}: gradient")


def case_inputs(case, n):
    """logits (randn·3 in T) and a soft k/255 or binary mask in its dtype, seeded by the case id"""
    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(case.id.encode()))
    x = (torch.randn(n, generator=gen, device="cuda") * 3.0).to(TORCH_DT[case.tx])
    if case.spec % 3 == 0:
        t = (torch.rand(n, generator=gen, device="cuda") < 0.3).float()
    else:
        t = torch.randint(0, 256, (n,), generator=gen, device="cuda").float() / 255.0
    return x, t.to(TORCH_DT[case.tm])


def case_settings(case, x, t):
    """weights, reduction, eps and grad_scale of a case: w_bce ≠ w_cel; the reduction alternates over dtype pairs"""
    k = geo.PAIRS.index((case.tx, case.tm))
    j = case.spec
    w_bce, w_cel = ((0.75, 1.5), (1.25, 0.5))[j % 2]
    reduction = ("mean", "sum")[(j + k) % 2]
    eps = (1e-6, 0.03 * x.numel())[(j // 2 + k) % 2]
    gs = 8.0
    if case.tx == "float16":
        gs = 65536.0
        peak = float(reference(x, t, reduction, w_bce, w_cel, 1.0, eps)["grad"].abs().max())
        while gs > 1.0 and peak * gs > 2.0 ** 14:
            gs /= 2
    return dict(reduction=reduction, w_bce=w_bce, w_cel=w_cel, grad_scale=gs, eps=eps)


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_loss_regime_parity(case):
    from distributed_sod_project_b200 import _lib
    sm, smem = _device()
    n, g = geo.resolve(case, sm, smem)
    assert g is not None, f"{case.id}: regime {geo.SPECS[case.spec]} is unreachable on {sm} SMs / {smem} B"
    sx, smb = geo.DTYPE_BYTES[case.tx], geo.DTYPE_BYTES[case.tm]
    x, t = case_inputs(case, n)
    kw = case_settings(case, x, t)
    r = reference(x, t, **kw)
    scalars, grad = run(x, t, mode=case.mode, **kw)
    assert grad.dtype == x.dtype
    check_against_reference(scalars, grad, r, max(g.chunks), x.dtype, case.id)

    # two identical launches: identical bytes
    s2, g2 = run(x, t, mode=case.mode, **kw)
    assert same_bits(scalars, s2) and same_bits(grad, g2), "two identical launches differ"

    # mode 1 refuses exactly where the model says the slice does not fit the resident kernel
    g1 = geo.launch(n, sx, smb, 1, sm, smem)
    if g1.kernel == "refused":
        with pytest.raises(_lib.SodError):
            run(x, t, mode=1, **kw)
    else:
        s1, gr1 = run(x, t, mode=1, **kw)
        s0, gr0 = (scalars, grad) if case.mode == 0 else run(x, t, mode=0, **kw)
        assert same_bits(s1, s0) and same_bits(gr1, gr0)

    # where mode 0 runs the resident kernel, the streamed kernel (mode 2) computes the same bits
    if geo.launch(n, sx, smb, 0, sm, smem).kernel == "resident":
        s0, gr0 = (scalars, grad) if case.mode == 0 else run(x, t, mode=0, **kw)
        s2, gr2 = (scalars, grad) if case.mode == 2 else run(x, t, mode=2, **kw)
        assert same_bits(s0, s2), f"scalars: resident {s0.tolist()} vs streamed {s2.tolist()}"
        assert same_bits(gr0, gr2), f"{int((gr0 != gr2).sum())} gradients differ between the resident and streamed kernels"
    RAN[case.id] = geo.cells(case, g, sm)


def test_every_regime_cell_ran_on_this_device():
    """every reachable cell (kernel instance × regime axis value) was reached by a passing case"""
    if not RAN:
        pytest.skip("the regime cases did not run in this session")
    missing_cases = [c.id for c in CASES if c.id not in RAN]
    assert not missing_cases, f"{len(missing_cases)} regime cases did not pass: {missing_cases[:5]}"
    missing = geo.required_cells() - set().union(*RAN.values())
    assert not missing, sorted(missing)


def test_fp64_reference_matches_the_oracle():
    """the GPU fp64 reference above is oracle/loss.py's arithmetic"""
    gen = torch.Generator().manual_seed(11)
    x = torch.randn(3000, generator=gen, dtype=torch.float64) * 4
    t = torch.randint(0, 256, (3000,), generator=gen).double() / 255
    for red in ("mean", "sum"):
        want = oloss.bce_cel_fwd_bwd(x.numpy(), t.numpy(), reduction=red, w_bce=0.75, w_cel=1.5, grad_scale=8.0, eps=0.5)
        r = reference(x.cuda(), t.cuda(), red, 0.75, 1.5, 8.0, 0.5)
        for k in ("bce", "cel", "total"):
            assert float(r[k]) == pytest.approx(want[k], rel=1e-12)
        assert float(r["sp"]) == pytest.approx(want["sum_p"], rel=1e-12)
        assert float((r["sp"] + r["st"] - r["sd"]) / 2) == pytest.approx(want["sum_pt"], rel=1e-12)
        np.testing.assert_allclose(r["grad"].cpu().numpy(), want["grad"], rtol=1e-10, atol=1e-15)


# ---- confident predictions: p ≈ t, where Σp + Σt − 2Σp·t cancels -------------------------------------------------------
CONFIDENT = [(dt, lo, edges) for dt in ("float32", "bfloat16", "float16") for lo in (4.0, 10.0, 14.0)
             for edges in ("binary", "soft")] + [("float32", -25.0, "background"), ("bfloat16", -25.0, "background")]


def confident_inputs(dtype, lo, edges, shape=(16, 1, 320, 320)):
    """30 % foreground; logits of the mask's sign at |x| in [lo, lo + 2].  soft: 2 % of the pixels are edge pixels with
    t = k/255 and the logit that predicts t.  background: t = 0 and x in [lo − 3, lo]"""
    gen = torch.Generator(device="cuda").manual_seed(int(abs(lo)) * 7 + len(edges))
    mag = torch.rand(shape, generator=gen, device="cuda") * 2.0
    if edges == "background":
        t = torch.zeros(shape, device="cuda")
        x = lo - 1.5 * mag
    else:
        t = (torch.rand(shape, generator=gen, device="cuda") < 0.3).float()
        x = torch.where(t > 0, 1.0, -1.0) * (lo + mag)
        if edges == "soft":
            edge = torch.rand(shape, generator=gen, device="cuda") < 0.02
            k = torch.randint(1, 255, shape, generator=gen, device="cuda").float()
            t = torch.where(edge, k / 255.0, t)
            x = torch.where(edge, torch.log(t / (1.0 - t)).clamp(-lo - 2.0, lo + 2.0), x)
    return x.to(TORCH_DT[dtype]), t


@pytest.mark.parametrize("dtype, lo, edges", CONFIDENT, ids=[f"{d}-{lo:g}-{e}" for d, lo, e in CONFIDENT])
def test_confident_predictions(dtype, lo, edges):
    x, t = confident_inputs(dtype, lo, edges)
    gs = 65536.0 if dtype == "float16" else 1.0
    kw = dict(reduction="mean", w_bce=1.0, w_cel=1.0, grad_scale=gs, eps=1e-6)
    r = reference(x, t, **kw)
    scalars, grad = run(x, t, **kw)
    s = scalars.double().cpu()
    # the reference's own fp32 arithmetic on this GPU
    xf = x.float()
    p = torch.sigmoid(xf)
    cel32 = float(((p - p * t).sum() + (t - p * t).sum()) / (p.sum() + t.sum() + 1e-6))
    bce32 = float(F.binary_cross_entropy_with_logits(xf, t))
    cel, bce = float(r["cel"]), float(r["bce"])
    err = dict(cel=abs(float(s[1]) - cel) / cel, bce=abs(float(s[0]) - bce) / bce)
    ref32 = dict(cel=abs(cel32 - cel) / cel, bce=abs(bce32 - bce) / bce)
    print(f"\n{dtype} |x|>={abs(lo):g} {edges}: CEL {cel:.6g} rel err kernel {err['cel']:.2e} torch-fp32 {ref32['cel']:.2e}; "
          f"BCE {bce:.6g} kernel {err['bce']:.2e} torch-fp32 {ref32['bce']:.2e}")
    for k in ("cel", "bce"):
        assert err[k] <= 4 * ref32[k] + 2e-6, f"{k}: kernel relative error {err[k]:.3g}, torch fp32 {ref32[k]:.3g}"
    sb = scalar_bounds(r, 8)            # the 320² bs-16 tensor has at most 4 chunks per CTA on ≥ 100 SMs
    tol = ulp(r["grad"], x.dtype) + grad_slack(r, sb["rel_den"], sb["rel_num"])
    assert_within(grad.ravel(), r["grad"], tol, "gradient")


# ---- sod_scale_by_device_scalar: the backward of a loss whose upstream gradient is not 1 -------------------------------
def _scale_sizes():
    sm, _ = _device()
    one_pass = 4 * sm * 256 * 8
    return list(range(1, 9)) + [8 * 1000 + 3, 8 * 4096 + 5, 2 * one_pass + 8 * 77 + 6, one_pass]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_scale_by_device_scalar_is_exact(dtype):
    """g ← (g·s) in fp32 rounded once to T: bit for bit against torch, for every size class of the kernel (the scalar
    tail alone, a whole packet, packets + tail, one and more than one grid-stride pass)"""
    from distributed_sod_project_b200 import _lib
    gen = torch.Generator(device="cuda").manual_seed(21)
    s = torch.tensor([0.3711], device="cuda")
    for n in _scale_sizes():
        buf = (torch.randn(n + 8, generator=gen, device="cuda") * 100).to(dtype)
        before = buf.clone()
        rc = _lib.lib().sod_scale_by_device_scalar(buf.data_ptr(), _lib.dtype_code(dtype), n, s.data_ptr(), _lib.stream_ptr())
        _lib.check(rc, "sod_scale_by_device_scalar")
        torch.cuda.synchronize()
        want = (before[:n].float() * s).to(dtype)
        assert same_bits(buf[:n], want), f"n={n}: {int((buf[:n] != want).sum())} elements differ"
        assert same_bits(buf[n:], before[n:]), f"n={n}: elements past the end changed"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_scaled_upstream_through_autograd(dtype):
    """logits and mask of one 16-bit dtype, loss·c backpropagated: the gradient is the kernel's own gradient times c,
    rounded once, and within 3 ulp + c·(fp32 slack) of the fp64 gradient times c"""
    from distributed_sod_project_b200.loss import FusedBCECEL
    gen = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.randn(3, 1, 37, 41, generator=gen, device="cuda") * 3).to(dtype).requires_grad_(True)
    t = (torch.randint(0, 256, x.shape, generator=gen, device="cuda").float() / 255).to(dtype)
    c = 0.3711
    (FusedBCECEL(w_bce=0.75, w_cel=1.5)(x, t) * c).backward()
    _, unscaled = run(x.detach(), t, w_bce=0.75, w_cel=1.5)
    want = (unscaled.float() * torch.tensor(c, device="cuda")).to(dtype)
    assert same_bits(x.grad, want)
    r = reference(x.detach(), t, "mean", 0.75, 1.5, 1.0, 1e-6)
    sb = scalar_bounds(r, 1)
    ref = r["grad"] * c
    assert_within(x.grad.ravel(), ref, 3 * ulp(ref, dtype) + c * grad_slack(r, sb["rel_den"], sb["rel_num"]), "scaled gradient")
