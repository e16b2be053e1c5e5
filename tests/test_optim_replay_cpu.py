"""oracle/optim_replay.py on the CPU: the fp32 FMA emulation against exact rational arithmetic, the recovered Adam β and
the pow margin of every (β, t) the GPU tests use, the replay against torch.optim.SGD / Adam, and the replay's power to
tell a fused multiply-add from a separate multiply and add."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import optim_replay as rp

F32_MAX = float(np.finfo(np.float32).max)


def _round_f32(q: Fraction, zero_sign: float) -> float:
    """the exact rational q rounded to nearest even in fp32 (subnormals and overflow included)"""
    if q == 0:
        return math.copysign(0.0, zero_sign)
    s = -1.0 if q < 0 else 1.0
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    e = max(e, -126)
    ulp = Fraction(2) ** (e - 23)
    m = a / ulp
    k = m.numerator // m.denominator
    r = m - k
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and k % 2 == 1):
        k += 1
    v = k * ulp
    if v >= Fraction(2) ** 128:
        return s * math.inf
    return s * float(v)


def _fma_exact(a, b, c):
    a, b, c = float(a), float(b), float(c)
    if not all(math.isfinite(x) for x in (a, b, c)):      # IEEE: inf·0, inf − inf and NaN give NaN, else ±inf
        with np.errstate(invalid="ignore"):
            return float(np.float64(a) * np.float64(b) + np.float64(c))
    prod = Fraction(a) * Fraction(b)
    exact = prod + Fraction(c)
    # an exact zero is −0 only when both addends are −0 (round to nearest)
    pz = math.copysign(1.0, a) * math.copysign(1.0, b)
    zs = -1.0 if (prod == 0 and pz < 0 and c == 0 and math.copysign(1.0, c) < 0) else 1.0
    return _round_f32(exact, zs)


def _bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def _check(a, b, c):
    got = rp.fma32(np.array(a, np.float32), np.array(b, np.float32), np.array(c, np.float32))
    for x, y, z, g in zip(np.atleast_1d(a), np.atleast_1d(b), np.atleast_1d(c), np.atleast_1d(got)):
        want = _fma_exact(np.float32(x), np.float32(y), np.float32(z))
        if math.isnan(want):
            assert math.isnan(g), (x, y, z)
        else:
            assert _bits(float(g)) == _bits(want), (float(x), float(y), float(z), float(g), want)


def test_fma_emulation_is_exact_on_random_triples():
    rng = np.random.default_rng(0)
    n = 100_000
    def spread():
        return (rng.standard_normal(n) * np.exp2(rng.integers(-40, 40, n))).astype(np.float32)
    a, b = spread(), spread()
    c = np.where(rng.random(n) < 0.5, -(a.astype(np.float64) * b * (1 + rng.standard_normal(n) * 2 ** -20)), spread())
    _check(a, b, c.astype(np.float32))


def test_fma_emulation_on_constructed_cases():
    one_ulp = float(np.float32(2.0 ** -23))
    cases = [
        (1.0 + one_ulp, 1.0 - one_ulp, -1.0),                    # exact −2⁻⁴⁶: no rounding, product rounding would give 0
        (1.0 + 2 ** -12, 1.0 + 2 ** -12, 0.0),                  # 1 + 2⁻¹¹ + 2⁻²⁴: exact halfway, ties to even
        (1.0 + 2 ** -12 + one_ulp, 1.0 + 2 ** -12, 0.0),        # just past halfway
        (1.0 + 2 ** -12, 1.0 - 2 ** -12, -1.0),                  # cancellation to −2⁻²⁴
        (3.0, 1.0 / 3.0, -1.0),                                   # cancellation to a tiny residual
        (2.0 ** -75, 2.0 ** -75, 0.0),                            # 2⁻¹⁵⁰: halfway to the smallest subnormal, ties to 0
        (2.0 ** -75, 1.5 * 2.0 ** -75, 0.0),                      # rounds up to 2⁻¹⁴⁹
        (2.0 ** -70, 2.0 ** -70, 2.0 ** -130),                    # subnormal result
        (1.0 + one_ulp, 2.0 ** -126, -2.0 ** -126),               # cancellation to a subnormal
        (2.0, 1.0, -2.0),                                          # exact 0 → +0
        (-0.0, 1.0, -0.0), (0.0, -1.0, -0.0), (-0.0, 1.0, 0.0),   # signs of zero
        (F32_MAX, 1.0, 0.0), (F32_MAX, 1.0 + one_ulp, 0.0),       # FLT_MAX and overflow
        (2.0 ** 64, 2.0 ** 64, -F32_MAX), (F32_MAX, 2.0, -F32_MAX),
        (2.0 ** 127, 1.0, 2.0 ** 103), (2.0 ** 127, 1.0, 2.0 ** 103 * (1 - 2 ** -20)),   # overflow threshold, both sides
        (math.inf, 1.0, 1.0), (math.inf, 0.0, 1.0), (math.inf, 1.0, -math.inf), (1.0, 1.0, math.nan),
        (-math.inf, -2.0, 5.0), (F32_MAX, F32_MAX, -math.inf),
    ]
    for a, b, c in cases:
        _check(np.float32(a), np.float32(b), np.float32(c))
    _check(*(np.array(x, np.float32) for x in zip(*cases)))


def test_split_variant_differs_where_the_product_rounds():
    assert rp.fma32(1.0 + 2 ** -23, 1.0 - 2 ** -23, -1.0) == np.float32(-(2.0 ** -46))
    assert rp.fma32_split(1.0 + 2 ** -23, 1.0 - 2 ** -23, -1.0) == 0.0


# ---- Adam's scalars ---------------------------------------------------------------------------------------------------
BETAS = [(0.9, 0.999), (0.8, 0.99), (0.5, 0.75), (0.0, 0.0), (0.95, 0.9999)]
STEP_COUNTS = [0, 1, 2, 3, 4, 5, 6, 7, 9, 10_000, 1_000_000]
# 3e-3, 5e-3 and 1e-2 are left out on purpose: at t = 1 with β1 = 0.9, fp32(lr)/0.1 lands within a few double ulps of an
# fp32 tie, so their step_size depends on the last bit of pow(0.9, 1) (adam_scalars_stable is False for them)
LRS = [0.0, 1e-3, 2e-3, 0.05, 0.1]


def test_recovered_beta_is_numpys_shortest_repr():
    for b1, b2 in BETAS:
        for b in (b1, b2):
            shortest = float(np.format_float_positional(np.float32(b), unique=True))
            assert rp.adam_beta(np.float32(b)) == shortest == b
    rng = np.random.default_rng(1)
    for b in rng.random(2000).astype(np.float32):
        assert rp.adam_beta(b) == float(np.format_float_scientific(b, unique=True))


def test_bias_corrections_clear_the_pow_margin():
    """the assumption the bit-exact GPU comparison rests on (module docstring of oracle/optim_replay.py)"""
    bad = [(lr, b, t) for lr in LRS for b in BETAS for t in STEP_COUNTS
           if not rp.adam_scalars_stable(lr, b[0], b[1], t)]
    assert bad == []
    assert not rp.adam_scalars_stable(3e-3, 0.9, 0.999, 0)          # the margin check does see a knife edge


# ---- the replay against torch's optimizers ----------------------------------------------------------------------------
U = 2.0 ** -24


def _state(n, seed):
    rng = np.random.default_rng(seed)
    p = (rng.standard_normal(n) * np.exp2(rng.integers(-4, 4, n))).astype(np.float32)
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-6, 2, n))).astype(np.float32)
    g = (rng.standard_normal(n) * np.exp2(rng.integers(-8, 4, n))).astype(np.float32)
    return p, v, g


@pytest.mark.parametrize("nesterov", [False, True])
def test_sgd_replay_matches_torch_sgd(nesterov):
    n, lr, wd, mu = 200_000, float(np.float32(0.05)), float(np.float32(5e-4)), float(np.float32(0.9))
    p0, v0, g0 = _state(n, 2)
    p, v = rp.sgd_update(p0, v0, g0, lr, wd, mu, nesterov)
    tp = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.SGD([tp], lr=lr, momentum=mu, weight_decay=wd, nesterov=nesterov, foreach=False)
    tp.grad = torch.tensor(g0)
    opt.state[tp]["momentum_buffer"] = torch.tensor(v0)
    opt.step()
    tv = opt.state[tp]["momentum_buffer"].numpy()
    a = np.abs
    mv = mu * a(v0) + a(g0) + wd * a(p0)                           # every term of v' and of d, in magnitude
    md = mv * (1 + mu) if nesterov else mv
    assert np.all(a(v.astype(np.float64) - tv) <= 4 * U * mv)
    assert np.all(a(p.astype(np.float64) - tp.detach().numpy()) <= 8 * U * (a(p0) + lr * md))


def test_adam_replay_matches_torch_adam():
    n = 200_000
    lr, wd, b1, b2, eps = (float(np.float32(x)) for x in (1e-3, 5e-4, 0.9, 0.999, 1e-8))
    rng = np.random.default_rng(3)
    p0, m0, g0 = _state(n, 3)
    v0 = (np.abs(rng.standard_normal(n)) * np.exp2(rng.integers(-20, 0, n))).astype(np.float32)
    for step0 in (0, 9):
        ss, bc = rp.adam_scalars(lr, b1, b2, step0)
        p, m, v = rp.adam_update(p0, m0, v0, g0, wd, np.float32(1 - 0.9), np.float32(b2), np.float32(1 - 0.999), ss, bc, eps)
        tp = torch.tensor(p0, requires_grad=True)
        opt = torch.optim.Adam([tp], lr=lr, betas=(0.9, 0.999), eps=eps, weight_decay=wd, foreach=False)
        tp.grad = torch.tensor(g0)
        opt.state[tp].update(step=torch.tensor(float(step0)), exp_avg=torch.tensor(m0), exp_avg_sq=torch.tensor(v0))
        opt.step()
        tm, tv = opt.state[tp]["exp_avg"].numpy(), opt.state[tp]["exp_avg_sq"].numpy()
        a = np.abs
        gg = a(g0.astype(np.float64)) + wd * a(p0)
        assert np.all(a(m.astype(np.float64) - tm) <= 4 * U * (a(m0) + gg))
        assert np.all(a(v.astype(np.float64) - tv) <= 6 * U * (b2 * a(v0) + (1 - b2) * gg * gg))
        den = np.sqrt(v.astype(np.float64)) / float(bc) + eps
        upd = float(ss) * a(m.astype(np.float64)) / den
        assert np.all(a(p.astype(np.float64) - tp.detach().numpy()) <= 16 * U * (a(p0) + upd))


def test_replay_tells_a_fused_update_from_a_split_one():
    """one SGD step and one Adam step on the random tier, FMAs fused against split: the share of elements that differ
    is what a kernel that lost its FMAs would show (measured: 28 % of the elements for SGD, 17 % for Adam)"""
    n = 200_000
    p0, v0, g0 = _state(n, 4)
    a = rp.sgd_update(p0, v0, g0, 0.05, 5e-4, 0.9, False)
    b = rp.sgd_update(p0, v0, g0, 0.05, 5e-4, 0.9, False, fma=rp.fma32_split)
    frac_sgd = float(np.mean((a[0] != b[0]) | (a[1] != b[1])))
    ss, bc = rp.adam_scalars(1e-3, 0.9, 0.999, 0)
    v1 = np.abs(v0)
    args = (5e-4, np.float32(0.1), np.float32(0.999), np.float32(0.001), ss, bc, np.float32(1e-8))
    c = rp.adam_update(p0, v0, v1, g0, *args)
    d = rp.adam_update(p0, v0, v1, g0, *args, fma=rp.fma32_split)
    frac_adam = float(np.mean((c[0] != d[0]) | (c[1] != d[1]) | (c[2] != d[2])))
    print(f"elements that differ: SGD {frac_sgd:.3f}, Adam {frac_adam:.3f}")
    assert frac_sgd > 0.2 and frac_adam > 0.1


def test_scaler_rules():
    assert rp.scaler_next(2.0 ** 23, 0, 2, False) == (2.0 ** 23, 1)
    assert rp.scaler_next(2.0 ** 23, 0, 1, False) == (2.0 ** 24, 1)
    assert rp.scaler_next(2.0 ** 24, 0, 1, False) == (2.0 ** 24, 1)
    assert rp.scaler_next(2.0 ** 40, 0, 1, False) == (2.0 ** 24, 1)             # growth applies the cap
    assert rp.scaler_next(2.0 ** 40, 5, 1, True) == (2.0 ** 39, 0)              # an overflow only halves
    assert rp.scaler_next(1.5, 3, 2, True) == (1.0, 0) and rp.scaler_next(1.0, 0, 0, False) == (1.0, 1)
