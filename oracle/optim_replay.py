"""ORACLE (test infrastructure only): the bits of the world-1 optimizer step of csrc/sgd.cu, replayed in numpy fp32.

`local_step_kernel` forms each element's update with explicit `fmaf` and with plain IEEE fp32 `*`, `+`, `-`, `sqrtf`
and `/` elsewhere (the library is built without fast-math: no flush to zero, IEEE division and square root, and the
source gives the compiler no multiply-add to contract).  This module restates that arithmetic in the same operation
order, so a correct kernel equals it bit for bit:

    gradient  g = g32 + float(g16)   (g16 alone on SOD_SEG_GRAD16 ranges, g32 alone without a 16-bit buffer)
              g = g × inv_scale      (scaler entry points: inv_scale = 1.0f / scale, an fp32 division)
    SGD       g' = fma(wd, p, g) ;  v = fma(mu, v, g') ;  d = fma(mu, v, g') if Nesterov else v ;  p = fma(−lr, d, p)
    Adam      g' = fma(wd, p, g) ;  m = fma(w1, g' − m, m) ;  v = fma(c2·g', g', v·β2) ;
              p = fma(−step_size, m / (sqrt(v) / bc2_sqrt + eps), p)
    shadow    the new p rounded to nearest even in bf16 or fp16

`fma32` emulates fp32's fused multiply-add exactly: the product of two fp32 values is exact in float64; a TwoSum with
the addend gives the float64 sum s and its error e exactly; when e ≠ 0, s is moved to its odd neighbour on the side of
e (round to odd at 53 bits), and the cast to float32 then rounds correctly, since 53 ≥ 24 + 2 bits — also for subnormal
results and at overflow.  Non-finite operands follow IEEE through the plain float64 expression.
tests/test_optim_replay_cpu.py checks it against exact `fractions.Fraction` arithmetic.

Adam's scalars.  The kernel recovers β as the shortest decimal that rounds to the segment's fp32 β (`adam_beta`, as
`%.*g` with 1 … 9 digits computes it), so w1 = fp32(1 − β1) and c2 = fp32(1 − β2) come from the same double as torch's
Python floats; then, once per CTA in double, step_size = fp32(lr / (1 − β1^t)) and bc2_sqrt = fp32(sqrt(1 − β2^t)),
t = step + 1.  The device's double `pow` is not guaranteed correctly rounded (CUDA documents a 2-ulp bound), so a
bit-exact comparison rests on one ASSUMPTION: for every (β, t) a test uses, moving the double β^t by up to
POW_MARGIN_ULPS = 4 double ulps either way does not change either fp32 scalar.  `adam_scalars_stable` checks that for a
given (lr, β1, β2, t); tests/test_optim_replay_cpu.py asserts it for every pair the GPU tests use.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
POW_MARGIN_ULPS = 4


# ---- fp32 fused multiply-add ----------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays (or scalars), correctly rounded"""
    a, b, c = (np.asarray(x, dtype=np.float32).astype(np.float64) for x in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        prod = a * b                                    # exact: 24 + 24 bits
        s = prod + c
        bp = s - prod
        e = (prod - (s - bp)) + (c - bp)                # TwoSum: s + e == prod + c exactly
        finite = np.isfinite(s) & np.isfinite(e)
        even = (s.view(np.uint64) & np.uint64(1)) == 0
        fix = finite & (e != 0) & even
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(np.float32)


def fma32_split(a, b, c):
    """the same expression with the product rounded on its own: fp32(fp32(a·b) + c)"""
    a, b, c = (np.asarray(x, dtype=np.float32) for x in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        return (a * b) + c


# ---- scalars --------------------------------------------------------------------------------------------------------
def adam_beta(b) -> float:
    """the shortest decimal (1 … 9 significant digits) whose double rounds to the fp32 value b, as csrc/sgd.cu finds it"""
    bf = F32(b)
    for digits in range(1, 10):
        d = float("%.*g" % (digits, float(bf)))
        if F32(d) == bf:
            return d
    return float(bf)


def _adam_scalars_from_pow(lr32, p1, p2):
    step_size = F32(float(lr32) / (1.0 - p1))
    bc2_sqrt = F32(np.sqrt(1.0 - p2))
    return step_size, bc2_sqrt


def adam_scalars(lr, beta1, beta2, step):
    """(step_size, bc2_sqrt) as fp32, for a segment of fp32 lr / β1 / β2 that has taken `step` steps"""
    t = float(step) + 1.0
    return _adam_scalars_from_pow(F32(lr), adam_beta(beta1) ** t, adam_beta(beta2) ** t)


def adam_scalars_stable(lr, beta1, beta2, step, ulps=POW_MARGIN_ULPS) -> bool:
    """True when β1^t and β2^t may each be off by up to `ulps` double ulps without changing adam_scalars"""
    t = float(step) + 1.0
    want = adam_scalars(lr, beta1, beta2, step)
    for base, other, k in ((adam_beta(beta1) ** t, adam_beta(beta2) ** t, 0), (adam_beta(beta2) ** t, adam_beta(beta1) ** t, 1)):
        for direction in (-np.inf, np.inf):
            x = base
            for _ in range(ulps):
                x = float(np.nextafter(x, direction))
                got = _adam_scalars_from_pow(F32(lr), *((x, other) if k == 0 else (other, x)))
                if got[0] != want[0] or got[1] != want[1]:
                    return False
    return True


# ---- per-element rules ----------------------------------------------------------------------------------------------
def sgd_update(p, v, g, lr, wd, mu, nesterov, fma=fma32):
    """sgd_update of csrc/sgd.cu on fp32 arrays; lr / wd / mu / nesterov broadcast.  Returns (p, v)."""
    lr, wd, mu = F32(lr) if np.isscalar(lr) else lr, F32(wd) if np.isscalar(wd) else wd, F32(mu) if np.isscalar(mu) else mu
    gg = fma(wd, p, g)
    v = fma(mu, v, gg)
    d = np.where(nesterov, fma(mu, v, gg), v)
    p = fma(-np.asarray(lr, np.float32), d, p)
    return p, v


def adam_update(p, m, v, g, wd, w1, b2, c2, step_size, bc2_sqrt, eps, fma=fma32):
    """adam_update1 of csrc/sgd.cu on fp32 arrays; the per-segment scalars broadcast.  Returns (p, m, v)."""
    f = lambda x: np.asarray(x, np.float32)            # noqa: E731
    wd, w1, b2, c2, step_size, bc2_sqrt, eps = (f(x) for x in (wd, w1, b2, c2, step_size, bc2_sqrt, eps))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore", under="ignore"):
        gg = fma(wd, p, g)
        m = fma(w1, gg - m, m)
        v = fma(c2 * gg, gg, v * b2)
        denom = np.sqrt(v) / bc2_sqrt + eps
        p = fma(-step_size, m / denom, p)
    return p, m, v


def round16(x, dtype):
    """fp32 → bf16 / fp16 with round-to-nearest-even, as float32 values ("bfloat16" or "float16")"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    return t.to(getattr(torch, dtype)).float().numpy()


# ---- one world-1 launch over flat buffers ---------------------------------------------------------------------------
FROZEN, GRAD16, NESTEROV = 1, 2, 4         # SOD_SEG_* of include/sod_b200.h


def step(rule, p, state, g32, g16, segs, *, inv_scale=1.0, scale=None, skip=False, zero_grad=True, steps=None,
         fma=fma32):
    """What one `sod_sgd_momentum` / `sod_adam` (or `*_scaler`) launch leaves in the flat buffers.

    rule: "sgd" or "adam"; p, g32: fp32 [n]; state: [v] or [m, v]; g16: the 16-bit gradient as fp32 values, or None;
    segs: dicts with begin, end (elements), lr, wd, flags and mu (SGD) or beta1, beta2, eps (Adam); `scale` (a scaler
    launch) replaces inv_scale by 1.0f / scale; steps: Adam's per-segment counts before the launch.
    Returns (p, state, g32, g16, updated) with `updated` the boolean mask of elements the rule ran on."""
    n = p.size
    p = p.astype(np.float32).copy()
    state = [s.astype(np.float32).copy() for s in state]
    g32_in = g32.astype(np.float32)
    inv = F32(1.0) / F32(scale) if scale is not None else F32(inv_scale)
    only16 = np.zeros(n, bool)
    updated = np.zeros(n, bool)
    seg_of = np.full(n, -1)
    for i, s in enumerate(segs):
        seg_of[s["begin"]:s["end"]] = i
        if g16 is not None and s["flags"] & GRAD16:
            only16[s["begin"]:s["end"]] = True
    with np.errstate(invalid="ignore", over="ignore"):
        g = g32_in.copy() if g16 is None else np.where(only16, g16, g32_in + g16.astype(np.float32)).astype(np.float32)
        g = g * inv
    for i, s in enumerate(segs):
        if skip or s["flags"] & FROZEN or s["end"] == s["begin"]:
            continue
        sl = slice(s["begin"], s["end"])
        updated[sl] = True
        if rule == "sgd":
            p[sl], state[0][sl] = sgd_update(p[sl], state[0][sl], g[sl], s["lr"], s["wd"], s["mu"],
                                             bool(s["flags"] & NESTEROV), fma=fma)
        else:
            b1, b2 = adam_beta(s["beta1"]), adam_beta(s["beta2"])
            ss, bc = adam_scalars(s["lr"], s["beta1"], s["beta2"], steps[i])
            p[sl], state[0][sl], state[1][sl] = adam_update(p[sl], state[0][sl], state[1][sl], g[sl], s["wd"], F32(1.0 - b1),
                                                            F32(s["beta2"]), F32(1.0 - b2), ss, bc, F32(s["eps"]), fma=fma)
    g_out = g32_in.copy()
    g16_out = None if g16 is None else g16.astype(np.float32).copy()
    if zero_grad:
        g_out[~only16] = 0.0
        if g16_out is not None:
            g16_out[:] = 0.0
    return p, state, g_out, g16_out, updated


def next_steps(steps, segs, skip):
    """Adam's per-segment counts after a launch: +1 for every non-frozen segment unless the step was skipped"""
    return [c + (0 if skip or s["flags"] & FROZEN else 1) for c, s in zip(steps, segs)]


MAX_LOSS_SCALE = 2.0 ** 24


def scaler_next(scale, unskipped, growth_interval, overflow):
    """the device loss scaler's rules (apex amp O1 with max_loss_scale = 2^24), in fp32: returns (scale, unskipped)"""
    if overflow:
        return float(max(F32(scale) * F32(0.5), F32(1.0))), 0
    unskipped += 1
    if growth_interval > 0 and unskipped % growth_interval == 0:
        scale = float(min(F32(scale) * F32(2.0), F32(MAX_LOSS_SCALE)))
    return float(F32(scale)), unskipped
