"""ORACLE (test infrastructure only): Adam over a flat fp32 buffer with per-segment lr / wd / betas / eps and a step
count per segment, behind the same gradient unscale as `oracle.sgd`.

Follows `torch.optim.Adam` single-tensor math — torch/optim/adam.py `_single_tensor_adam` with amsgrad=False,
maximize=False and L2 (not decoupled) weight decay — as the reference's `make_optimizer(..., "adam")` builds it
(utils/pipeline_ops.py:287-294: betas (0.9, 0.999), eps 1e-8, one group over `model.parameters()`):

    g' = g*inv_scale + wd*p ;  m = m + (1-β1)*(g'-m) ;  v = v*β2 + (1-β2)*g'*g'
    t = step+1 ;  step_size = fp32(lr / (1-β1^t)) ;  bc2_sqrt = fp32(sqrt(1-β2^t))     (Python / fp64 scalars)
    p = p - step_size * (m / (sqrt(v)/bc2_sqrt + eps))

`adam_step` carries the elementwise arithmetic in fp32 in that order, so the GPU result can be compared tightly;
`adam_step_f64` is the exact-arithmetic answer for tolerance sizing.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np


@dataclass
class Segment:
    begin: int          # element offsets into the flat buffers, [begin, end)
    end: int
    lr: float
    weight_decay: float
    beta1: float = 0.9
    beta2: float = 0.999
    eps: float = 1e-8
    frozen: bool = False    # True: p / m / v are not touched and the step count does not advance


def adam_step(p: np.ndarray, m: np.ndarray, v: np.ndarray, g: np.ndarray, segments: list[Segment], steps: list[int],
              inv_scale: float = 1.0) -> bool:
    """In-place fp32 step; `steps[i]` is segment i's count before the step and is advanced.  Returns False (and touches
    nothing) when a gradient is non-finite (the amp overflow skip)."""
    if not np.all(np.isfinite(g)):
        return False
    f = np.float32
    for i, s in enumerate(segments):
        if s.frozen:
            continue
        sl = slice(s.begin, s.end)
        t = steps[i] + 1
        gg = g[sl].astype(np.float32) * f(inv_scale)
        gg = gg + f(s.weight_decay) * p[sl]
        m[sl] = m[sl] + f(1.0 - s.beta1) * (gg - m[sl])
        v[sl] = v[sl] * f(s.beta2) + (f(1.0 - s.beta2) * gg) * gg
        step_size = f(s.lr / (1.0 - s.beta1 ** t))
        bc2_sqrt = f(math.sqrt(1.0 - s.beta2 ** t))
        denom = np.sqrt(v[sl]) / bc2_sqrt + f(s.eps)
        p[sl] = p[sl] - step_size * (m[sl] / denom)
        steps[i] = t
    return True


def adam_step_f64(p, m, v, g, segments, steps, inv_scale=1.0):
    """Returns (p, m, v, steps) in float64; the inputs are left alone."""
    p = p.astype(np.float64).copy(); m = m.astype(np.float64).copy(); v = v.astype(np.float64).copy()
    g = g.astype(np.float64); steps = list(steps)
    for i, s in enumerate(segments):
        if s.frozen:
            continue
        sl = slice(s.begin, s.end)
        t = steps[i] + 1
        gg = g[sl] * inv_scale + s.weight_decay * p[sl]
        m[sl] = s.beta1 * m[sl] + (1.0 - s.beta1) * gg
        v[sl] = s.beta2 * v[sl] + (1.0 - s.beta2) * gg * gg
        p[sl] = p[sl] - s.lr / (1.0 - s.beta1 ** t) * m[sl] / (np.sqrt(v[sl]) / math.sqrt(1.0 - s.beta2 ** t) + s.eps)
        steps[i] = t
    return p, m, v, steps
