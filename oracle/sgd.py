"""ORACLE (test infrastructure only): SGD-momentum over a flat fp32 buffer with per-segment lr / wd,
gradient unscale, and the flat all-reduce-mean that precedes it.

Follows
* `torch.optim.SGD` single-tensor math — torch/optim/sgd.py:343-380 (weight decay folded into the
  gradient, `buf = g` on the first step else `buf = mu*buf + g`, dampening 0; Nesterov in `sgd_step_f64` only), as
  configured by the reference `make_optimizer(..., "f3_trick")` — utils/pipeline_ops.py:295-313
  (backbone lr×0.1, head lr×1, names starting with `div_2` in no group), stepped at train.py:303;
* apex `DistributedDataParallel(delay_allreduce=True)` published semantics (train.py:185): one flat
  buffer, SUM all-reduce, then ×1/world_size (parity unpinned — apex is not in the reference repository);
* apex `amp.scale_loss` exit: grads ×1/S, step skipped if any grad is non-finite (train.py:299).
* `CustomScheduler` — utils/pipeline_ops.py:185-232.

`sgd_step` carries the arithmetic in fp32 (np.float32) with every multiply and add rounded separately, in the order of
torch's single-tensor formula; the kernel fuses them (`fmaf`), so the two differ by a few ulps.
`oracle/optim_replay.py` is the kernel's own operation order, bit for bit; `sgd_step_f64` gives the exact-arithmetic
answer for tolerance sizing.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class Segment:
    begin: int          # element offsets into the flat buffers, [begin, end)
    end: int
    lr: float
    weight_decay: float
    momentum: float = 0.9
    frozen: bool = False    # True: gradients are still averaged, but p / v are not touched (div_2.*)
    nesterov: bool = False  # torch.optim.SGD(nesterov=True): p -= lr*(g + mu*v) after the momentum update


def allreduce_mean(rank_grads: list[np.ndarray]) -> np.ndarray:
    """SUM over ranks in rank order, then × 1/W (fp32)."""
    acc = rank_grads[0].astype(np.float32).copy()
    for g in rank_grads[1:]:
        acc += g.astype(np.float32)
    acc *= np.float32(1.0 / len(rank_grads))
    return acc


def sgd_step(p: np.ndarray, v: np.ndarray, g: np.ndarray, segments: list[Segment],
             inv_scale: float = 1.0) -> bool:
    """In-place fp32 step of plain momentum (a Nesterov segment raises: `sgd_step_f64` restates it).  Returns False
    (and touches nothing) when a gradient is non-finite (the amp overflow-skip)."""
    if any(s.nesterov for s in segments):
        raise NotImplementedError("sgd_step restates plain momentum only; use sgd_step_f64 for Nesterov segments")
    if not np.all(np.isfinite(g)):
        return False
    f = np.float32
    for s in segments:
        if s.frozen:
            continue
        sl = slice(s.begin, s.end)
        gg = g[sl].astype(np.float32) * f(inv_scale)
        gg = gg + f(s.weight_decay) * p[sl]
        v[sl] = f(s.momentum) * v[sl] + gg
        p[sl] = p[sl] - f(s.lr) * v[sl]
    return True


def sgd_step_f64(p, v, g, segments, inv_scale=1.0):
    p = p.astype(np.float64).copy(); v = v.astype(np.float64).copy(); g = g.astype(np.float64)
    for s in segments:
        if s.frozen:
            continue
        sl = slice(s.begin, s.end)
        gg = g[sl] * inv_scale + s.weight_decay * p[sl]
        v[sl] = s.momentum * v[sl] + gg
        p[sl] = p[sl] - s.lr * (gg + s.momentum * v[sl] if s.nesterov else v[sl])
    return p, v


def lr_coefficient(kind: str, curr: int, total: int, lr_decay: float = 0.9, warmup_epoch: int = 1) -> float:
    """utils/pipeline_ops.py:194-223 for one call (the reference's in-place edit of `total_num` in the
    warmup branches, :206/:217, is a per-call side effect that compounds; restated literally by
    `SchedulerState`)."""
    return SchedulerState(total, kind, lr_decay, warmup_epoch).coefficient(curr)


class SchedulerState:
    def __init__(self, total_num: int, kind: str, lr_decay: float = 0.9, warmup_epoch: int = 1):
        self.total_num, self.kind, self.lr_decay, self.warmup_epoch = total_num, kind, lr_decay, warmup_epoch

    def coefficient(self, curr: int) -> float:
        k = self.kind
        if k == "poly":
            return pow(1 - float(curr) / self.total_num, self.lr_decay)  # builtin pow: complex when base<0, like the reference
        if k in ("poly_warmup", "cosine_warmup"):
            turn = self.warmup_epoch
            if curr < turn:
                return 1 / turn * (1 + curr)
            curr -= turn - 1
            self.total_num -= turn - 1       # reference mutates its own state here
            if k == "poly_warmup":
                return pow(1 - float(curr) / self.total_num, self.lr_decay)  # builtin pow: complex when base<0, like the reference
            return float((1 + np.cos(np.pi * curr / self.total_num)) / 2)
        if k == "f3_sche":
            return 1 - abs((curr + 1) / (self.total_num + 1) * 2 - 1)
        raise NotImplementedError(k)
