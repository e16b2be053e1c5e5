"""ORACLE (test infrastructure only): synchronized batch-norm over W ranks, numpy fp64.

Restates the published semantics of `apex.parallel.SyncBatchNorm` as installed by
`convert_syncbn_model` (reference train.py:180; apex itself is NOT in the reference repository —
**parity unpinned**), using the readable in-container equivalent as the arithmetic spec:
torch/nn/modules/_functions.py:7-209 (`SyncBatchNorm`): training statistics are taken over
N·H·W of ALL ranks (equal per-rank counts here), running_mean/var use momentum 0.1 with the
UNBIASED variance, eps 1e-5; backward all-reduces (Σdy, Σdy·(x-mean)) and keeps dγ/dβ local.

Cross-check used by the tests: W-rank SyncBN == plain BN on the rank-concatenated batch.

The fused epilogues mirror the three patterns the model plugins use
(distributed_sod_project_b200/network/blocks.py `bn_act`):
    y = relu?( BN(x [+ pre_add]) [+ residual] )
"""
from __future__ import annotations

import numpy as np


def _cstats(z: np.ndarray):
    """per-channel (sum, sumsq, count) of an [N,C,H,W] array"""
    return z.sum(axis=(0, 2, 3)), (z * z).sum(axis=(0, 2, 3)), z.shape[0] * z.shape[2] * z.shape[3]


def syncbn_forward(xs, gamma, beta, running_mean=None, running_var=None, momentum=0.1, eps=1e-5,
                   pre_adds=None, residuals=None, relu=False):
    """xs: list (one per rank) of [N,C,H,W]. Returns dict(ys, mean, invstd, var_biased,
    running_mean, running_var, zs)."""
    W = len(xs)
    zs = [np.asarray(x, np.float64) + (0 if pre_adds is None else np.asarray(pre_adds[r], np.float64))
          for r, x in enumerate(xs)]
    s = sum(_cstats(z)[0] for z in zs)
    q = sum(_cstats(z)[1] for z in zs)
    n = sum(_cstats(z)[2] for z in zs)
    mean = s / n
    var = np.maximum(q / n - mean * mean, 0.0)
    invstd = 1.0 / np.sqrt(var + eps)
    g = np.asarray(gamma, np.float64)[None, :, None, None]
    b = np.asarray(beta, np.float64)[None, :, None, None]
    ys = []
    for r, z in enumerate(zs):
        y = (z - mean[None, :, None, None]) * invstd[None, :, None, None] * g + b
        if residuals is not None:
            y = y + np.asarray(residuals[r], np.float64)
        if relu:
            y = np.maximum(y, 0.0)
        ys.append(y)
    out = dict(ys=ys, mean=mean, invstd=invstd, var_biased=var, zs=zs, count=n)
    if running_mean is not None:
        unbiased = var * (n / max(n - 1, 1))
        out["running_mean"] = (1 - momentum) * np.asarray(running_mean, np.float64) + momentum * mean
        out["running_var"] = (1 - momentum) * np.asarray(running_var, np.float64) + momentum * unbiased
    return out


def syncbn_backward(dys, zs, ys, mean, invstd, gamma, relu=False):
    """dys/zs/ys: per-rank lists. Returns dict(dzs, dgammas, dbetas, dresiduals):
    dz is the gradient of both x and pre_add; dresidual (= relu-masked dy) of the residual input;
    dγ/dβ are per-rank LOCAL sums (DDP averages them later)."""
    W = len(dys)
    m = mean[None, :, None, None]
    r_ = invstd[None, :, None, None]
    g = np.asarray(gamma, np.float64)[None, :, None, None]
    dms = []
    for r in range(W):
        d = np.asarray(dys[r], np.float64)
        if relu:
            d = d * (np.asarray(ys[r]) > 0)
        dms.append(d)
    n = sum(z.shape[0] * z.shape[2] * z.shape[3] for z in zs)
    sum_dy = sum(d.sum(axis=(0, 2, 3)) for d in dms)
    sum_dy_xmu = sum((d * (z - m)).sum(axis=(0, 2, 3)) for d, z in zip(dms, zs))
    mean_dy = (sum_dy / n)[None, :, None, None]
    mean_dy_xmu = (sum_dy_xmu / n)[None, :, None, None]
    dzs, dgs, dbs = [], [], []
    for d, z in zip(dms, zs):
        dzs.append((d - mean_dy - (z - m) * r_ * r_ * mean_dy_xmu) * r_ * g)
        dgs.append((d * (z - m) * r_).sum(axis=(0, 2, 3)))
        dbs.append(d.sum(axis=(0, 2, 3)))
    return dict(dzs=dzs, dgammas=dgs, dbetas=dbs, dresiduals=dms)
