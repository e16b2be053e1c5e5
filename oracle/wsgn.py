"""ORACLE (test infrastructure only): GroupNorm(32) with the residual / ReLU epilogue and weight standardisation of the
WS-GN backbone, numpy fp64.

Restates reference backbone/wsgn/customized_func.py:12-29: `nn.GroupNorm(32, C)` (biased variance over C/G channels ×
H × W per sample, eps 1e-5) and the weight standardisation Ŵ = (W − mean) / (std_unbiased + 1e-5) per output filter,
with their gradients written out by hand:
    GroupNorm: dx = rstd · (γ·dz − mean_g(γ·dz) − x̂ · mean_g(γ·dz·x̂)),  dγ = Σ dz·x̂,  dβ = Σ dz
    WS:        dW = (g − mean(g)) / s − v · Σ(g·v) / (s² · (K − 1) · σ),  v = W − μ,  s = σ + eps
The fused epilogue is the bottleneck's: y = relu?(GN(x) [+ residual]) (network/blocks.py `bn_act`).
"""
from __future__ import annotations

import numpy as np

GROUPS = 32


def group_norm_forward(x, gamma, beta, residual=None, relu=False, eps=1e-5, groups=GROUPS):
    """x: [N,C,H,W].  Returns dict(y, mean [N,G], rstd [N,G], xhat)"""
    x = np.asarray(x, np.float64)
    n, c, h, w = x.shape
    xg = x.reshape(n, groups, c // groups * h * w)
    mean = xg.mean(axis=2)
    var = ((xg - mean[:, :, None]) ** 2).mean(axis=2)
    rstd = 1.0 / np.sqrt(var + eps)
    xhat = ((xg - mean[:, :, None]) * rstd[:, :, None]).reshape(n, c, h, w)
    y = xhat * np.asarray(gamma, np.float64)[None, :, None, None] + np.asarray(beta, np.float64)[None, :, None, None]
    if residual is not None:
        y = y + np.asarray(residual, np.float64)
    if relu:
        y = np.maximum(y, 0.0)
    return dict(y=y, mean=mean, rstd=rstd, xhat=xhat)


def group_norm_backward(dy, x, gamma, beta, residual=None, relu=False, eps=1e-5, groups=GROUPS):
    """Returns dict(dx, dres, dgamma, dbeta) of the forward above"""
    f = group_norm_forward(x, gamma, beta, residual, relu, eps, groups)
    dz = np.asarray(dy, np.float64) * ((f["y"] > 0) if relu else 1.0)
    n, c, h, w = dz.shape
    g = np.asarray(gamma, np.float64)[None, :, None, None]
    dxh = (dz * g).reshape(n, groups, -1)
    xh = f["xhat"].reshape(n, groups, -1)
    dx = f["rstd"][:, :, None] * (dxh - dxh.mean(axis=2, keepdims=True) - xh * (dxh * xh).mean(axis=2, keepdims=True))
    return dict(dx=dx.reshape(n, c, h, w), dres=dz if residual is not None else None,
                dgamma=(dz * f["xhat"]).sum(axis=(0, 2, 3)), dbeta=dz.sum(axis=(0, 2, 3)))


def ws_forward(w, eps=1e-5):
    """w: [O, ...]; Ŵ of the same shape"""
    w = np.asarray(w, np.float64)
    v = w.reshape(w.shape[0], -1)
    v = v - v.mean(axis=1, keepdims=True)
    s = v.std(axis=1, ddof=1, keepdims=True) + eps
    return (v / s).reshape(w.shape)


def ws_backward(w, g, eps=1e-5):
    """dW of Ŵ = ws_forward(w) for the upstream gradient g = dŴ"""
    w = np.asarray(w, np.float64)
    k = w[0].size
    v = w.reshape(w.shape[0], -1)
    v = v - v.mean(axis=1, keepdims=True)
    sigma = v.std(axis=1, ddof=1, keepdims=True)
    s = sigma + eps
    g = np.asarray(g, np.float64).reshape(w.shape[0], -1)
    dw = (g - g.mean(axis=1, keepdims=True)) / s - v * (g * v).sum(axis=1, keepdims=True) / (s * s * (k - 1) * sigma)
    return dw.reshape(w.shape)
