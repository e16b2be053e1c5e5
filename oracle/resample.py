"""ORACLE (test infrastructure only): float64 restatements of the resampling ops of csrc/resample.cu and csrc/maxpool.cu.

* `upsample2x` / `upsample2x_bwd`: bilinear ×2, align_corners=False, written as explicit taps along each axis.  Output
  index 2k takes .25·in[k−1] + .75·in[k] and 2k+1 takes .75·in[k] + .25·in[k+1]; at the borders (2k = 0, 2k+1 = 2H−1)
  the output is in[0] / in[H−1] alone.  A tap of weight zero is absent, so an infinite input reaches exactly the
  outputs it has a weight in.  (torch's `upsample_bilinear2d` weights in[1] by 0 at output 0, so ±inf in row or column 1
  makes its output row / column 0 NaN; the mathematics, and the kernel, give a finite value there.)
* `avgpool2x2` / `avgpool2x2_bwd`: the 2×2 / stride-2 mean and its backward dy/4 on each of the four inputs.
* `maxpool_fwd` / `maxpool_bwd`: MaxPool2d(3, 2, 1) as the kernel computes it, on [N, H, W, C] arrays: the window
  scanned kh, kw ascending, replace on (v > max or v is NaN), the window position kh·3 + kw of the winner per element,
  and the gather backward over the ≤ 4 windows that contain an input pixel.

The first four take [..., H, W] arrays (the last two axes are the spatial ones) and work on numpy arrays and on torch
tensors alike; the caller picks float64.
"""
from __future__ import annotations

import numpy as np


def _zeros(x, shape):
    if isinstance(x, np.ndarray):
        return np.zeros(shape, x.dtype)
    return x.new_zeros(shape)


def _up_axis(x, axis):
    """×2 bilinear along `axis` (−2 or −1) with explicit taps"""
    x = x if axis == -1 else x.swapaxes(-1, -2) if isinstance(x, np.ndarray) else x.transpose(-1, -2)
    n = x.shape[-1]
    y = _zeros(x, x.shape[:-1] + (2 * n,))
    y[..., 0] = x[..., 0]
    y[..., 2 * n - 1] = x[..., n - 1]
    if n > 1:
        y[..., 2:2 * n:2] = 0.25 * x[..., :n - 1] + 0.75 * x[..., 1:]
        y[..., 1:2 * n - 1:2] = 0.75 * x[..., :n - 1] + 0.25 * x[..., 1:]
    if axis == -2:
        y = y.swapaxes(-1, -2) if isinstance(y, np.ndarray) else y.transpose(-1, -2)
    return y


def _up_axis_bwd(dy, axis):
    """adjoint of `_up_axis`: input k gathers .25·dy[2k−1] + .75·dy[2k] + .75·dy[2k+1] + .25·dy[2k+2], with weight 1 for
    the border outputs 0 and 2H−1"""
    dy = dy if axis == -1 else dy.swapaxes(-1, -2) if isinstance(dy, np.ndarray) else dy.transpose(-1, -2)
    n = dy.shape[-1] // 2
    dx = _zeros(dy, dy.shape[:-1] + (n,))
    even, odd = dy[..., 0::2], dy[..., 1::2]               # dy[2k], dy[2k+1]
    if n == 1:
        dx[..., 0] = even[..., 0] + odd[..., 0]
    else:
        dx[..., 0] = even[..., 0] + 0.75 * odd[..., 0] + 0.25 * even[..., 1]
        dx[..., n - 1] = 0.25 * odd[..., n - 2] + 0.75 * even[..., n - 1] + odd[..., n - 1]
        if n > 2:
            dx[..., 1:n - 1] = (0.25 * odd[..., :n - 2] + 0.75 * even[..., 1:n - 1] + 0.75 * odd[..., 1:n - 1]
                                + 0.25 * even[..., 2:])
    if axis == -2:
        dx = dx.swapaxes(-1, -2) if isinstance(dx, np.ndarray) else dx.transpose(-1, -2)
    return dx


def upsample2x(x, add=None):
    y = _up_axis(_up_axis(x, -2), -1)
    return y if add is None else y + add


def upsample2x_bwd(dy):
    return _up_axis_bwd(_up_axis_bwd(dy, -1), -2)


def avgpool2x2(x):
    return 0.25 * (x[..., 0::2, 0::2] + x[..., 0::2, 1::2] + x[..., 1::2, 0::2] + x[..., 1::2, 1::2])


def avgpool2x2_bwd(dy):
    q = 0.25 * dy
    dx = _zeros(dy, dy.shape[:-2] + (2 * dy.shape[-2], 2 * dy.shape[-1]))
    for i in (0, 1):
        for j in (0, 1):
            dx[..., i::2, j::2] = q
    return dx


def _where(x, cond, a, b):
    if isinstance(x, np.ndarray):
        return np.where(cond, a, b)
    import torch
    return torch.where(cond, a, b)


def _isnan(v):
    return np.isnan(v) if isinstance(v, np.ndarray) else v.isnan()


def maxpool_fwd(x):
    """x [N,H,W,C] → (y [N,HO,WO,C], arg [N,HO,WO,C]: window position kh·3 + kw of the element each output took)"""
    n, h, w, c = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    xp = _zeros(x, (n, 2 * ho + 1, 2 * wo + 1, c))          # one row / column of padding before, enough after
    xp[:, 1:h + 1, 1:w + 1] = x
    oh = np.arange(ho)[None, :, None, None]
    ow = np.arange(wo)[None, None, :, None]
    m = _zeros(x, (n, ho, wo, c)) - float("inf")
    # the scan starts at the first in-bounds position: (kh, kw) = (1, ·) in output row 0, (·, 1) in output column 0
    a = np.ascontiguousarray(np.broadcast_to(np.where(oh == 0, 3, 0) + np.where(ow == 0, 1, 0), (n, ho, wo, c)))
    if not isinstance(x, np.ndarray):
        import torch
        a = torch.from_numpy(a).to(x.device)
    for kh in range(3):
        for kw in range(3):
            ih, iw = 2 * oh - 1 + kh, 2 * ow - 1 + kw
            valid = (ih >= 0) & (ih < h) & (iw >= 0) & (iw < w)
            if not isinstance(x, np.ndarray):
                import torch
                valid = torch.from_numpy(valid).to(x.device)
            v = xp[:, kh:kh + 2 * ho:2, kw:kw + 2 * wo:2]
            take = valid & ((v > m) | _isnan(v))
            m = _where(x, take, v, m)
            a = _where(x, take, kh * 3 + kw, a)
    return m, a


def maxpool_bwd(dy, arg, h, w):
    """dy [N,HO,WO,C], arg as `maxpool_fwd` returns it → dx [N,H,W,C]: each output's gradient goes to the input its
    window position names"""
    n, ho, wo, c = dy.shape
    dxp = _zeros(dy, (n, 2 * ho + 1, 2 * wo + 1, c))
    for kh in range(3):
        for kw in range(3):
            dxp[:, kh:kh + 2 * ho:2, kw:kw + 2 * wo:2] += _where(dy, arg == kh * 3 + kw, dy, _zeros(dy, dy.shape))
    return dxp[:, 1:h + 1, 1:w + 1]
