"""Executable model of csrc/maxpool.cu (experimental MaxPool2d(3,2,1) kernels): the same window / candidate arithmetic,
replayed in Python on small tensors and compared with torch's CPU max_pool2d forward and autograd backward — odd and
even sizes, ties, -inf, NaN.  The kernels themselves can only run on a GPU; what can go wrong silently is this index
arithmetic (which windows contain an input pixel, which byte code a position gets, who wins a tie)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F


def fwd_model(x):                       # x [N,H,W,C] float32 → y [N,HO,WO,C], arg uint8 [N,HO,WO,C]
    n, h, w, c = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    y = np.empty((n, ho, wo, c), np.float32)
    arg = np.empty((n, ho, wo, c), np.uint8)
    for oh in range(ho):
        for ow in range(wo):
            h0, w0 = 2 * oh - 1, 2 * ow - 1
            m = a = None
            for kh in range(3):
                ih = h0 + kh
                if ih < 0 or ih >= h:
                    continue
                for kw in range(3):
                    iw = w0 + kw
                    if iw < 0 or iw >= w:
                        continue
                    pos = kh * 3 + kw
                    v = x[:, ih, iw, :]
                    if m is None:
                        m = np.full_like(v, -np.inf)
                        a = np.full(v.shape, pos, np.uint8)
                    take = (v > m) | np.isnan(v)
                    m = np.where(take, v, m)
                    a = np.where(take, np.uint8(pos), a)
            y[:, oh, ow, :], arg[:, oh, ow, :] = m, a
    return y, arg


def bwd_model(dy, arg, h, w):           # gather: every input pixel looks at the ≤4 windows containing it
    n, ho, wo, c = dy.shape
    dx = np.zeros((n, h, w, c), np.float32)
    for ih in range(h):
        for iw in range(w):
            noh, now = (2 if ih & 1 else 1), (2 if iw & 1 else 1)
            oh0 = (ih - 1) // 2 if ih & 1 else ih // 2
            ow0 = (iw - 1) // 2 if iw & 1 else iw // 2
            acc = np.zeros((n, c), np.float32)
            for a in range(noh):
                oh = oh0 + a
                if oh >= ho:
                    continue
                kh = (2 if a == 0 else 0) if ih & 1 else 1
                for b in range(now):
                    ow = ow0 + b
                    if ow >= wo:
                        continue
                    kw = (2 if b == 0 else 0) if iw & 1 else 1
                    pos = kh * 3 + kw
                    acc += np.where(arg[:, oh, ow, :] == pos, dy[:, oh, ow, :], 0).astype(np.float32)
            dx[:, ih, iw, :] = acc
    return dx


@pytest.mark.parametrize("h,w", [(8, 8), (9, 7), (1, 1), (2, 5), (13, 16), (6, 3)])
@pytest.mark.parametrize("kind", ["random", "ties", "special"])
def test_model_matches_torch(h, w, kind):
    g = torch.Generator().manual_seed(h * 100 + w)
    n, c = 2, 8
    if kind == "random":
        x = torch.randn(n, c, h, w, generator=g)
    elif kind == "ties":
        x = torch.randint(0, 3, (n, c, h, w), generator=g).float()          # many equal maxima: first in scan order wins
    else:
        x = torch.randn(n, c, h, w, generator=g)
        x[0, 0] = float("-inf")
        if h * w > 2:
            x[1, 1, h // 2, w // 2] = float("nan")
    xt = x.clone().requires_grad_(True)
    yt = F.max_pool2d(xt, 3, 2, 1)
    dy = torch.randn(yt.shape, generator=g)
    yt.backward(dy)
    y, arg = fwd_model(x.permute(0, 2, 3, 1).numpy())
    np.testing.assert_array_equal(y, yt.detach().permute(0, 2, 3, 1).numpy())
    dx = bwd_model(dy.permute(0, 2, 3, 1).numpy(), arg, h, w)
    np.testing.assert_allclose(dx, xt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-6, atol=1e-6)
    # every output element names a position inside its own window
    assert arg.max() <= 8


def test_cpu_tensors_keep_the_torch_op():
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.network import blocks
    assert resample.MAXPOOL_ENABLED is True        # default on: checked against torch by tests/test_gpu_resample.py
    pool = blocks._StemPool(3, 2, 1)
    x = torch.randn(1, 8, 6, 6)
    assert torch.equal(pool(x), F.max_pool2d(x, 3, 2, 1))                   # CPU / disabled → torch op
