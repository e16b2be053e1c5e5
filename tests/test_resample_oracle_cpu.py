"""oracle/resample.py (the float64 up-sample and average-pool restatements the GPU regime tests hold the kernels to)
against torch's CPU ops in float64: values, the backward through autograd, sizes 1 … 9 in each axis, and ±inf / NaN.
torch's bilinear weights in[1] by 0 at output 0 (in[0] when the axis has one element), which makes ±inf or NaN there
a NaN in output row / column 0; the oracle has no such tap, so those outputs are compared only where torch's product
is finite."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import resample as ors

SIZES = [(1, 1), (1, 2), (2, 1), (2, 2), (3, 5), (5, 3), (4, 9), (9, 7)]


def _x(h, w, seed, special=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 3, h, w, generator=g, dtype=torch.float64)
    if special:
        x[0, 0, 0, 0] = float("inf")
        x[0, 1, h - 1, w - 1] = float("-inf")
        x[1, 2, h // 2, 0] = float("nan")
        x[1, 0, 0, w - 1] = float("inf")
    return x


@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("special", [False, True])
@pytest.mark.parametrize("fmt", ["numpy", "torch"])
def test_upsample_oracle_matches_interpolate(h, w, special, fmt):
    x = _x(h, w, h * 10 + w, special)
    add = _x(2 * h, 2 * w, 99)
    want = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False) + add
    got = ors.upsample2x(x.numpy() if fmt == "numpy" else x, add.numpy() if fmt == "numpy" else add)
    got = torch.as_tensor(got)
    if special:
        # torch reads in[min(1, H − 1)] with weight 0 at output row 0 (and likewise for columns): keep those outputs out
        # where that input is not finite
        keep = torch.ones_like(want, dtype=torch.bool)
        r, c = min(1, h - 1), min(1, w - 1)
        def near(v):            # output 2k and 2k+1 read inputs k − 1 … k + 1
            return F.max_pool1d((~v.isfinite()).double(), 3, 1, 1).bool().repeat_interleave(2, -1)
        keep[:, :, 0, :] &= ~near(x[:, :, r, :])
        keep[:, :, :, 0] &= ~near(x[:, :, :, c])
        want, got = want[keep], got[keep]
    torch.testing.assert_close(got, want, rtol=1e-15, atol=1e-15, equal_nan=True)


@pytest.mark.parametrize("h,w", SIZES)
def test_upsample_oracle_backward_matches_autograd(h, w):
    x = _x(h, w, 7 * h + w).requires_grad_(True)
    dy = _x(2 * h, 2 * w, 3)
    F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False).backward(dy)
    torch.testing.assert_close(torch.as_tensor(ors.upsample2x_bwd(dy.numpy())), x.grad, rtol=1e-15, atol=1e-15)
    torch.testing.assert_close(ors.upsample2x_bwd(dy), x.grad, rtol=1e-15, atol=1e-15)


def test_upsample_oracle_keeps_border_infinities():
    """an infinite in[0] gives ±inf (not NaN) in output row and column 0, as the mathematics does"""
    x = torch.zeros(1, 1, 3, 3, dtype=torch.float64)
    x[0, 0, 0, 0] = float("inf")
    x[0, 0, 2, 2] = float("-inf")
    y = torch.as_tensor(ors.upsample2x(x.numpy()))
    assert y[0, 0, 0, 0] == float("inf") and y[0, 0, 0, 1] == float("inf") and y[0, 0, 1, 0] == float("inf")
    assert y[0, 0, 5, 5] == float("-inf")
    assert not bool(y[0, 0, :2, :2].isnan().any())


@pytest.mark.parametrize("h,w", [(1, 1), (1, 3), (3, 1), (2, 5), (4, 4)])
@pytest.mark.parametrize("special", [False, True])
def test_avgpool_oracle_matches_torch(h, w, special):
    x = _x(2 * h, 2 * w, h + 13 * w, special).requires_grad_(True)
    want = F.avg_pool2d(x, 2, 2)
    torch.testing.assert_close(torch.as_tensor(ors.avgpool2x2(x.detach().numpy())), want.detach(), rtol=1e-15, atol=1e-15,
                               equal_nan=True)
    dy = _x(h, w, 5)
    want.backward(dy)
    torch.testing.assert_close(torch.as_tensor(ors.avgpool2x2_bwd(dy.numpy())), x.grad, rtol=0, atol=0)


@pytest.mark.parametrize("h,w", [(1, 1), (2, 5), (9, 7), (6, 3)])
def test_maxpool_oracle_is_the_same_on_numpy_and_torch(h, w):
    x = _x(h, w, 17 * h + w, special=True).permute(0, 2, 3, 1).contiguous()
    if h > 1 and w > 1:
        x[0, 0, 0, 1] = x[0, 0, 1, 1]                        # a tie
    y, a = ors.maxpool_fwd(x.numpy())
    yt, at = ors.maxpool_fwd(x)
    np.testing.assert_array_equal(y, yt.numpy())
    np.testing.assert_array_equal(a, at.numpy())
    dy = _x(y.shape[1], y.shape[2], 4).permute(0, 2, 3, 1).contiguous()
    np.testing.assert_array_equal(ors.maxpool_bwd(dy.numpy(), a, h, w), ors.maxpool_bwd(dy, at, h, w).numpy())
