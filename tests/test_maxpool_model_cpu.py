"""Executable model of csrc/maxpool.cu (the stem's MaxPool2d(3,2,1) kernels; oracle/resample.py `maxpool_fwd` /
`maxpool_bwd`): the same window / candidate arithmetic, replayed in Python on small tensors and compared with torch's
CPU max_pool2d forward and autograd backward — odd and even sizes, ties, -inf, NaN.  tests/test_gpu_resample_regimes.py
holds the kernels to this model; what can go wrong silently here is the index arithmetic (which windows contain an
input pixel, which byte code a position gets, who wins a tie)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.resample import maxpool_bwd as bwd_model, maxpool_fwd as fwd_model


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
