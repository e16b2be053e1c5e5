"""Channels-last ×2 bilinear (+fused add) and 2×2 average-pool kernels against torch's own ops (fwd and bwd)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import resample_geometry as geo

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _enable():
    from distributed_sod_project_b200 import resample
    old, resample.ENABLED = resample.ENABLED, True
    yield
    resample.ENABLED = old


def _mk(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(shape, generator=g).to(dtype).cuda().contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("shape", [(2, 32, 5, 7), (16, 64, 10, 10), (3, 8, 1, 1), (2, 64, 40, 40), (1, 128, 2, 9)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_add", [False, True])
def test_upsample2x_matches_interpolate(shape, dtype, with_add):
    from distributed_sod_project_b200 import resample
    n, c, h, w = shape
    x1 = _mk(shape, dtype, 1).requires_grad_(True)
    lat1 = _mk((n, c, 2 * h, 2 * w), dtype, 2).requires_grad_(True) if with_add else None
    lat2 = lat1.detach().clone().requires_grad_(True) if with_add else None
    y1 = resample.upsample2x_add(x1, lat1) if with_add else resample.upsample2x(x1, (2 * h, 2 * w))
    assert y1 is not None and y1.is_contiguous(memory_format=torch.channels_last)
    # against float64: one ulp of the dtype plus the fp32 slack of the weighted sums (test_upsample2x_past_one_grid_pass)
    x2 = x1.detach().double().requires_grad_(True)
    ref = F.interpolate(x2, size=(2 * h, 2 * w), mode="bilinear", align_corners=False)
    mag = F.interpolate(x2.detach().abs(), size=(2 * h, 2 * w), mode="bilinear", align_corners=False)
    if with_add:
        ref = ref + lat2.double()
        mag = mag + lat2.double().abs()
    assert bool(((y1.double() - ref.detach()).abs() <= _ulp(ref.detach(), dtype) + 2.0 ** -20 * mag).all())
    dy = _mk((n, c, 2 * h, 2 * w), dtype, 3)
    y1.backward(dy)
    ref.backward(dy.double())
    x0 = torch.zeros_like(x2).requires_grad_(True)
    F.interpolate(x0, size=(2 * h, 2 * w), mode="bilinear", align_corners=False).backward(dy.double().abs())
    assert bool(((x1.grad.double() - x2.grad).abs() <= _ulp(x2.grad, dtype) + 2.0 ** -20 * x0.grad).all())
    if with_add:
        assert torch.equal(lat1.grad, dy)


@pytest.mark.parametrize("shape", [(2, 32, 6, 8), (16, 64, 20, 20), (1, 8, 2, 2)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_avgpool2x2_matches_torch(shape, dtype):
    from distributed_sod_project_b200 import resample
    x1 = _mk(shape, dtype, 5).requires_grad_(True)
    x2 = x1.detach()
    y1 = resample.avgpool2x2(x1)
    ref = F.avg_pool2d(x2.double(), 2, 2)
    # against float64: one ulp plus the rounding of the fp32 sum of four (2⁻²² of the mean of |x|)
    assert bool(((y1.double() - ref).abs() <= _ulp(ref, dtype) + 2.0 ** -22 * F.avg_pool2d(x2.double().abs(), 2, 2)).all())
    dy = _mk(tuple(ref.shape), dtype, 6)
    y1.backward(dy)
    assert torch.equal(x1.grad, F.interpolate(dy.double() / 4, scale_factor=2, mode="nearest").to(dtype))   # dy/4: exact


def test_unsupported_shapes_fall_back_and_backward_is_deterministic():
    from distributed_sod_project_b200 import resample
    x = _mk((2, 32, 5, 7), torch.bfloat16, 1)
    assert resample.upsample2x(x, (11, 14)) is None            # not exactly ×2
    assert resample.avgpool2x2(_mk((1, 32, 5, 6), torch.float32, 2)) is None   # odd height
    assert resample.upsample2x(torch.zeros(1, 8, 2, 2), (4, 4)) is None        # CPU
    xs = _mk((4, 64, 20, 20), torch.bfloat16, 3).requires_grad_(True)
    dy = _mk((4, 64, 40, 40), torch.bfloat16, 4)
    grads = []
    for _ in range(3):
        xs.grad = None
        resample.upsample2x(xs, (40, 40)).backward(dy)
        grads.append(xs.grad.clone())
    assert torch.equal(grads[0], grads[1]) and torch.equal(grads[0], grads[2])


@pytest.mark.parametrize("shape", [(16, 64, 160, 160), (2, 8, 9, 7), (3, 32, 1, 1), (2, 64, 2, 5), (4, 16, 13, 16)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("ties", [False, True])
def test_maxpool3x3s2_matches_torch(shape, dtype, ties):
    """csrc/maxpool.cu against F.max_pool2d(3, 2, 1): forward bit-exact (incl. which element wins a tie, through the
    backward), backward equal up to the rounding of ≤4-term fp32 sums"""
    from distributed_sod_project_b200 import resample
    x1 = _mk(shape, dtype, 5)
    if ties:
        x1 = (x1 * 2).round() / 2                      # many equal maxima inside a window
    x1 = x1.requires_grad_(True)
    x2 = x1.detach().clone().requires_grad_(True)
    y1 = resample._MaxPool3x3s2.apply(x1)
    y2 = F.max_pool2d(x2, 3, 2, 1)
    assert y1.shape == y2.shape and torch.equal(y1, y2)
    dy = _mk(tuple(y2.shape), dtype, 6)
    y1.backward(dy)
    y2.backward(dy)
    torch.cuda.synchronize()
    tol = dict(rtol=1e-6, atol=1e-6) if dtype == torch.float32 else dict(rtol=1e-2, atol=1e-2) if dtype == torch.bfloat16 \
        else dict(rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(x1.grad.float(), x2.grad.float(), **tol)
    # the routed module: identical to nn.MaxPool2d when the switch is on
    from distributed_sod_project_b200.network import blocks
    old, resample.MAXPOOL_ENABLED = resample.MAXPOOL_ENABLED, True
    try:
        if shape[1] % 8 == 0:
            assert torch.equal(blocks._StemPool(3, 2, 1)(x1.detach()), y2.detach())
    finally:
        resample.MAXPOOL_ENABLED = old


@pytest.mark.parametrize("shape", [(16, 64, 160, 160), (3, 8, 5, 7), (2, 2048, 3, 3), (1, 64, 1, 1), (4, 256, 20, 20)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_colsum_matches_torch_and_is_deterministic(shape, dtype):
    from distributed_sod_project_b200 import resample
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(shape, generator=g).to(dtype).cuda().contiguous(memory_format=torch.channels_last)
    got = resample.colsum(x)
    sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    rows = x.permute(0, 2, 3, 1).reshape(-1, shape[1]).float().cpu().numpy()
    want = torch.from_numpy(geo.colsum_replay(rows, sm)).to(dtype)
    assert torch.equal(got.cpu(), want), "the column sum is not the kernel's fp32 summation order rounded once"
    assert all(torch.equal(resample.colsum(x), got) for _ in range(3))


def test_conv_with_colsum_bias_gradient_matches_autograd():
    """the five `trans*` convolutions (1x1, 64 outputs, bias): forward identical, input / weight gradients cuDNN's, bias
    gradient = deterministic column sum"""
    from distributed_sod_project_b200 import resample
    old, resample.ENABLED = resample.ENABLED, True
    try:
        for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 2e-2)):
            conv = torch.nn.Conv2d(256, 64, 1).cuda().to(dtype).to(memory_format=torch.channels_last)
            x = torch.randn(4, 256, 20, 20, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
            dy = torch.randn(4, 64, 20, 20, device="cuda").to(dtype).contiguous(memory_format=torch.channels_last)
            res = []
            for mine in (False, True):
                xx = x.clone().requires_grad_(True)
                w = conv.weight.detach().clone().requires_grad_(True); b = conv.bias.detach().clone().requires_grad_(True)
                y = resample.conv_bias(conv, xx, w, b) if mine else torch.nn.functional.conv2d(xx, w, b)
                assert y is not None
                y.backward(dy)
                res.append((y.detach(), xx.grad, w.grad, b.grad))
            assert torch.equal(res[0][0], res[1][0])
            assert torch.equal(res[1][3], resample.colsum(dy).to(dtype))        # the bias gradient IS the column sum
            for a, bb in zip(res[0][1:], res[1][1:]):
                assert float((a.float() - bb.float()).abs().max()) <= tol * max(1.0, float(a.float().abs().max()))
    finally:
        resample.ENABLED = old


def _ulp(ref, dtype):
    mant, emin = {torch.float32: (23, -126), torch.bfloat16: (7, -126), torch.float16: (10, -14)}[dtype]
    return torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin))) - mant)


def _past_two_grid_passes(c):
    """an (N, C, H, W) input with more than two passes of the grid-stride loops (16 CTAs of 256 threads per SM, one 16-byte
    packet per thread) and a ragged last pass, at the INPUT's size (the smaller tensor of both launches)"""
    per_pass = 16 * torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 256
    w = 38
    h = -(-(2 * per_pass + per_pass // 3) // (w * c // 8))
    return (1, c, h + h % 2, w)                                  # even: the avg-pool takes the same input


LARGE = ["grid", (16, 64, 160, 160), (16, 64, 40, 40)]           # the TestModel's bs-16 up-samples at 320² (and 80²)


@pytest.mark.parametrize("shape", LARGE)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_upsample2x_past_one_grid_pass(shape, dtype):
    """against float64 bilinear interpolation: one ulp of the output dtype plus the fp32 slack of the 4-term (forward)
    / ≤16-term (backward) weighted sums (2⁻²⁰ of the same sums taken over |values|)"""
    from distributed_sod_project_b200 import resample
    shape = _past_two_grid_passes(64) if shape == "grid" else shape
    n, c, h, w = shape
    x = _mk(shape, dtype, 11).requires_grad_(True)
    lat = _mk((n, c, 2 * h, 2 * w), dtype, 12)
    y = resample.upsample2x_add(x, lat)
    x64 = x.detach().double().requires_grad_(True)
    ref = F.interpolate(x64, size=(2 * h, 2 * w), mode="bilinear", align_corners=False) + lat.double()
    mag = F.interpolate(x64.detach().abs(), size=(2 * h, 2 * w), mode="bilinear", align_corners=False) + lat.double().abs()
    assert bool(((y.double() - ref.detach()).abs() <= _ulp(ref.detach(), dtype) + 2.0 ** -20 * mag).all())
    dy = _mk((n, c, 2 * h, 2 * w), dtype, 13)
    y.backward(dy)
    ref.backward(dy.double())
    x0 = torch.zeros_like(x64).requires_grad_(True)
    F.interpolate(x0, size=(2 * h, 2 * w), mode="bilinear", align_corners=False).backward(dy.double().abs())
    assert bool(((x.grad.double() - x64.grad).abs() <= _ulp(x64.grad, dtype) + 2.0 ** -20 * x0.grad).all())


@pytest.mark.parametrize("shape", LARGE[:2])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_avgpool2x2_past_one_grid_pass(shape, dtype):
    """against float64: a mean of four values of a 2-byte type is exact in fp32, so the output is the correctly rounded
    fp64 mean; fp32 inputs get one ulp plus the rounding of the fp32 sum (2⁻²² of the mean of |x|).  The backward
    (dy / 4) is exact in every dtype."""
    from distributed_sod_project_b200 import resample
    shape = _past_two_grid_passes(64) if shape == "grid" else shape
    x = _mk(shape, dtype, 14).requires_grad_(True)
    y = resample.avgpool2x2(x)
    ref = F.avg_pool2d(x.detach().double(), 2, 2)
    if dtype == torch.float32:
        assert bool(((y.double() - ref).abs() <= _ulp(ref, dtype) + 2.0 ** -22 * F.avg_pool2d(x.detach().double().abs(), 2, 2)).all())
    else:
        assert torch.equal(y, ref.to(dtype))
    dy = _mk(tuple(ref.shape), dtype, 15)
    y.backward(dy)
    want = F.interpolate(dy.double() / 4, scale_factor=2, mode="nearest").to(dtype)
    assert torch.equal(x.grad, want)
