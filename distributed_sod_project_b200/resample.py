"""Channels-last ×2 bilinear up-sampling (+ fused add), 2×2 average pooling and nearest ×2 up-sampling, backed by
csrc/resample.cu and csrc/nearest.cu.

These are the reference's `cus_sample` / `upsample_add` (utils/tensor_ops.py:12-25), `h2l_pool`
(module/MyLightModule.py:14) and LightAIM's `nn.Upsample(scale_factor=2, mode="nearest")` (module/MyLightModule.py:64,146).
The model plugins call `upsample2x` / `upsample2x_add` / `avgpool2x2` / `upsample2x_nearest` through
`network/blocks.py`; anything the kernels do not cover (CPU tensors, a ratio other than exactly 2, C % 8 != 0)
returns None so the caller keeps the torch op — those are shapes the TestModel never produces on the hot path.
"""
from __future__ import annotations

import os

import torch

from . import _lib

ENABLED = False     # switched on by the engine (engine.Trainer)
# the ResNet stem's MaxPool2d(3, 2, 1) and VGG16-BN's MaxPool2d(2, 2) through csrc/maxpool.cu (checked against torch by
# tests/test_gpu_resample.py and tests/test_gpu_maxpool2.py; SOD_MAXPOOL=0 → torch op)
MAXPOOL_ENABLED = os.environ.get("SOD_MAXPOOL", "1") == "1"
# bias gradient of the convolutions that do not feed a BatchNorm as a deterministic column sum (SOD_COLSUM=0 → autograd's reduction)
COLSUM_ENABLED = os.environ.get("SOD_COLSUM", "1") == "1"


def _ok(x: torch.Tensor) -> bool:
    return (ENABLED and x.is_cuda and x.dim() == 4 and x.shape[1] % 8 == 0
            and x.dtype in (torch.bfloat16, torch.float16, torch.float32))


def _rows(t: torch.Tensor) -> torch.Tensor:
    return t if t.is_contiguous(memory_format=torch.channels_last) else t.contiguous(memory_format=torch.channels_last)


class _Up2x(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, add):
        x = _rows(x)
        n, c, h, w = x.shape
        if add is not None:
            add = _rows(add).to(x.dtype)
        y = torch.empty((n, c, 2 * h, 2 * w), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_upsample2x_bilinear_fwd(x.data_ptr(), add.data_ptr() if add is not None else None, y.data_ptr(),
                                                    n, h, w, c, _lib.dtype_code(x.dtype), _lib.stream_ptr())
        _lib.check(rc, "sod_upsample2x_bilinear_fwd")
        _lib.count_launch()
        ctx.shape = (n, c, h, w)
        ctx.has_add = add is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        n, c, h, w = ctx.shape
        dy = _rows(dy)
        dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_upsample2x_bilinear_bwd(dy.data_ptr(), dx.data_ptr(), n, h, w, c, _lib.dtype_code(dy.dtype),
                                                    _lib.stream_ptr())
        _lib.check(rc, "sod_upsample2x_bilinear_bwd")
        _lib.count_launch()
        return dx, (dy if ctx.has_add else None)


class _AvgPool2x2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _rows(x)
        n, c, h, w = x.shape
        y = torch.empty((n, c, h // 2, w // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_avgpool2x2_fwd(x.data_ptr(), y.data_ptr(), n, h // 2, w // 2, c, _lib.dtype_code(x.dtype), _lib.stream_ptr())
        _lib.check(rc, "sod_avgpool2x2_fwd")
        _lib.count_launch()
        ctx.shape = (n, c, h, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        n, c, h, w = ctx.shape
        dy = _rows(dy)
        dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_avgpool2x2_bwd(dy.data_ptr(), dx.data_ptr(), n, h // 2, w // 2, c, _lib.dtype_code(dy.dtype), _lib.stream_ptr())
        _lib.check(rc, "sod_avgpool2x2_bwd")
        _lib.count_launch()
        return dx


def upsample2x(x: torch.Tensor, out_hw) -> torch.Tensor | None:
    """bilinear to `out_hw` if that is exactly twice the input size, else None (caller falls back to F.interpolate)"""
    if not _ok(x) or tuple(out_hw) != (2 * x.shape[2], 2 * x.shape[3]):
        return None
    return _Up2x.apply(x, None)


def upsample2x_add(coarse: torch.Tensor, lateral: torch.Tensor) -> torch.Tensor | None:
    """lateral + bilinear(coarse → lateral's size), one kernel; None if not exactly ×2"""
    if not _ok(coarse) or tuple(lateral.shape[2:]) != (2 * coarse.shape[2], 2 * coarse.shape[3]) \
            or lateral.shape[:2] != coarse.shape[:2] or lateral.dtype != coarse.dtype:
        return None
    return _Up2x.apply(coarse, lateral)


def avgpool2x2(x: torch.Tensor) -> torch.Tensor | None:
    if not _ok(x) or x.shape[2] % 2 or x.shape[3] % 2:
        return None
    return _AvgPool2x2.apply(x)


class _UpNearest2x(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _rows(x)
        n, c, h, w = x.shape
        y = torch.empty((n, c, 2 * h, 2 * w), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_upsample2x_nearest_fwd(x.data_ptr(), y.data_ptr(), n, h, w, c, _lib.dtype_code(x.dtype), _lib.stream_ptr())
        _lib.check(rc, "sod_upsample2x_nearest_fwd")
        _lib.count_launch()
        ctx.shape = (n, c, h, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        n, c, h, w = ctx.shape
        dy = _rows(dy)
        dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_upsample2x_nearest_bwd(dy.data_ptr(), dx.data_ptr(), n, h, w, c, _lib.dtype_code(dy.dtype), _lib.stream_ptr())
        _lib.check(rc, "sod_upsample2x_nearest_bwd")
        _lib.count_launch()
        return dx


def upsample2x_nearest(x: torch.Tensor) -> torch.Tensor | None:
    """`nn.Upsample(scale_factor=2, mode="nearest")` of the LightAIM neck, in x's dtype; None where the kernels do not
    cover x (caller falls back to F.interpolate)"""
    if not _ok(x):
        return None
    return _UpNearest2x.apply(x)


class _MaxPool3x3s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _rows(x)
        n, c, h, w = x.shape
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        y = torch.empty((n, c, ho, wo), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        arg = torch.empty(n * ho * wo * c, dtype=torch.uint8, device=x.device)      # window position kh*3+kw per element
        rc = _lib.lib().sod_maxpool3x3s2_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), n, h, w, c, _lib.dtype_code(x.dtype),
                                             _lib.stream_ptr())
        _lib.check(rc, "sod_maxpool3x3s2_fwd")
        _lib.count_launch()
        ctx.shape = (n, c, h, w)
        ctx.save_for_backward(arg)
        return y

    @staticmethod
    def backward(ctx, dy):
        (arg,) = ctx.saved_tensors
        n, c, h, w = ctx.shape
        dy = _rows(dy)
        dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_maxpool3x3s2_bwd(dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), n, h, w, c, _lib.dtype_code(dy.dtype),
                                             _lib.stream_ptr())
        _lib.check(rc, "sod_maxpool3x3s2_bwd")
        _lib.count_launch()
        return dx


def maxpool3x3s2(x: torch.Tensor) -> torch.Tensor | None:
    """MaxPool2d(3, stride 2, padding 1); None (caller keeps the torch op) when the kernel is switched off or does not cover x"""
    if not (MAXPOOL_ENABLED and _ok(x)):
        return None
    return _MaxPool3x3s2.apply(x)


class _MaxPool2x2s2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _rows(x)
        n, c, h, w = x.shape
        y = torch.empty((n, c, h // 2, w // 2), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
        arg = torch.empty(y.numel(), dtype=torch.uint8, device=x.device)      # window position kh*2+kw per element
        rc = _lib.lib().sod_maxpool2x2s2_fwd(x.data_ptr(), y.data_ptr(), arg.data_ptr(), n, h, w, c, _lib.dtype_code(x.dtype),
                                             _lib.stream_ptr())
        _lib.check(rc, "sod_maxpool2x2s2_fwd")
        _lib.count_launch()
        ctx.shape = (n, c, h, w)
        ctx.save_for_backward(arg)
        return y

    @staticmethod
    def backward(ctx, dy):
        (arg,) = ctx.saved_tensors
        n, c, h, w = ctx.shape
        dy = _rows(dy)
        dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
        rc = _lib.lib().sod_maxpool2x2s2_bwd(dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), n, h, w, c, _lib.dtype_code(dy.dtype),
                                             _lib.stream_ptr())
        _lib.check(rc, "sod_maxpool2x2s2_bwd")
        _lib.count_launch()
        return dx


def maxpool2x2s2(x: torch.Tensor) -> torch.Tensor | None:
    """MaxPool2d(2, stride 2) of VGG16-BN, floor mode; None (caller keeps the torch op) when the kernel is switched off or
    does not cover x"""
    if not (MAXPOOL_ENABLED and _ok(x)) or x.shape[2] < 2 or x.shape[3] < 2:
        return None
    return _MaxPool2x2s2.apply(x)


# ---- convolution whose bias gradient is a deterministic column sum (csrc/resample.cu: sod_colsum) ------------------------
_colsum_ws: dict = {}


def colsum(x: torch.Tensor) -> torch.Tensor:
    """Σ over N, H, W of a channels-last [N,C,H,W] tensor → [C] (same dtype)"""
    x = _rows(x)
    n, c, h, w = x.shape
    ws = _colsum_ws.get(x.device.index)
    if ws is None:
        ws = _colsum_ws[x.device.index] = torch.zeros(int(_lib.lib().sod_colsum_workspace_bytes()), dtype=torch.uint8, device=x.device)
    out = torch.empty(c, dtype=x.dtype, device=x.device)
    rc = _lib.lib().sod_colsum(x.data_ptr(), out.data_ptr(), n * h * w, c, _lib.dtype_code(x.dtype), ws.data_ptr(), ws.numel(),
                               _lib.stream_ptr())
    _lib.check(rc, "sod_colsum")
    _lib.count_launch()
    return out


class _ConvBias(torch.autograd.Function):
    """conv2d with bias (cuDNN fuses the bias add into the forward); backward = cuDNN dgrad/wgrad + `colsum` for the bias"""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding, dilation, groups):
        y = torch.nn.functional.conv2d(x, weight, bias, stride, padding, dilation, groups)
        ctx.conf = (stride, padding, dilation, groups)
        ctx.save_for_backward(x if x.dtype == y.dtype else x.to(y.dtype), weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        stride, padding, dilation, groups = ctx.conf
        dx, dw, _ = torch.ops.aten.convolution_backward(dy, x, weight, None, list(stride), list(padding), list(dilation), False, [0, 0],
                                                        groups, [ctx.needs_input_grad[0], ctx.needs_input_grad[1], False])
        db = colsum(dy).to(weight.dtype) if ctx.needs_input_grad[2] else None
        return dx, dw, db, None, None, None, None


def conv_bias(conv: torch.nn.Conv2d, x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor) -> torch.Tensor | None:
    """`conv(x)` with the bias gradient taken by `colsum`; None when the kernel does not cover the case"""
    c = weight.shape[0]
    if not (ENABLED and COLSUM_ENABLED and x.is_cuda and bias is not None and c % 8 == 0 and c <= 2048 and (c // 8) & (c // 8 - 1) == 0
            and x.dtype in (torch.bfloat16, torch.float16, torch.float32) and weight.dtype == x.dtype and torch.is_grad_enabled()):
        return None
    return _ConvBias.apply(x, weight, bias, conv.stride, conv.padding, conv.dilation, conv.groups)
