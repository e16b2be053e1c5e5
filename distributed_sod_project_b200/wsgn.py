"""GroupNorm / weight-standardisation seam of the WS-GN backbone (`wsgn_res50`, `cp_wsgn_res50`), backed by csrc/wsgn.cu.

`convert_wsgn_model(model)` walks the module tree like `convert_syncbn_model` and swaps
* every affine `nn.GroupNorm` with 32 groups for `GroupNorm32` (other GroupNorms stay torch modules), whose
  `fused_forward(x, residual=, relu=)` runs GroupNorm(32) with the bottleneck's residual add and ReLU as one kernel pair
  per direction (the model's `bn_act` drives it unchanged);
* every `network.blocks.WSConv2d` for `FusedWSConv2d`, which standardises its fp32 master weight with one kernel per
  direction and hands the convolution Ŵ in the convolution's dtype (under autocast: rounded once from fp32, as apex O1
  standardises in fp32 and casts afterwards).  The ResNeXt backbone's 32-group 3×3 convolutions run on the
  csrc/gconv.cu kernels where those measured faster than cuDNN (`grouped_conv_on_kernels`), their fp32 weight
  gradient going straight into the standardisation's backward, and on cuDNN elsewhere; a grouped WS convolution outside
  the kernels' geometry raises SodError.
The swapped modules SHARE the original Parameter objects, so an optimizer built before the conversion keeps training
them.  Models without GroupNorm or WS convolutions come back untouched.  There is no CPU or torch fallback: a CPU tensor
or a shape the kernels do not cover raises SodError.

Both backward kernels add the parameter gradients straight into a bound fp32 `.grad` (FusedSGD / FusedAdam's flat
buffer) when there is one, and bump `_lib.grad_writes` so `zero_grad` sees the write.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib
from .network.blocks import WSConv2d

# one workspace per device and user ("groupnorm": zero-filled tickets the kernels keep at zero; "gconv": the grouped
# convolutions' wgrad partials), grown when a larger shape arrives; outgrown buffers are kept alive because a captured
# CUDA graph may still hold their address
_workspaces: dict = {}


def _workspace(device: torch.device, nbytes: int, user: str = "groupnorm") -> torch.Tensor:
    bufs = _workspaces.setdefault((device.index, user), [])
    if not bufs or bufs[-1].numel() < nbytes:
        if torch.cuda.is_current_stream_capturing():
            raise _lib.SodError(f"{user} workspace of {nbytes} bytes needed while a CUDA graph is being captured; "
                                "run the shape eagerly once first")
        bufs.append(torch.zeros(max(nbytes, 1 << 20), dtype=torch.uint8, device=device))
    return bufs[-1]


def _as_rows(t: torch.Tensor) -> torch.Tensor:
    return t if t.is_contiguous(memory_format=torch.channels_last) else t.contiguous(memory_format=torch.channels_last)


def _bound_fp32_grad(p: torch.Tensor) -> torch.Tensor | None:
    g = getattr(p, "grad", None)
    if g is not None and p.requires_grad and g.dtype == torch.float32 and g.stride() == p.stride():
        return g
    return None


class _GroupNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, eps, relu):
        x = _as_rows(x)
        res = _as_rows(residual).to(x.dtype) if residual is not None else None
        n, c, h, w = x.shape
        nbytes = int(_lib.lib().sod_groupnorm_workspace_bytes(n, h * w, c, _lib.SOD_GN_GROUPS))
        if nbytes == 0:
            raise _lib.SodError(f"GroupNorm(32) kernels do not cover the shape [N={n}, C={c}, H={h}, W={w}] (C must be "
                                "a power-of-two multiple of 8 from 32 to 2048, N at most 65535)")
        ws = _workspace(x.device, nbytes)
        y = torch.empty_like(x)
        stats = torch.empty(n * _lib.SOD_GN_GROUPS * 2, dtype=torch.float32, device=x.device)
        rc = _lib.lib().sod_groupnorm_fwd(
            x.data_ptr(), res.data_ptr() if res is not None else None, y.data_ptr(), _lib.dtype_code(x.dtype),
            weight.data_ptr(), bias.data_ptr(), stats.data_ptr(), n, h * w, c, _lib.SOD_GN_GROUPS, float(eps), int(relu),
            ws.data_ptr(), ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "sod_groupnorm_fwd")
        _lib.count_launch(2)
        ctx.relu, ctx.has_res = bool(relu), res is not None
        ctx.weight_ref, ctx.bias_ref = weight, bias
        ctx.save_for_backward(x, y if relu else None, weight, stats)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, weight, stats = ctx.saved_tensors
        n, c, h, w = x.shape
        dy = _as_rows(dy).to(x.dtype)
        wg, bg = _bound_fp32_grad(ctx.weight_ref), _bound_fp32_grad(ctx.bias_ref)
        direct = wg is not None and bg is not None
        if direct:
            dgamma, dbeta, flags = wg, bg, _lib.SOD_BN_ACCUMULATE_PARAM_GRADS
            _lib.grad_writes += 1          # bound .grad buffers change behind autograd's back (FusedSGD.zero_grad looks at this)
        else:
            dgamma = torch.empty(c, dtype=torch.float32, device=x.device)
            dbeta = torch.empty(c, dtype=torch.float32, device=x.device)
            flags = 0
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_res else None
        ws = _workspace(x.device, int(_lib.lib().sod_groupnorm_workspace_bytes(n, h * w, c, _lib.SOD_GN_GROUPS)))
        rc = _lib.lib().sod_groupnorm_bwd(
            dy.data_ptr(), x.data_ptr(), y.data_ptr() if y is not None else None, dx.data_ptr(),
            dres.data_ptr() if dres is not None else None, _lib.dtype_code(x.dtype), weight.data_ptr(), stats.data_ptr(),
            dgamma.data_ptr(), dbeta.data_ptr(), n, h * w, c, _lib.SOD_GN_GROUPS, int(ctx.relu), ws.data_ptr(), ws.numel(),
            flags, _lib.stream_ptr())
        _lib.check(rc, "sod_groupnorm_bwd")
        _lib.count_launch(2)
        gw, gb = (None, None) if direct else (dgamma.to(weight.dtype), dbeta.to(weight.dtype))
        return dx, dres, gw, gb, None, None


def group_norm(x, weight, bias, eps: float = 1e-5, residual=None, relu: bool = False) -> torch.Tensor:
    """y = act(GroupNorm(32)(x) [+ residual]) on the sm_90a kernels (CUDA, 4-D; fp32 γ/β)"""
    if not x.is_cuda:
        raise _lib.SodError("GroupNorm32: expected a CUDA tensor (the sm_90a kernel has no CPU fallback; keep nn.GroupNorm "
                            "for CPU runs)")
    if x.dim() != 4:
        raise _lib.SodError(f"GroupNorm32 expects 4-D input, got {x.dim()}-D")
    if weight.dtype != torch.float32 or bias.dtype != torch.float32:
        raise _lib.SodError(f"GroupNorm32 expects fp32 affine parameters, got {weight.dtype}")
    return _GroupNormFn.apply(x, residual, weight, bias, eps, relu)


class GroupNorm32(nn.GroupNorm):
    """Drop-in for the backbone's `nn.GroupNorm(32, C)` that `convert_wsgn_model` installs."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.fused_forward(x)

    def fused_forward(self, x, pre_add=None, residual=None, relu=False, conv_bias=(None, None)):
        """the `bn_act` entry: y = act(GN(x) [+ residual]); the decoder-only operands (pre_add, folded conv biases) are
        not part of this layer's uses and are refused"""
        if pre_add is not None or any(b is not None for b in conv_bias):
            raise _lib.SodError("GroupNorm32.fused_forward: pre_add / conv_bias are not supported")
        if self.num_groups != _lib.SOD_GN_GROUPS or not self.affine:
            raise _lib.SodError(f"GroupNorm32: only affine GroupNorm with {_lib.SOD_GN_GROUPS} groups is on the hot path")
        return group_norm(x, self.weight, self.bias, self.eps, residual=residual, relu=relu)


class _WSFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weight, dtype, eps):
        w_hat = torch.empty_like(weight, dtype=dtype)              # the master's (dense) memory order
        rc = _lib.lib().sod_ws_fwd(weight.data_ptr(), w_hat.data_ptr(), _lib.dtype_code(dtype), weight.shape[0],
                                   weight[0].numel(), float(eps), _lib.stream_ptr())
        _lib.check(rc, "sod_ws_fwd")
        _lib.count_launch()
        ctx.eps = eps
        ctx.weight_ref = weight
        ctx.save_for_backward(weight)
        return w_hat

    @staticmethod
    def backward(ctx, dw_hat):
        (weight,) = ctx.saved_tensors
        if dw_hat.stride() != weight.stride():
            dw_hat = torch.empty_like(weight, dtype=dw_hat.dtype).copy_(dw_hat)
        bound = _bound_fp32_grad(ctx.weight_ref)
        if bound is not None:
            dw, flags = bound, _lib.SOD_BN_ACCUMULATE_PARAM_GRADS
            _lib.grad_writes += 1
        else:
            dw, flags = torch.empty_like(weight, dtype=torch.float32), 0
        rc = _lib.lib().sod_ws_bwd(weight.data_ptr(), dw_hat.data_ptr(), _lib.dtype_code(dw_hat.dtype), dw.data_ptr(),
                                   weight.shape[0], weight[0].numel(), float(ctx.eps), flags, _lib.stream_ptr())
        _lib.check(rc, "sod_ws_bwd")
        _lib.count_launch()
        return (None if bound is not None else dw.to(weight.dtype)), None, None


def standardize_weight(weight: torch.Tensor, dtype: torch.dtype, eps: float = 1e-5) -> torch.Tensor:
    """Ŵ = (W − mean) / (std + eps) per filter, written in `dtype` from the fp32 master (CUDA only)"""
    if not weight.is_cuda:
        raise _lib.SodError("weight standardisation: expected a CUDA tensor (the sm_90a kernel has no CPU fallback)")
    if weight.dtype != torch.float32:
        raise _lib.SodError(f"weight standardisation reads an fp32 master weight, got {weight.dtype}")
    if weight[0].numel() < 2 or not (weight.is_contiguous() or weight.is_contiguous(memory_format=torch.channels_last)):
        raise _lib.SodError(f"weight standardisation does not cover the weight of shape {tuple(weight.shape)} and strides "
                            f"{weight.stride()} (each filter must be dense, with at least 2 elements)")
    return _WSFn.apply(weight, dtype, eps)


class _WSGroupConvFn(torch.autograd.Function):
    """y = conv3x3(x, WS(weight), groups=32, padding 1, stride s) on csrc/gconv.cu; the backward hands the fp32 dŴ of
    the wgrad kernel to sod_ws_bwd unrounded (an autograd edge between two Functions would round it to Ŵ's dtype)"""

    @staticmethod
    def forward(ctx, x, weight, dtype, eps, stride):
        x = _as_rows(x).to(dtype)
        n, c, h, w = x.shape
        w_hat = torch.empty_like(weight, dtype=dtype)              # the master's memory order
        rc = _lib.lib().sod_ws_fwd(weight.data_ptr(), w_hat.data_ptr(), _lib.dtype_code(dtype), weight.shape[0],
                                   weight[0].numel(), float(eps), _lib.stream_ptr())
        _lib.check(rc, "sod_ws_fwd")
        w_hat = _as_rows(w_hat)                                    # [C_out][3][3][C_in / 32], the kernels' order
        y = torch.empty((n, c, (h - 1) // stride + 1, (w - 1) // stride + 1), dtype=dtype, device=x.device,
                        memory_format=torch.channels_last)
        rc = _lib.lib().sod_gconv3x3_fwd(x.data_ptr(), w_hat.data_ptr(), y.data_ptr(), _lib.dtype_code(dtype), n, h, w,
                                         c, _lib.SOD_GCONV_GROUPS, stride, _lib.stream_ptr())
        _lib.check(rc, "sod_gconv3x3_fwd")
        _lib.count_launch(2)
        ctx.eps, ctx.stride, ctx.weight_ref = eps, stride, weight
        ctx.save_for_backward(x, weight, w_hat)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, w_hat = ctx.saved_tensors
        n, c, h, w = x.shape
        dy = _as_rows(dy).to(x.dtype)
        code, G, s, lib = _lib.dtype_code(x.dtype), _lib.SOD_GCONV_GROUPS, ctx.stride, _lib.lib()
        dx = torch.empty_like(x)
        _lib.check(lib.sod_gconv3x3_dgrad(dy.data_ptr(), w_hat.data_ptr(), dx.data_ptr(), code, n, h, w, c, G, s,
                                          _lib.stream_ptr()), "sod_gconv3x3_dgrad")
        dw_hat = torch.empty(weight.shape, dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
        ws = _workspace(x.device, int(lib.sod_gconv3x3_wgrad_workspace_bytes(n, h, w, c, G, s)), "gconv")
        _lib.check(lib.sod_gconv3x3_wgrad(x.data_ptr(), dy.data_ptr(), dw_hat.data_ptr(), code, n, h, w, c, G, s,
                                          ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "sod_gconv3x3_wgrad")
        if dw_hat.stride() != weight.stride():
            dw_hat = torch.empty_like(weight, dtype=torch.float32).copy_(dw_hat)
        bound = _bound_fp32_grad(ctx.weight_ref)
        if bound is not None:
            dw, flags = bound, _lib.SOD_BN_ACCUMULATE_PARAM_GRADS
            _lib.grad_writes += 1
        else:
            dw, flags = torch.empty_like(weight, dtype=torch.float32), 0
        _lib.check(lib.sod_ws_bwd(weight.data_ptr(), dw_hat.data_ptr(), _lib.SOD_F32, dw.data_ptr(), weight.shape[0],
                                  weight[0].numel(), float(ctx.eps), flags, _lib.stream_ptr()), "sod_ws_bwd")
        _lib.count_launch(4)
        return dx, (None if bound is not None else dw.to(weight.dtype)), None, None, None


def grouped_conv_covered(conv: nn.Conv2d) -> bool:
    """the geometry of csrc/gconv.cu: 32 groups of 4, 8, 16 or 32 channels, C_in = C_out, 3×3, padding 1, dilation 1,
    stride 1 or 2, no bias"""
    cpg = conv.in_channels // conv.groups
    return (conv.groups == _lib.SOD_GCONV_GROUPS and conv.in_channels == conv.out_channels and cpg in (4, 8, 16, 32)
            and conv.kernel_size == (3, 3) and conv.padding == (1, 1) and conv.dilation == (1, 1)
            and conv.stride in ((1, 1), (2, 2)) and conv.bias is None and conv.padding_mode == "zeros")


def grouped_conv_on_kernels(conv: nn.Conv2d) -> bool:
    """which covered grouped convolutions run on csrc/gconv.cu rather than cuDNN: measured per shape on an H100
    (DESIGN §4.13, tools/bench_wsgn.py --model wsgn_resnext50), fwd + dgrad + wgrad of the kernels beat cuDNN only at
    8 channels per group and stride 2 (layer2.0), where cuDNN's dgrad is 3.6× slower; at every other shape of the
    backbone cuDNN's grouped kernels are 1.3–8.5× faster than these"""
    return conv.in_channels // conv.groups == 8 and conv.stride == (2, 2)


class FusedWSConv2d(WSConv2d):
    """Drop-in for `WSConv2d` that `convert_wsgn_model` installs: the standardisation runs as sm_90a kernels, and so
    does a 32-group 3×3 convolution where they beat cuDNN (`grouped_conv_on_kernels`)."""

    def forward(self, x):
        if not x.is_cuda:
            raise _lib.SodError("FusedWSConv2d: expected a CUDA tensor (keep network.blocks.WSConv2d for CPU runs)")
        dtype = torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else self.weight.dtype
        if self.groups != 1:
            if not grouped_conv_covered(self) or x.dim() != 4 or self.weight.dtype != torch.float32:
                raise _lib.SodError(
                    f"FusedWSConv2d: the grouped-convolution kernels do not cover groups={self.groups}, "
                    f"{self.in_channels}->{self.out_channels} channels, kernel {self.kernel_size}, stride {self.stride}, "
                    f"padding {self.padding}, dilation {self.dilation}, bias={self.bias is not None}, "
                    f"{x.dim()}-D {x.dtype} input, {self.weight.dtype} weight (32 groups of 4/8/16/32 channels, 3x3, "
                    "padding 1, stride 1 or 2, no bias, fp32 master weight)")
            if grouped_conv_on_kernels(self):
                return _WSGroupConvFn.apply(x, self.weight, dtype, self.eps, self.stride[0])
        return self._conv_forward(x, standardize_weight(self.weight, dtype, self.eps), self.bias)


def _swap(module: nn.Module) -> nn.Module:
    if (isinstance(module, nn.GroupNorm) and not isinstance(module, GroupNorm32) and module.affine
            and module.num_groups == _lib.SOD_GN_GROUPS):
        new = GroupNorm32(module.num_groups, module.num_channels, module.eps, module.affine, device="meta")
        new.weight, new.bias = module.weight, module.bias                  # same Parameter objects
        new.train(module.training)
        return new
    if isinstance(module, WSConv2d) and not isinstance(module, FusedWSConv2d):
        # built on the meta device: no random draws, no storage; the Parameters are the original ones
        new = FusedWSConv2d(module.in_channels, module.out_channels, module.kernel_size, module.stride, module.padding,
                            module.dilation, module.groups, module.bias is not None, module.padding_mode, device="meta")
        new.weight, new.bias = module.weight, module.bias
        new.train(module.training)
        return new
    return module


def convert_wsgn_model(module: nn.Module) -> nn.Module:
    """the model with every affine 32-group `nn.GroupNorm` replaced by `GroupNorm32` and every `WSConv2d` by
    `FusedWSConv2d`, parameters shared with the originals.  A converted GroupNorm must then see 4-D input."""
    swapped = _swap(module)
    if swapped is not module:
        return swapped
    for name, child in list(module.named_children()):
        converted = convert_wsgn_model(child)
        if converted is not child:
            if isinstance(module, nn.Sequential):
                module[int(name)] = converted
            else:
                setattr(module, name, converted)
    return module
