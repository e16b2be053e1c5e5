"""Restatement of the nearest ×2 kernels of csrc/resample.cu (`sod_upsample2x_nearest_fwd` / `_bwd`) that
tests/test_aim_cpu.py and tests/test_gpu_upsample_nearest.py compare against.  Not a test module.

Forward: out[2i + a][2j + b] = in[i][j].  Backward: dx[i][j] = (((0 + dy[2i][2j]) + dy[2i][2j+1]) + dy[2i+1][2j]) +
dy[2i+1][2j+1], each add in fp32, rounded once to the gradient's dtype.  Elementwise fp32 adds round the same on every
IEEE device, so this CPU form is bit-exact against the kernel."""
from __future__ import annotations

import torch


def upsample2x_nearest_fwd(x: torch.Tensor) -> torch.Tensor:
    """[N, C, H, W] → [N, C, 2H, 2W], every value copied"""
    return x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)


def upsample2x_nearest_bwd(dy: torch.Tensor) -> torch.Tensor:
    """[N, C, 2H, 2W] → [N, C, H, W] in dy's dtype, the four taps summed in the kernel's order in fp32"""
    d = dy.float()
    acc = torch.zeros_like(d[:, :, 0::2, 0::2])
    for a, b in ((0, 0), (0, 1), (1, 0), (1, 1)):
        acc = acc + d[:, :, a::2, b::2]
    return acc.to(dy.dtype)


def upsample2x_nearest_bwd64(dy: torch.Tensor) -> torch.Tensor:
    """the same sum in float64, unrounded"""
    d = dy.double()
    return d[:, :, 0::2, 0::2] + d[:, :, 0::2, 1::2] + d[:, :, 1::2, 0::2] + d[:, :, 1::2, 1::2]
