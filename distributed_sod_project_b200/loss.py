"""Loss seam of the reference, backed by the fused sm_90a kernel (csrc/loss.cu).

Reference surface kept (paths in the reference repo):
* `BCEWithLogitsLoss(reduction=...)`  — train.py:203
* `CEL()`                              — loss/CEL.py:10-23 (eps 1e-6, `__str__`)
* `get_total_loss(preds, masks, loss_funcs) -> (Tensor, list[str])` — utils/pipeline_ops.py:19-43

`get_total_loss` recognises the reference's `[BCEWithLogitsLoss, CEL]` list and issues ONE kernel that
produces both values and d(total)/d(logits); each loss object also works on its own (the kernel runs
with the other weight at 0).  Both report strings come from one 32-byte device→host copy instead of
one `.item()` sync per loss.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib

_workspaces: dict = {}


def _workspace(device: torch.device) -> torch.Tensor:
    key = ("loss", device.index, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None:
        ws = torch.zeros(_lib.lib().sod_loss_workspace_bytes(), dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def bce_cel_fwd_bwd(logits: torch.Tensor, mask: torch.Tensor, *, reduction: str = "mean", w_bce: float = 1.0,
                    w_cel: float = 1.0, grad_scale: float = 1.0, eps: float = 1e-6, mode: int = 0,
                    grad_scale_dev: torch.Tensor | None = None):
    """Raw call into `sod_loss_bce_cel_fwd_bwd`. Returns (scalars[8] fp32 device tensor, grad like logits).
    scalars = [bce, cel, total, Σp, Σt, Σp·t, bce_sum, n].  grad_scale_dev (fp32 device scalar, e.g. the amp loss scale):
    the gradient is multiplied by it before it is rounded to the logits dtype (`sod_loss_bce_cel_fwd_bwd_scaled`)."""
    if not logits.is_cuda:
        raise _lib.SodError("the fused BCE+CEL loss runs on CUDA tensors only (no CPU fallback)")
    if reduction not in ("mean", "sum"):
        raise ValueError(f"reduction must be 'mean' or 'sum', got {reduction!r}")
    if logits.shape != mask.shape:
        raise ValueError(f"logits {tuple(logits.shape)} and mask {tuple(mask.shape)} differ in shape")
    x = logits.detach()
    # any dense layout is fine for an elementwise+global-sum loss as long as x, mask and grad share it
    if not (x.is_contiguous() or x.is_contiguous(memory_format=torch.channels_last)):
        x = x.contiguous()
    m = mask.detach()
    if m.dtype not in (torch.float32, x.dtype):
        m = m.float()
    if m.stride() != x.stride():
        m = m.contiguous() if x.is_contiguous() else m.contiguous(memory_format=torch.channels_last)
    grad = torch.empty_like(x)
    scalars = torch.empty(8, dtype=torch.float32, device=x.device)
    ws = _workspace(x.device)
    if grad_scale_dev is not None:
        if grad_scale_dev.dtype != torch.float32 or grad_scale_dev.numel() != 1 or grad_scale_dev.device != x.device:
            raise _lib.SodError("grad_scale_dev must be one fp32 element on the logits' device")
        rc = _lib.lib().sod_loss_bce_cel_fwd_bwd_scaled(
            x.data_ptr(), _lib.dtype_code(x.dtype), m.data_ptr(), _lib.dtype_code(m.dtype), grad.data_ptr(),
            _lib.dtype_code(x.dtype), scalars.data_ptr(), x.numel(), 1 if reduction == "sum" else 0,
            float(w_bce), float(w_cel), float(grad_scale), grad_scale_dev.data_ptr(), float(eps), int(mode), ws.data_ptr(),
            ws.numel(), _lib.stream_ptr())
        _lib.check(rc, "sod_loss_bce_cel_fwd_bwd_scaled")
        _lib.count_launch()
        return scalars, grad
    rc = _lib.lib().sod_loss_bce_cel_fwd_bwd(
        x.data_ptr(), _lib.dtype_code(x.dtype), m.data_ptr(), _lib.dtype_code(m.dtype), grad.data_ptr(),
        _lib.dtype_code(x.dtype), scalars.data_ptr(), x.numel(), 1 if reduction == "sum" else 0,
        float(w_bce), float(w_cel), float(grad_scale), float(eps), int(mode), ws.data_ptr(), ws.numel(),
        _lib.stream_ptr())
    _lib.check(rc, "sod_loss_bce_cel_fwd_bwd")
    _lib.count_launch()
    return scalars, grad


class _FusedLossFn(torch.autograd.Function):
    """apply(logits, mask, reduction, w_bce, w_cel, eps, unit_upstream, mode, holder[, scale_dev]).

    scale_dev (optional, fp32 0-d device tensor — the amp loss scale): the gradient is formed as scale_dev × d total/d logits
    and rounded once, and backward hands it to autograd untouched.  Contract: `.backward()` is called on
    `total * scale_dev` with that same tensor (what `amp.scale_loss` yields), so the upstream gradient IS scale_dev."""

    @staticmethod
    def forward(ctx, logits, mask, reduction, w_bce, w_cel, eps, unit_upstream, mode, holder, *scale_dev):
        sdev = scale_dev[0] if scale_dev else None
        scalars, grad = bce_cel_fwd_bwd(logits, mask, reduction=reduction, w_bce=w_bce, w_cel=w_cel, eps=eps, mode=mode,
                                        grad_scale_dev=sdev)
        ctx.save_for_backward(grad)
        ctx.unit_upstream = unit_upstream or sdev is not None
        ctx.n_extra = len(scale_dev)
        holder.append(scalars)          # side channel: the 8 report scalars, no extra kernel
        return scalars[2]               # 0-d view of the kernel's output buffer

    @staticmethod
    def backward(ctx, g_total):
        (grad,) = ctx.saved_tensors
        if not ctx.unit_upstream:
            # general case: the loss was scaled / combined further downstream
            g = g_total.detach().reshape(1).float().contiguous()
            rc = _lib.lib().sod_scale_by_device_scalar(grad.data_ptr(), _lib.dtype_code(grad.dtype), grad.numel(),
                                                       g.data_ptr(), _lib.stream_ptr())
            _lib.check(rc, "sod_scale_by_device_scalar")
            _lib.count_launch()
        return (grad,) + (None,) * (8 + ctx.n_extra)


class FusedBCECEL(nn.Module):
    """total = w_bce * BCEWithLogits(reduction) + w_cel * CEL, one kernel for value and gradient.

    `unit_upstream=True` promises that `.backward()` is called directly on the returned total (or on a sum
    it enters with weight 1), which lets backward hand the precomputed gradient to autograd untouched."""

    def __init__(self, reduction: str = "mean", w_bce: float = 1.0, w_cel: float = 1.0, eps: float = 1e-6,
                 unit_upstream: bool = False, mode: int = 0):
        super().__init__()
        self.reduction, self.w_bce, self.w_cel, self.eps = reduction, w_bce, w_cel, eps
        self.unit_upstream, self.mode = unit_upstream, mode
        self.last_scalars: torch.Tensor | None = None

    def forward(self, pred: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        holder: list = []
        total = _FusedLossFn.apply(pred, target, self.reduction, self.w_bce, self.w_cel, self.eps,
                                   self.unit_upstream, self.mode, holder)
        self.last_scalars = holder[0]
        return total


class BCEWithLogitsLoss(FusedBCECEL):
    """Stand-in for torch.nn.BCEWithLogitsLoss at reference train.py:203."""

    def __init__(self, reduction: str = "mean", **kw):
        super().__init__(reduction=reduction, w_bce=1.0, w_cel=0.0, **kw)


class CEL(FusedBCECEL):
    """Stand-in for the reference loss/CEL.py:10-23."""

    def __init__(self, **kw):
        super().__init__(reduction="mean", w_bce=0.0, w_cel=1.0, **kw)

    def __str__(self):
        return "You are using `CEL`!"


def _as_pair(loss_funcs):
    """(reduction, eps) if the list is the reference's [BCEWithLogits, CEL] pair, else None."""
    if len(loss_funcs) != 2:
        return None
    a, b = loss_funcs
    is_bce = isinstance(a, BCEWithLogitsLoss) or (isinstance(a, nn.BCEWithLogitsLoss) and a.weight is None
                                                   and a.pos_weight is None)
    is_cel = isinstance(b, CEL) or (type(b).__name__ == "CEL" and hasattr(b, "eps"))
    if not (is_bce and is_cel) or a.reduction not in ("mean", "sum"):
        return None
    return a.reduction, float(getattr(b, "eps", 1e-6))


def get_total_loss(train_preds: torch.Tensor, train_masks: torch.Tensor, loss_funcs: list,
                   unit_upstream: bool = False, scale_dev: torch.Tensor | None = None):
    """Signature and return contract of reference utils/pipeline_ops.py:19-43.  scale_dev: the amp loss scale the fused
    pair's gradient is formed with (see `_FusedLossFn`); backward must then run on `total * scale_dev`."""
    assert len(loss_funcs) != 0, "请指定损失函数`loss_funcs`"
    pair = _as_pair(loss_funcs) if train_preds.is_cuda else None
    if pair is not None:
        reduction, eps = pair
        holder: list = []
        extra = (scale_dev,) if scale_dev is not None else ()
        total = _FusedLossFn.apply(train_preds, train_masks, reduction, 1.0, 1.0, eps, unit_upstream, 0, holder, *extra)
        host = holder[0][:2].tolist()          # one 8-byte D2H + one sync for both report strings
        return total, [f"{host[0]:.5f}", f"{host[1]:.5f}"]
    loss_list, items = [], []
    for loss in loss_funcs:
        out = loss(train_preds, train_masks)
        loss_list.append(out)
        items.append(f"{out.item():.5f}")
    return sum(loss_list), items
