"""amp seam: `amp.initialize`, `amp.scale_loss`, `amp.state_dict/load_state_dict` of the reference
(apex.amp O1; train.py:15,181-183,298-300, utils/pipeline_ops.py:74,121).

Default: bf16 autocast, loss scale fixed at 1.0 — bf16 has fp32's exponent range, so the dynamic
scaler of apex O1 has nothing to do; weights, gradients and optimizer state stay fp32 ("fp32 master") exactly
as under O1.  `dtype=torch.float16` keeps apex's dynamic-scale behaviour (init 2^16, ÷2 and skip the step on
overflow, ×2 every 2000 clean steps): the unscale factor and the overflow flag are consumed INSIDE the fused
optimizer kernel, the only extra work is one read of the gradients by `sod_grad_nonfinite`.
"""
from __future__ import annotations

import contextlib
import functools

import torch

from . import _lib
from .optim import FusedSGD

import os

# SOD_STEAL_WGRADS=0: bind every shadow leaf's .grad to the flat buffer (autograd then launches one add per tensor)
STEAL_WEIGHT_GRADS = os.environ.get("SOD_STEAL_WGRADS", "1") == "1"

_cfg = {"enabled": False, "dtype": torch.bfloat16, "scale": 1.0, "dynamic": False, "good_steps": 0,
        "growth_interval": 2000, "found_inf": None}


def _install_shadow_weights(model, flat) -> int:
    """Point every Conv2d whose parameters live in `flat` at the bf16 shadow copy: under autocast the convolution
    then takes its weight without a per-iteration cast kernel, and autograd accumulates the (bf16) weight gradient
    straight into the flat bf16 gradient buffer the fused step consumes.  fp32 masters stay the module Parameters
    (state_dict / checkpoints / optimizer groups are unaffected)."""
    import torch.nn as nn
    managed = {id(p) for p, _ in flat.slots}
    count = 0
    for m in model.modules():
        if not isinstance(m, nn.Conv2d) or id(m.weight) not in managed or hasattr(m, "_sod_w16"):
            continue
        w16 = flat.view16(flat.shadow16, m.weight)
        w16.requires_grad_(m.weight.requires_grad)
        if m.weight.requires_grad:
            # weights: `.grad` stays None — autograd then keeps cuDNN's wgrad tensor as it is and the fused step
            # gathers all of them with one launch (no per-parameter accumulate kernel at the end of backward)
            flat.shadow_leaves.append((w16, flat.offset_of(m.weight), STEAL_WEIGHT_GRADS))
            if not STEAL_WEIGHT_GRADS:
                w16.grad = flat.view16(flat.grad16, m.weight)
        m._sod_w16, m._sod_b16 = w16, None
        if m.bias is not None and id(m.bias) in managed:
            b16 = flat.view16(flat.shadow16, m.bias)
            b16.requires_grad_(m.bias.requires_grad)
            if m.bias.requires_grad:
                # biases: bound view — the SyncBN backward adds the folded-bias gradient straight into it
                b16.grad = flat.view16(flat.grad16, m.bias)
                flat.shadow_leaves.append((b16, flat.offset_of(m.bias), False))
            m._sod_b16 = b16
        elif m.bias is not None:
            continue

        def forward(x, m=m):
            if torch.is_autocast_enabled() and x.is_cuda:
                if m._sod_b16 is not None and m.padding_mode == "zeros" and x.dtype == m._sod_w16.dtype:
                    from . import resample
                    y = resample.conv_bias(m, x, m._sod_w16, m._sod_b16)     # bias gradient by sod_colsum
                    if y is not None:
                        return y
                return m._conv_forward(x, m._sod_w16, m._sod_b16)
            return m._conv_forward(x, m.weight, m.bias)         # eval / fp32 use: the master copy

        m.forward = forward
        count += 1
    def _seen(grad, flat=flat):
        flat.master_grads_seen = True          # a gradient reached an fp32 master: the bf16 buffer is no longer the whole story
        return grad

    for m in model.modules():
        if isinstance(m, nn.Conv2d) and hasattr(m, "_sod_w16"):
            for p in (m.weight, m.bias):
                if p is not None and id(p) in managed and p.requires_grad:
                    p.register_hook(_seen)
    model.register_load_state_dict_post_hook(lambda mod, incompatible: flat.refresh_shadow())
    return count


def initialize(model, optimizer=None, opt_level: str = "O1", dtype: torch.dtype = torch.bfloat16, shadow_weights: bool = True,
               **_ignored):
    """Returns (model, optimizer) like apex. The model's forward runs under autocast(dtype)."""
    if opt_level not in ("O0", "O1"):
        raise _lib.SodError(f"opt_level {opt_level!r}: only O0/O1 semantics are provided")
    _cfg["enabled"] = opt_level == "O1"
    _cfg["dtype"] = dtype
    _cfg["dynamic"] = _cfg["enabled"] and dtype == torch.float16
    _cfg["scale"] = 65536.0 if _cfg["dynamic"] else 1.0
    if _cfg["enabled"]:
        inner = model.forward

        @functools.wraps(inner)
        def autocast_forward(*a, **k):
            with torch.autocast("cuda", dtype=_cfg["dtype"]):
                return inner(*a, **k)

        model.forward = autocast_forward
        if shadow_weights and dtype == torch.bfloat16 and isinstance(optimizer, FusedSGD) and optimizer.flat.param.is_cuda:
            optimizer.flat.enable_shadow(dtype)
            _install_shadow_weights(model, optimizer.flat)
    return (model, optimizer) if optimizer is not None else model


@contextlib.contextmanager
def scale_loss(loss, optimizer):
    """`with amp.scale_loss(loss, optimizer) as scaled: scaled.backward()` (reference train.py:299)."""
    if not _cfg["dynamic"]:
        yield loss
        return
    if not isinstance(optimizer, FusedSGD):
        raise _lib.SodError("fp16 dynamic loss scaling is wired into FusedSGD only")
    scale = _cfg["scale"]
    yield loss * scale
    flat = optimizer.flat
    if _cfg["found_inf"] is None:
        _cfg["found_inf"] = torch.zeros(1, dtype=torch.int32, device=flat.grad.device)
    finf = _cfg["found_inf"]
    finf.zero_()
    rc = _lib.lib().sod_grad_nonfinite(flat.grad.data_ptr(), flat.numel, finf.data_ptr(), _lib.stream_ptr())
    _lib.check(rc, "sod_grad_nonfinite")
    _lib.count_launch()
    if flat.arena is not None:
        torch.distributed.all_reduce(finf, op=torch.distributed.ReduceOp.MAX)   # identical verdict on all ranks
    optimizer.inv_scale = 1.0 / scale
    optimizer.found_inf = finf
    if int(finf.item()):                       # apex syncs here too
        _cfg["scale"] = max(scale / 2.0, 1.0)
        _cfg["good_steps"] = 0
    else:
        _cfg["good_steps"] += 1
        if _cfg["good_steps"] % _cfg["growth_interval"] == 0:
            _cfg["scale"] = scale * 2.0


def state_dict():
    return {"loss_scaler0": {"loss_scale": _cfg["scale"], "unskipped": _cfg["good_steps"]}}


def load_state_dict(sd):
    s = sd.get("loss_scaler0", {})
    _cfg["scale"] = float(s.get("loss_scale", _cfg["scale"]))
    _cfg["good_steps"] = int(s.get("unskipped", 0))
