"""amp seam: `amp.initialize`, `amp.scale_loss`, `amp.state_dict/load_state_dict` of the reference
(apex.amp O1; train.py:15,181-183,298-300, utils/pipeline_ops.py:74,121).

Default: bf16 autocast, loss scale fixed at 1.0 — bf16 has fp32's exponent range, so the dynamic
scaler of apex O1 has nothing to do; weights, gradients and optimizer state stay fp32 ("fp32 master") exactly
as under O1.  `dtype=torch.float16` keeps apex's dynamic-scale behaviour (init 2^16, ÷2 and skip the step on
overflow, never below 1, ×2 after every `growth_interval` (2000) clean steps in a row, never above apex's
max_loss_scale 2^24).  The scaler lives on the device
(`sod_loss_scaler`, include/sod_b200.h): the loss gradient is formed already scaled, the overflow checks ride on the
gradient gather, and the fused step kernel reads the verdict and 1/scale and advances the scaler itself — so an fp16
iteration has no host round trip and replays from a CUDA graph like a bf16 one.  Both dtypes use the 16-bit shadow weights.

`_cfg["scale"]` / `_cfg["good_steps"]` are a host mirror of the device scaler: an eager step reads it back (the one host
sync that path makes anyway), a graph replay does not (`read_scaler()` does, on demand); a host write to `_cfg["scale"]`,
`_cfg["good_steps"]` or `_cfg["growth_interval"]` is pushed to the device before the next iteration.
"""
from __future__ import annotations

import contextlib
import functools

import torch

from . import _lib
from .optim import FusedOptimizer, is_plain_conv

import os

# SOD_STEAL_WGRADS=0: bind every shadow leaf's .grad to the flat buffer (autograd then launches one add per tensor)
STEAL_WEIGHT_GRADS = os.environ.get("SOD_STEAL_WGRADS", "1") == "1"

_cfg = {"enabled": False, "dtype": torch.bfloat16, "scale": 1.0, "dynamic": False, "good_steps": 0,
        "growth_interval": 2000, "owner": None, "dev": None}
# owner: the FusedOptimizer whose flat buffers hold the device scaler (fp16 only); dev: the mirror values last known to be
# on the device, {"scale", "good_steps", "growth_interval"} — a host value that differs from it is pushed


def _install_shadow_weights(model, flat) -> int:
    """Point every Conv2d whose parameters live in `flat` at the 16-bit (bf16 or fp16) shadow copy: under autocast the
    convolution then takes its weight without a per-iteration cast kernel, and autograd accumulates the 16-bit weight
    gradient straight into the flat 16-bit gradient buffer the fused step consumes.  fp32 masters stay the module Parameters
    (state_dict / checkpoints / optimizer groups are unaffected).  Convolution subclasses with their own forward (the
    weight-standardised ones) are left alone, `optim.is_plain_conv`."""
    import torch.nn as nn
    managed = {id(p) for p, _ in flat.slots}
    count = 0
    for m in model.modules():
        if not is_plain_conv(m) or id(m.weight) not in managed or hasattr(m, "_sod_w16"):
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
    _cfg["good_steps"] = 0
    _cfg["owner"] = _cfg["dev"] = None
    if _cfg["enabled"]:
        inner = model.forward

        @functools.wraps(inner)
        def autocast_forward(*a, **k):
            with torch.autocast("cuda", dtype=_cfg["dtype"]):
                return inner(*a, **k)

        model.forward = autocast_forward
        fused_cuda = isinstance(optimizer, FusedOptimizer) and optimizer.flat.param.is_cuda
        if _cfg["dynamic"] and fused_cuda:
            optimizer.flat.enable_scaler(_cfg["scale"], _cfg["growth_interval"])
            _cfg["owner"] = optimizer
            _cfg["dev"] = {k: _cfg[k] for k in ("scale", "good_steps", "growth_interval")}
            optimizer._scaler_readback = _read_back
        if shadow_weights and dtype in (torch.bfloat16, torch.float16) and fused_cuda:
            optimizer.flat.enable_shadow(dtype)
            _install_shadow_weights(model, optimizer.flat)
    return (model, optimizer) if optimizer is not None else model


def _scaler() -> torch.Tensor | None:
    """the device scaler (int32[SOD_LOSS_SCALER_WORDS], `sod_loss_scaler`), or None when the loss scale is static"""
    owner = _cfg.get("owner")
    return owner.flat.scaler if (_cfg["dynamic"] and owner is not None) else None


def scale_tensor() -> torch.Tensor | None:
    """0-d fp32 view of the device loss scale (what `scale_loss` multiplies the loss by and the fused loss kernel scales its
    gradient by), or None when the loss scale is static"""
    s = _scaler()
    return s.view(torch.float32)[1] if s is not None else None


def push() -> None:
    """bring host writes of `_cfg["scale"]` / `["good_steps"]` / `["growth_interval"]` to the device scaler (stream-ordered
    fills, no sync; a no-op when nothing changed and while a CUDA graph is being captured)"""
    s = _scaler()
    if s is None or torch.cuda.is_current_stream_capturing():
        return
    dev = _cfg["dev"]
    if _cfg["scale"] != dev["scale"]:
        s.view(torch.float32)[1].fill_(float(_cfg["scale"]))
    if _cfg["good_steps"] != dev["good_steps"]:
        s[2].fill_(int(_cfg["good_steps"]))
    if _cfg["growth_interval"] != dev["growth_interval"]:
        s[3].fill_(int(_cfg["growth_interval"]))
    _cfg["dev"] = {k: _cfg[k] for k in ("scale", "good_steps", "growth_interval")}


def _read_back() -> None:
    s = _scaler()
    if s is None:
        return
    w = s[:4].cpu()                                        # one 16-byte D2H copy (host sync)
    _cfg["scale"] = float(w.view(torch.float32)[1])
    _cfg["good_steps"] = int(w[2])
    _cfg["growth_interval"] = int(w[3])
    _cfg["dev"] = {k: _cfg[k] for k in ("scale", "good_steps", "growth_interval")}


def read_scaler() -> dict:
    """the device scaler as the host sees it after a sync — {"scale", "unskipped", "found_inf"} — and the host mirror
    brought up to date (after graph replays, which do not update it)"""
    s = _scaler()
    if s is None:
        return {"scale": _cfg["scale"], "unskipped": _cfg["good_steps"], "found_inf": 0}
    push()
    _read_back()
    return {"scale": _cfg["scale"], "unskipped": _cfg["good_steps"], "found_inf": int(s[0].item())}


@contextlib.contextmanager
def scale_loss(loss, optimizer):
    """`with amp.scale_loss(loss, optimizer) as scaled: scaled.backward()` (reference train.py:299).  fp16: yields
    loss × the device scale; the overflow check, the skip and the scale update happen inside `optimizer.step()`."""
    if not _cfg["dynamic"]:
        yield loss
        return
    if not isinstance(optimizer, FusedOptimizer):
        raise _lib.SodError("fp16 dynamic loss scaling is wired into the fused optimizers (FusedSGD, FusedAdam) only")
    if optimizer is not _cfg["owner"] or optimizer.flat.scaler is None:
        raise _lib.SodError("fp16 dynamic loss scaling needs the optimizer that was passed to amp.initialize (on CUDA)")
    push()
    yield loss * scale_tensor()


def state_dict():
    if _scaler() is not None:
        read_scaler()
    return {"loss_scaler0": {"loss_scale": _cfg["scale"], "unskipped": _cfg["good_steps"]}}


def load_state_dict(sd):
    s = sd.get("loss_scaler0", {})
    _cfg["scale"] = float(s.get("loss_scale", _cfg["scale"]))
    _cfg["good_steps"] = int(s.get("unskipped", 0))
    push()
