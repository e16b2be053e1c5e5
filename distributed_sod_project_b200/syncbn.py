"""SyncBatchNorm seam: `convert_syncbn_model` + `SyncBatchNorm`, backed by csrc/syncbn.cu.

Reference surface kept: `apex.parallel.convert_syncbn_model(model)` (reference train.py:16,180) — walks the
module tree and swaps every BatchNorm for a synchronized one, returning the model.

Decisions that differ from apex, on purpose (SURVEY §8a):
* Q2 — the swapped module SHARES the original `weight` / `bias` Parameter objects, so an optimizer built
  before the conversion (reference train.py:157 vs :180) keeps training γ/β.
* the module also exposes `fused_forward(x, pre_add=, residual=, relu=)`, used by the model plugins'
  `bn_act` helper to fold the neighbouring add / ReLU into the same kernel.
* one kernel launch per direction also when world_size == 1 (plain BN): the statistics "exchange" is then
  the intra-GPU broadcast of the same packet mechanism.
Inputs are processed as channels-last [N·H·W, C] matrices; other layouts are converted on entry.
"""
from __future__ import annotations

import os

import torch
import torch.nn as nn

from . import _lib, comm

_state: dict = {}
DEBUG_FLAGS = 0             # tools/bn_phases.py sets SOD_DEBUG_TIMING (4)
# how the kernels are launched (csrc/syncbn.cu launch_bn): "plain", "coop" (cooperative launch: the driver guarantees
# that the whole grid is co-resident, which the packet exchange relies on) or "pdl" (programmatic dependent launch)
LAUNCH_MODE = os.environ.get("SOD_BN_LAUNCH", "plain")


def _launch_flags() -> int:
    return {"plain": 0, "coop": _lib.SOD_BN_LAUNCH_COOP, "pdl": _lib.SOD_BN_LAUNCH_PDL}[LAUNCH_MODE]

FORCE_LOCAL = False         # bench.py roofline replay: run single-rank (no exchange) even inside a process group
# BN+ReLU layers without a residual re-derive the ReLU mask from x in the backward instead of reading y (one input stream
# less); dz is identical to the y-mask variant (tools/ab_bn_bwd_variants.py compares them).  SOD_BN_MASK_FROM_X=0 turns it off.
MASK_FROM_X = os.environ.get("SOD_BN_MASK_FROM_X", "1") == "1"
# L2 eviction-priority hints on the backward's bulk copies (same A/B; SOD_BN_L2_HINTS=0 turns them off)
L2_HINTS = os.environ.get("SOD_BN_L2_HINTS", "1") == "1"
TRACE: list | None = None   # bench.py: when a list, every forward call appends (n, c, h, w, has_pre, has_res, relu)


def _dev_state(device: torch.device) -> dict:
    st = _state.get(device.index)
    if st is None:
        nbytes = int(_lib.lib().sod_syncbn_workspace_bytes(1, 2048)) + 16384   # + room for debug stamps (kMaxGrid x 8 x 8 bytes)
        st = {"ws": torch.zeros(nbytes, dtype=torch.uint8, device=device), "seq": 0,
              "epoch": torch.zeros(1, dtype=torch.int32, device=device), "graph": False, "idx": 0}
        _state[device.index] = st
    return st


def begin_iteration(device: torch.device, graph: bool) -> None:
    """graph=True: tags of the coming BN calls are (device epoch, call index) so that the captured iteration can
    be replayed; the captured code must end with `end_iteration` (epoch += 1 on the device)."""
    st = _dev_state(device)
    st["graph"], st["idx"] = graph, 0


def end_iteration(device: torch.device) -> None:
    st = _dev_state(device)
    if st["graph"]:
        st["epoch"].add_(1)          # captured: one tiny kernel per replay
        st["graph"] = False


def _next_call(device: torch.device):
    """(workspace, seq, epoch_ptr, comm_ref, stats_off).  Eager: one global sequence over ALL BN launches of this
    process (tags must be unique across forward and backward calls sharing slots).  Graph capture: call index
    within the iteration + the device-side epoch."""
    st = _dev_state(device)
    if st["graph"]:
        st["idx"] += 1
        if st["idx"] > 1023:
            raise _lib.SodError("more than 1023 SyncBN launches in one captured iteration")
        seq, epoch = st["idx"], st["epoch"].data_ptr()
    else:
        st["seq"] = (st["seq"] + 1) & 0x7FFFFFFF or 1
        seq, epoch = st["seq"], None
    arena = None if FORCE_LOCAL else comm.small_arena()
    if arena is None:
        return st["ws"], seq, epoch, None, 0
    return st["ws"], seq, epoch, arena.ref, arena.bn_slots[seq % len(arena.bn_slots)]


def _as_rows(t: torch.Tensor) -> torch.Tensor:
    """dense channels-last view of an NCHW-shaped tensor (copy only if it is not already laid out so)"""
    if t.dim() != 4:
        raise _lib.SodError(f"SyncBatchNorm expects 4-D input, got {t.dim()}-D")
    return t if t.is_contiguous(memory_format=torch.channels_last) else t.contiguous(memory_format=torch.channels_last)


class _SyncBNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, pre_add, residual, weight, bias, running_mean, running_var, nbt, momentum, eps, relu, training,
                cb1=None, cb2=None):
        x = _as_rows(x)
        pre = _as_rows(pre_add).to(x.dtype) if pre_add is not None else None
        res = _as_rows(residual).to(x.dtype) if residual is not None else None
        n, c, h, w = x.shape
        rows = n * h * w
        if TRACE is not None:
            TRACE.append((n, c, h, w, pre is not None, res is not None, bool(relu)))
        y = torch.empty_like(x)  # preserves channels-last strides
        dev = x.device
        if training:
            mean = torch.empty(c, dtype=torch.float32, device=dev)        # the kernel saves the batch statistics
            invstd = torch.empty(c, dtype=torch.float32, device=dev)
        elif any(ctx.needs_input_grad):
            # eval with grad: the backward differentiates through the running statistics as they are now
            mean = running_mean.detach().float().clone()
            invstd = 1.0 / torch.sqrt(running_var.detach().float() + eps)
        else:
            mean = invstd = None
        cbs = [t for t in (cb1, cb2) if t is not None]
        cb_dtype = _lib.dtype_code(cbs[0].dtype) if cbs else 0
        if len(cbs) == 2 and cbs[0].dtype != cbs[1].dtype:
            raise _lib.SodError("folded conv biases must share a dtype")
        ws, seq, epoch, cref, soff = _next_call(dev)
        rc = _lib.lib().sod_syncbn_fwd(
            x.data_ptr(), pre.data_ptr() if pre is not None else None, res.data_ptr() if res is not None else None,
            y.data_ptr(), _lib.dtype_code(x.dtype), weight.data_ptr(), bias.data_ptr(),
            running_mean.data_ptr() if running_mean is not None else None,
            running_var.data_ptr() if running_var is not None else None,
            mean.data_ptr() if training else None, invstd.data_ptr() if training else None, rows, c, float(momentum),
            float(eps), int(relu), int(training),
            cref, soff, seq, epoch, nbt.data_ptr() if nbt is not None else None,
            cb1.data_ptr() if cb1 is not None else None, cb2.data_ptr() if cb2 is not None else None, cb_dtype,
            ws.data_ptr(), ws.numel(), DEBUG_FLAGS | _launch_flags(), _lib.stream_ptr())
        _lib.check(rc, "sod_syncbn_fwd")
        _lib.count_launch()
        ctx.relu, ctx.has_pre, ctx.has_res = bool(relu), pre is not None, res is not None
        ctx.training = bool(training)
        ctx.weight_ref, ctx.bias_ref = weight, bias
        ctx.cb = (cb1, cb2)
        ctx.save_for_backward(x, pre, y if relu else None, weight, mean, invstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, pre, y, weight, mean, invstd = ctx.saved_tensors
        # when γ/β already carry a bound fp32 .grad (FusedSGD's flat buffer) the kernel adds into it directly and
        # autograd gets None: saves two AccumulateGrad launches per layer
        wg, bg = getattr(ctx.weight_ref, "grad", None), getattr(ctx.bias_ref, "grad", None)
        direct = (wg is not None and bg is not None and wg.dtype == torch.float32 and bg.dtype == torch.float32
                  and wg.is_contiguous() and bg.is_contiguous() and ctx.weight_ref.requires_grad and ctx.bias_ref.requires_grad)
        # folded conv biases: the kernel adds Σ_rows dz into a bound .grad (FusedSGD's bf16/fp32 flat buffers) when there
        # is one, else into a zeroed temporary that is handed to autograd (always for a non-leaf bias, such as the sum of
        # two biases that `blocks.conv3_bn_act` folds into one slot: autograd routes it on)
        cb1, cb2 = ctx.cb
        dcb, ret_cb = [None, None], [None, None]
        for i, cb in enumerate((cb1, cb2)):
            if cb is None or not cb.requires_grad:
                continue
            gbound = cb.grad if cb.is_leaf else None
            if gbound is not None and gbound.dtype == cb.dtype and gbound.is_contiguous():
                dcb[i] = gbound
            else:
                dcb[i] = torch.zeros_like(cb)
                ret_cb[i] = dcb[i]
        if ctx.training:
            dz, dres, dgamma, dbeta = raw_backward(_as_rows(dy).to(x.dtype), x, pre, y, weight, mean, invstd, ctx.relu,
                                                   ctx.has_res, into=(wg, bg) if direct else None, conv_bias=(cb1, cb2),
                                                   dconv_bias=dcb, bias=ctx.bias_ref)
        else:
            dz, dres, dgamma, dbeta = _eval_backward(_as_rows(dy).to(x.dtype), x, pre, y, weight, mean, invstd, ctx.relu,
                                                     ctx.has_res, (cb1, cb2), dcb)
            if direct:
                wg.add_(dgamma)
                bg.add_(dbeta)
        gw, gb = (None, None) if direct else (dgamma.to(weight.dtype), dbeta.to(weight.dtype))
        return (dz, dz if ctx.has_pre else None, dres, gw, gb, None, None, None, None, None, None, None, ret_cb[0], ret_cb[1])


def _eval_backward(dy, x, pre, y, weight, mean, invstd, relu: bool, want_dres: bool, conv_bias, dconv_bias):
    """backward of the eval-mode forward y = act(γ·(x + pre + cb − running_mean)·invstd + β [+ residual]) in fp32 torch ops:
    the statistics are constants here, so dz = dout·γ·invstd with no batch-mean terms.  Off the training path (a frozen
    BN while fine-tuning, input-gradient saliency).  Adds Σ dz into `dconv_bias`; returns (dz, dres|None, dγ, dβ)."""
    c = x.shape[1]
    dout = dy.float()
    if relu:
        dout = dout * (y > 0)
    z = x.float() if pre is None else x.float() + pre.float()
    for cb in conv_bias:
        if cb is not None:
            z = z + cb.detach().float().view(1, c, 1, 1)
    xhat = (z - mean.view(1, c, 1, 1)) * invstd.view(1, c, 1, 1)
    dz32 = dout * (weight.detach().float() * invstd).view(1, c, 1, 1)
    if any(d is not None for d in dconv_bias):
        s = dz32.sum(dim=(0, 2, 3))
        for d in dconv_bias:
            if d is not None:
                d.copy_(d.float() + s)
    dz = dz32.to(x.dtype).contiguous(memory_format=torch.channels_last)
    dres = dout.to(x.dtype).contiguous(memory_format=torch.channels_last) if want_dres else None
    return dz, dres, (dout * xhat).sum(dim=(0, 2, 3)), dout.sum(dim=(0, 2, 3))


def raw_backward(dy, x, pre, y, weight, mean, invstd, relu: bool, want_dres: bool, into=None, conv_bias=(None, None),
                 dconv_bias=(None, None), bias=None):
    """one `sod_syncbn_bwd` launch on channels-last tensors; returns (dz, dres|None, dgamma, dbeta).
    `into=(weight_grad, bias_grad)`: accumulate the parameter gradients into those fp32 tensors instead.
    `bias` (β) is only read by the MASK_FROM_X variant."""
    n, c, h, w = x.shape
    dz = torch.empty_like(x)
    dres = torch.empty_like(x) if want_dres else None
    if into is not None:
        dgamma, dbeta = into
        flags = DEBUG_FLAGS | _launch_flags() | _lib.SOD_BN_ACCUMULATE_PARAM_GRADS
        _lib.grad_writes += 1          # bound .grad buffers change behind autograd's back (FusedSGD.zero_grad looks at this)
    else:
        dgamma = torch.empty(c, dtype=torch.float32, device=x.device)
        dbeta = torch.empty(c, dtype=torch.float32, device=x.device)
        flags = DEBUG_FLAGS | _launch_flags()
    if any(d is not None for d in dconv_bias):
        _lib.grad_writes += 1          # so does a folded conv bias's bound .grad (or a temporary: a harmless extra memset)
    if MASK_FROM_X and relu and not want_dres and bias is not None:
        flags |= _lib.SOD_BN_BWD_MASK_FROM_X
    if L2_HINTS:
        flags |= _lib.SOD_BN_L2_HINTS
    ws, seq, epoch, cref, soff = _next_call(x.device)
    rc = _lib.lib().sod_syncbn_bwd(
        dy.data_ptr(), x.data_ptr(), pre.data_ptr() if pre is not None else None,
        y.data_ptr() if (relu and y is not None) else None, dz.data_ptr(), dres.data_ptr() if dres is not None else None,
        _lib.dtype_code(x.dtype), weight.data_ptr(), bias.data_ptr() if bias is not None else None,
        mean.data_ptr(), invstd.data_ptr(), dgamma.data_ptr(),
        dbeta.data_ptr(), n * h * w, c, int(relu), cref, soff, seq, epoch,
        *(t.data_ptr() if t is not None else None for t in (conv_bias[0], conv_bias[1], dconv_bias[0], dconv_bias[1])),
        next((_lib.dtype_code(t.dtype) for t in conv_bias if t is not None), 0),
        ws.data_ptr(), ws.numel(), flags, _lib.stream_ptr())
    _lib.check(rc, "sod_syncbn_bwd")
    _lib.count_launch()
    return dz, dres, dgamma, dbeta


class SyncBatchNorm(nn.BatchNorm2d):
    """Drop-in for the module `convert_syncbn_model` installs (reference train.py:180)."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.fused_forward(x)

    def fused_forward(self, x, pre_add=None, residual=None, relu=False, conv_bias=(None, None)):
        """`conv_bias`: biases of the (bias-less) convolutions that produced `x` / `pre_add`, folded into the kernel"""
        if not x.is_cuda:
            raise _lib.SodError("SyncBatchNorm: expected a CUDA tensor (the sm_90a kernel has no CPU fallback; "
                                "keep nn.BatchNorm2d for CPU runs)")
        if x.shape[1] != self.num_features:
            raise ValueError(f"expected {self.num_features} channels, got {x.shape[1]}")
        training = self.training or self.running_mean is None
        momentum, nbt = 0.0, None
        if training and self.track_running_stats:
            nbt = self.num_batches_tracked          # incremented inside the kernel (saves 84 tiny launches / iteration)
            if self.momentum is None:
                raise _lib.SodError("momentum=None (cumulative moving average) is not on the reference's hot path")
            momentum = self.momentum
        rm = self.running_mean if self.track_running_stats else None
        rv = self.running_var if self.track_running_stats else None
        weight = self.weight if self.affine else torch.ones(self.num_features, device=x.device)
        bias = self.bias if self.affine else torch.zeros(self.num_features, device=x.device)
        return _SyncBNFn.apply(x, pre_add, residual, weight, bias, rm, rv, nbt, momentum, self.eps, relu, training,
                               conv_bias[0], conv_bias[1])


def convert_syncbn_model(module: nn.Module, process_group=None, channel_last: bool = True) -> nn.Module:
    """Same call shape as apex's (reference train.py:180): returns the model with every `_BatchNorm` replaced
    by `SyncBatchNorm`, parameters and buffers shared with the originals."""
    if isinstance(module, nn.modules.batchnorm._BatchNorm) and not isinstance(module, SyncBatchNorm):
        if not isinstance(module, nn.BatchNorm2d):
            raise _lib.SodError(f"only BatchNorm2d is on the hot path, found {type(module).__name__}")
        new = SyncBatchNorm(module.num_features, module.eps, module.momentum, module.affine, module.track_running_stats)
        if module.affine:
            new.weight, new.bias = module.weight, module.bias          # same Parameter objects (Q2)
        new.running_mean, new.running_var = module.running_mean, module.running_var
        new.num_batches_tracked = module.num_batches_tracked
        new.train(module.training)
        return new
    for name, child in list(module.named_children()):
        converted = convert_syncbn_model(child, process_group, channel_last)
        if converted is not child:
            if isinstance(module, nn.Sequential):
                module[int(name)] = converted
            else:
                setattr(module, name, converted)
    return module
