"""Optimizer seam: `make_optimizer`, `CustomScheduler`, `FusedSGD` and `FusedAdam` (csrc/sgd.cu underneath).

Reference surface kept (paths in the reference repo):
* `make_optimizer(model, optimizer_type, optimizer_info)`          — utils/pipeline_ops.py:235-316
  (`sgd_trick`, `sgd_r3`, `sgd_all`, `f3_trick` → FusedSGD, `nesterov` honoured for sgd_trick / f3_trick;
  `adam` → FusedAdam)
* `CustomScheduler(optimizer, total_num, scheduler_type, scheduler_info).step(optimizer, curr_epoch)`
                                                                     — utils/pipeline_ops.py:185-232
* the `torch.optim.Optimizer` protocol the loop relies on: `.param_groups[i]["lr"]` mutated from outside,
  `.zero_grad()`, `.step()`, `.state_dict()/.load_state_dict()` with per-parameter `momentum_buffer` (SGD) or
  `step` / `exp_avg` / `exp_avg_sq` (Adam) (utils/pipeline_ops.py:73,118), `str(optimizer)` (train.py:176).

The fused optimizers (`FusedOptimizer` and its two subclasses) keep parameters, gradients and optimizer state in flat
fp32 buffers laid out group-major ([group 0 | group 1 | … | parameters in no group]); every `p.data` / `p.grad` is a
view into them.  `step()` is one kernel: world 1 → `sod_sgd_momentum` / `sod_adam`; world > 1 (after
`DistributedDataParallel` has moved the flat parameter and gradient buffers into symmetric memory) →
`sod_allreduce_sgd` / `sod_allreduce_adam`, which also do the gradient averaging, so nothing else runs between
backward and the next forward.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
from torch.optim import Optimizer

from . import _lib

flat_registry: dict = {}   # id(param) → FlatParams (lets DistributedDataParallel find the optimizer's layout)

_ALIGN = 64  # elements; keeps every tensor view 256-byte aligned and every segment float4-aligned


class FlatParams:
    """Group-major flat storage for a set of parameters."""

    def __init__(self, groups: list[list[nn.Parameter]], leftovers: list[nn.Parameter], bf16_grad_ids: set | None = None):
        """`bf16_grad_ids`: ids of the parameters whose gradient will exist in bf16 only once the amp shadow is installed
        (convolution weights / biases).  Inside every bucket those come first, so that each bucket is at most two
        contiguous ranges — [bf16-gradient part | fp32-gradient part] — and the kernels can take the gradient of the
        first from the bf16 buffer alone (SOD_SEG_GRAD16)."""
        bf16_grad_ids = bf16_grad_ids or set()
        groups = [sorted(g, key=lambda p: id(p) not in bf16_grad_ids) for g in groups]       # stable: order kept inside each part
        leftovers = sorted(leftovers, key=lambda p: id(p) not in bf16_grad_ids)
        self.groups, self.leftovers = groups, leftovers
        all_params = [p for g in groups for p in g] + leftovers
        if not all_params:
            raise ValueError("no parameters")
        dev = all_params[0].device
        if any(p.device != dev or p.dtype != torch.float32 for p in all_params):
            raise _lib.SodError("the fused optimizers need fp32 parameters on one device")
        self.device = dev
        self.slots: list[tuple[nn.Parameter, int]] = []      # (param, element offset)
        self.ranges: list[tuple[int, int]] = []               # per group [begin, end), then leftovers
        self.splits: list[int] = []                           # per bucket: end of its bf16-gradient part
        off = 0
        for bucket in [*groups, leftovers]:
            begin = mid = off
            for p in bucket:
                self.slots.append((p, off))
                off += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
                if id(p) in bf16_grad_ids:
                    mid = off
            self.ranges.append((begin, off))
            self.splits.append(mid)
        self.numel = off
        self.param = torch.zeros(off, dtype=torch.float32, device=dev)
        self.grad = torch.zeros(off, dtype=torch.float32, device=dev)
        self.mom = torch.zeros(off, dtype=torch.float32, device=dev)
        self.arena = None          # set by DistributedDataParallel when world > 1
        self.param_off = self.grad_off = self.grad16_off = 0
        self.shadow16: torch.Tensor | None = None   # bf16/fp16 copy of `param`, refreshed by the fused step (amp O1 shadow)
        self.grad16: torch.Tensor | None = None     # 16-bit gradients (the shadow's dtype) autograd makes for the shadowed tensors
        # amp fp16: the device-resident loss scaler (`sod_loss_scaler`, int32 words; the scale is word 1 as fp32 bits), in
        # the symmetric arena at scaler_off when world > 1
        self.scaler: torch.Tensor | None = None
        self.scaler_off = 0
        # bf16 shadow leaves the convolutions consume (amp._install_shadow_weights): (leaf, element offset, steal)
        # steal=True: `.grad` is left None so that autograd hands over cuDNN's gradient tensor as it is (no accumulate
        # kernel per parameter); the fused step collects all of them into `grad16` with one sod_grad_gather16 launch
        self.shadow_leaves: list[tuple[torch.Tensor, int, bool]] = []
        # set by a hook on the fp32 masters of shadowed parameters (amp._install_shadow_weights) when a gradient reaches one
        # of them — the model ran outside autocast — and cleared by the step that has consumed it
        self.master_grads_seen = False
        self._bind(copy_from_params=True)

    # -- mixed precision: 16-bit shadow of the fp32 master ---------------------------------------------------
    def enable_shadow(self, dtype: torch.dtype = torch.bfloat16) -> None:
        """bf16 (amp bf16) or fp16 (amp fp16, with the device loss scaler); `grad16` takes the same dtype"""
        if dtype not in (torch.bfloat16, torch.float16):
            raise _lib.SodError(f"the shadow copy is bf16 or fp16, not {dtype}")
        if self.shadow16 is not None and self.shadow16.dtype != dtype:
            raise _lib.SodError(f"the shadow copy is already {self.shadow16.dtype}")
        if self.shadow16 is None:
            self.shadow16 = torch.zeros(self.numel, dtype=dtype, device=self.device)
            self.grad16 = torch.zeros(self.numel, dtype=dtype, device=self.device)
        self.refresh_shadow()

    def enable_scaler(self, scale: float, growth_interval: int) -> None:
        """the device-resident dynamic loss scale of amp fp16 (include/sod_b200.h `sod_loss_scaler`)"""
        if self.scaler is None:
            self.scaler = torch.zeros(_lib.SOD_LOSS_SCALER_WORDS, dtype=torch.int32, device=self.device)
        self.scaler.zero_()
        self.scaler.view(torch.float32)[1].fill_(float(scale))
        self.scaler[3].fill_(int(growth_interval))

    @property
    def flags16(self) -> int:
        """the step kernels' flag for the 16-bit buffers' format"""
        return _lib.SOD_GRAD16_F16 if self.grad16 is not None and self.grad16.dtype == torch.float16 else 0

    def refresh_shadow(self) -> None:
        if self.shadow16 is not None:
            self.shadow16.copy_(self.param)

    def offset_of(self, p: nn.Parameter) -> int:
        for q, off in self.slots:
            if q is p:
                return off
        raise KeyError("parameter not managed")

    def view16(self, buf: torch.Tensor, p: nn.Parameter) -> torch.Tensor:
        return self._view(buf, self.offset_of(p), p.data)

    @staticmethod
    def _view(buf: torch.Tensor, off: int, p: torch.Tensor) -> torch.Tensor:
        """view of buf[off:off+numel] with p's shape AND memory format (channels-last conv weights keep their
        KRSC physical order, so cuDNN's NHWC kernels need no per-iteration weight transpose)"""
        flat = buf[off:off + p.numel()]
        if p.dim() == 4 and not p.is_contiguous() and p.is_contiguous(memory_format=torch.channels_last):
            n, c, h, w = p.shape
            return flat.view(n, h, w, c).permute(0, 3, 1, 2)
        return flat.view(p.shape)

    def _bind(self, copy_from_params: bool):
        with torch.no_grad():
            for p, off in self.slots:
                view = self._view(self.param, off, p.data)
                if copy_from_params:
                    view.copy_(p.data)
                g = self._view(self.grad, off, p.data)
                p.data = view
                p.grad = g

    def relocate(self, arena, param_off: int, grad_off: int):
        """Move the flat parameter / gradient buffers into a symmetric arena (momentum stays local)."""
        new_p = arena.view(param_off, self.numel, torch.float32)
        new_g = arena.view(grad_off, self.numel, torch.float32)
        new_p.copy_(self.param)
        new_g.copy_(self.grad)
        self.param, self.grad = new_p, new_g
        self.arena, self.param_off, self.grad_off = arena, param_off, grad_off
        self._bind(copy_from_params=False)
        if self.grad16 is not None:
            # the bf16 gradients cross NVLink as they are (csrc/sgd.cu reduce_vec16): they have to be peer-readable too
            self.grad16_off = arena.alloc(2 * self.numel)
            new16 = arena.view(self.grad16_off, self.numel, self.grad16.dtype)
            new16.copy_(self.grad16)
            self.grad16 = new16
            for leaf, off, steal in self.shadow_leaves:
                if not steal and leaf.requires_grad:
                    leaf.grad = self._view(self.grad16, off, leaf)
        if self.scaler is not None:
            # every rank's step kernel reads every rank's overflow flag: the scaler has to be peer-readable
            self.scaler_off = arena.alloc(4 * _lib.SOD_LOSS_SCALER_WORDS)
            new_s = arena.view(self.scaler_off, _lib.SOD_LOSS_SCALER_WORDS, torch.int32)
            new_s.copy_(self.scaler)
            self.scaler = new_s
        self.refresh_shadow()

    def momentum_view(self, p: nn.Parameter) -> torch.Tensor:
        for q, off in self.slots:
            if q is p:
                return self._view(self.mom, off, p.data)
        raise KeyError("parameter not managed")


def _same_physical_order(a: torch.Tensor, b: torch.Tensor) -> bool:
    """both dense, and their elements laid out in memory in the same order — strides of size-1 dimensions carry no
    information (a [K,C,1,1] weight is the same bytes channels-last or contiguous, but reports different strides)"""
    if a.shape != b.shape:
        return False
    sa = [st for st, n in zip(a.stride(), a.shape) if n > 1]
    sb = [st for st, n in zip(b.stride(), b.shape) if n > 1]
    if sa != sb:
        return False
    need = 1
    for st, n in sorted((st, n) for st, n in zip(a.stride(), a.shape) if n > 1):
        if st != need:
            return False
        need *= n
    return True


def is_plain_conv(m: nn.Module) -> bool:
    """an nn.Conv2d whose class keeps nn.Conv2d's forward and _conv_forward: the convolution runs on the weight Parameter as
    it is, so amp may hand it a 16-bit shadow of that weight and the gradient arrives in 16 bit.  A subclass that computes
    its operand from the weight (the weight-standardised convolutions: network.blocks.WSConv2d, the reference's
    backbone/wsgn/customized_func.Conv2d) is left alone: a shadow of the raw master would be the wrong operand, and its
    gradient reaches the fp32 master through the subclass's own computation."""
    return (isinstance(m, nn.Conv2d) and type(m).forward is nn.Conv2d.forward
            and type(m)._conv_forward is nn.Conv2d._conv_forward)


class FusedOptimizer(Optimizer):
    """What the fused optimizers share: the flat group-major layout (`FlatParams`), the segment table the kernels walk,
    the device learning-rate table, the bf16 gradient gather, `zero_grad`, the shard bounds of world > 1 and the
    collective gather of sharded state.  A subclass names its state buffers and its kernels (`_segment`, `_launch_local`,
    `_launch_allreduce`) and keeps its own torch.optim state_dict layout."""

    def __init__(self, params, defaults: dict, model: nn.Module | None):
        super().__init__(params, defaults)
        if 2 * (len(self.param_groups) + 1) > _lib.SOD_MAX_SEGMENTS:
            raise _lib.SodError(f"at most {_lib.SOD_MAX_SEGMENTS // 2 - 1} parameter groups")
        grouped = {id(p) for g in self.param_groups for p in g["params"]}
        leftovers = [p for p in model.parameters() if id(p) not in grouped] if model is not None else []
        # parameters whose gradient the amp shadow will deliver in 16 bit: those of plain convolutions (amp._install_shadow_weights)
        conv_ids = {id(p) for m in model.modules() if is_plain_conv(m)
                    for p in (m.weight, m.bias) if p is not None} if model is not None else set()
        self.flat = FlatParams([list(g["params"]) for g in self.param_groups], leftovers, bf16_grad_ids=conv_ids)
        for p, _ in self.flat.slots:
            flat_registry[id(p)] = self.flat
        self.inv_scale = 1.0                   # static loss scale: 1/S for the coming step
        self._found_inf: torch.Tensor | None = None  # static loss scale: device uint32 flag, or None
        self._scaler_readback = None           # amp fp16: refreshes amp's host mirror after an eager step
        self._grads_clean = True
        self._clean_version = self._grad_versions()
        self._stepped = False
        self.steps = 0
        # learning rates as the kernels read them: a device table, rewritten (tiny fill kernels, by value) only when a
        # param_group's lr has changed — so a captured iteration follows the scheduler without being re-captured
        self._lr_dev = torch.zeros(_lib.SOD_MAX_SEGMENTS, dtype=torch.float32, device=self.flat.device) \
            if self.flat.device.type == "cuda" else None
        self._lr_sent: list[float | None] = [None] * _lib.SOD_MAX_SEGMENTS

    # -- what a subclass provides ---------------------------------------------------------------------------
    def _state_buffers(self) -> list[torch.Tensor]:
        """the flat optimizer-state buffers (full length; at world > 1 each rank keeps only its shard current)"""
        raise NotImplementedError

    def _segment(self, b: int, e: int, g: dict | None, flags: int):
        """one entry of the kernels' segment table; g is None for the frozen parameters outside every group"""
        raise NotImplementedError

    def _launch_local(self, segs, n, lr_dev, g16, s16, finf, scaler) -> None:
        """scaler: address of the device loss scaler (then finf / inv_scale are not used), or None"""
        raise NotImplementedError

    def _launch_allreduce(self, segs, n, lr_dev, g16, s16, finf, scaler) -> None:
        raise NotImplementedError

    @property
    def found_inf(self) -> torch.Tensor | None:
        """device uint32 overflow flag of the last step: with amp fp16 a view of the loss scaler's found_inf word"""
        if self.flat.scaler is not None:
            return self.flat.scaler[0:1]
        return self._found_inf

    @found_inf.setter
    def found_inf(self, t: torch.Tensor | None) -> None:
        self._found_inf = t

    # -------------------------------------------------------------------------------------------------------
    def _grad_versions(self):
        f = self.flat
        return (f.grad._version, f.grad16._version if f.grad16 is not None else -1, id(f.grad), _lib.grad_writes)

    def sync_lr(self) -> None:
        """bring the device learning-rate table in line with `param_groups[i]["lr"]` (stream-ordered; a no-op while a
        CUDA graph is being captured — the captured kernels read the table, whoever replays them calls this first)"""
        if self._lr_dev is None or torch.cuda.is_current_stream_capturing():
            return
        for n, (_, _, g, _) in enumerate(self._segment_plan()):
            lr = float(g["lr"]) if g is not None else 0.0
            if self._lr_sent[n] != lr:
                self._lr_dev[n].fill_(lr)
                self._lr_sent[n] = lr

    def _bf16_exclusive(self) -> bool:
        """True when the gradients of the convolution parameters exist in the bf16 buffer only: the shadow is installed and
        no gradient has reached an fp32 master since the last step (one does when the model ran outside autocast — then the
        kernels fall back to reading both buffers).  (Version counters cannot tell: at world > 1 the flat buffers are views
        of ONE symmetric allocation and share its counter.)"""
        f = self.flat
        return f.grad16 is not None and bool(f.shadow_leaves) and not f.master_grads_seen

    def _segment_plan(self):
        """[(begin, end, param_group | None for the frozen leftovers, bf16_only)] — the kernels' segment table; the layout
        (not the flags) is fixed at construction, so the number of segments and their order never change"""
        plan = []
        buckets = list(zip([*self.param_groups, None], self.flat.ranges, self.flat.splits))
        for g, (b, e), mid in buckets:
            if e <= b:
                continue
            if self.flat.grad16 is not None and b < mid < e:
                plan.append((b, mid, g, True)); plan.append((mid, e, g, False))
            else:
                plan.append((b, e, g, self.flat.grad16 is not None and mid == e))
        return plan

    def _group_segments(self) -> list[list[int]]:
        """per param_group, the indices of its segments in `_segment_plan()`"""
        out: list[list[int]] = [[] for _ in self.param_groups]
        ids = [id(g) for g in self.param_groups]
        for n, (_, _, g, _) in enumerate(self._segment_plan()):
            if g is not None:
                out[ids.index(id(g))].append(n)
        return out

    # -- torch.optim.Optimizer protocol -------------------------------------------------------------------
    def zero_grad(self, set_to_none: bool = False):
        """One memset of the flat gradient buffer (a no-op right after a fused step, which already cleared it).
        Gradients stay bound as views — `set_to_none` is accepted and ignored."""
        # the fused step clears the buffer in-kernel; autograd's in-place accumulation bumps the (shared)
        # version counter of the flat buffer, so an unchanged version means nothing has written since
        if not (self._grads_clean and self._grad_versions() == self._clean_version):
            self.flat.grad.zero_()
            if self.flat.grad16 is not None:
                self.flat.grad16.zero_()
        self._grads_clean = False
        # autograd may have replaced a .grad (e.g. after an external `p.grad = None`): rebind
        for p, off in self.flat.slots:
            if p.grad is None or p.grad.data_ptr() != self.flat.grad.data_ptr() + 4 * off:
                p.grad = FlatParams._view(self.flat.grad, off, p.data)
        for leaf, off, steal in self.flat.shadow_leaves:
            if steal:
                leaf.grad = None
            elif leaf.grad is None or leaf.grad.data_ptr() != self.flat.grad16.data_ptr() + 2 * off:
                leaf.grad = FlatParams._view(self.flat.grad16, off, leaf)

    def _gather_stolen(self, finf: int | None = None) -> set:
        """16-bit gradients autograd left in their own tensors (shadow leaves with steal=True, or any leaf whose `.grad`
        was replaced) → flat `grad16`, one launch for all of them.  finf (amp fp16): address of the overflow flag the
        gather ORs the non-finiteness of what it copies into.  Returns the offsets of the leaves it gathered."""
        f = self.flat
        gathered = set()
        if not f.shadow_leaves:
            return gathered
        base = f.grad16.data_ptr()
        items = []
        for leaf, off, _ in f.shadow_leaves:
            g = leaf.grad
            if g is None or g.data_ptr() == base + 2 * off:
                continue
            if g.dtype == f.grad16.dtype and g.is_cuda and g.numel() == leaf.numel() and _same_physical_order(g, leaf):
                items.append((g.data_ptr(), off, g.numel()))
                gathered.add(off)
            else:                                            # unusual layout / dtype: plain torch accumulate
                FlatParams._view(f.grad16, off, leaf).add_(g.to(f.grad16.dtype))
        if items:
            key = tuple(items)
            if getattr(self, "_gather_key", None) != key:    # eager steps see new addresses every time, graph capture once
                self._gather_key = key
                self._gather_arr = (_lib.sod_gather_item * len(items))(*[_lib.sod_gather_item(a, b, c) for a, b, c in items])
            arr = self._gather_arr
            if finf is None:
                rc = _lib.lib().sod_grad_gather16(arr, len(items), base, f.numel, _lib.stream_ptr())
                _lib.check(rc, "sod_grad_gather16")
            else:
                rc = _lib.lib().sod_grad_gather16_checked(arr, len(items), base, f.numel, _lib.dtype_code(f.grad16.dtype),
                                                          finf, _lib.stream_ptr())
                _lib.check(rc, "sod_grad_gather16_checked")
            _lib.count_launch((len(items) + _lib.SOD_GATHER_MAX_ITEMS - 1) // _lib.SOD_GATHER_MAX_ITEMS)
        return gathered

    def _check_rest(self, finf: int, gathered: set) -> None:
        """amp fp16: OR into the flag the non-finiteness of every gradient the checked gather did not read — the fp32
        gradients of the ranges without SOD_SEG_GRAD16 (BN γ/β, leftovers) and the 16-bit gradients accumulated in place
        (folded convolution biases).  After a forward outside autocast (fp32 gradients for the convolution parameters
        too) the whole fp32 buffer is read instead."""
        f = self.flat
        exclusive = self._bf16_exclusive()
        ranges = [] if not exclusive else \
            [(b, e, 0) for b, e, _, part16 in self._segment_plan() if not part16]
        for leaf, off, _ in f.shadow_leaves:
            if off not in gathered:
                ranges.append((off, off + leaf.numel(), _lib.SOD_SEG_GRAD16))
        if not exclusive:
            rc = _lib.lib().sod_grad_nonfinite(f.grad.data_ptr(), f.numel, finf, _lib.stream_ptr())
            _lib.check(rc, "sod_grad_nonfinite")
            _lib.count_launch()
        if not ranges:
            return
        key = tuple(ranges)
        if getattr(self, "_check_key", None) != key:
            self._check_key = key
            self._check_arr = (_lib.sod_check_range * len(ranges))(*[_lib.sod_check_range(b, e, fl) for b, e, fl in ranges])
        g16 = f.grad16.data_ptr() if f.grad16 is not None else None
        rc = _lib.lib().sod_grad_check_ranges(f.grad.data_ptr(), g16, f.numel, self._check_arr, len(ranges), f.flags16, finf,
                                              _lib.stream_ptr())
        _lib.check(rc, "sod_grad_check_ranges")
        _lib.count_launch((len(ranges) + _lib.SOD_CHECK_MAX_RANGES - 1) // _lib.SOD_CHECK_MAX_RANGES)

    def _segments(self):
        plan = self._segment_plan()
        exclusive = self._bf16_exclusive()
        entries = []
        for b, e, g, bf16_part in plan:
            flags = _lib.SOD_SEG_GRAD16 if (bf16_part and exclusive) else 0
            entries.append(self._segment(b, e, g, flags | _lib.SOD_SEG_FROZEN if g is None else flags))
        return (type(entries[0]) * len(entries))(*entries), len(plan)

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise _lib.SodError("closures are not supported by the fused step")
        f = self.flat
        if not f.param.is_cuda:
            raise _lib.SodError(f"{type(self).__name__}.step needs CUDA parameters (no CPU fallback)")
        segs, n = self._segments()
        self.sync_lr()
        lr_dev = self._lr_dev.data_ptr()
        scaler = f.scaler.data_ptr() if f.scaler is not None else None
        if scaler is not None:
            # amp fp16: clear the flag (stream order puts this after the previous step, which every peer has left), then
            # the checks: the gather checks what it copies, one small launch the rest; the step reads the verdict
            f.scaler[0:1].zero_()
            self._check_rest(scaler, self._gather_stolen(finf=scaler))
            finf = None
        else:
            self._gather_stolen()
            finf = self._found_inf.data_ptr() if self._found_inf is not None else None
        g16 = f.grad16.data_ptr() if f.grad16 is not None else None
        s16 = f.shadow16.data_ptr() if f.shadow16 is not None else None
        if f.arena is None:
            self._launch_local(segs, n, lr_dev, g16, s16, finf, scaler)
        else:
            if g16 is not None and not self._bf16_exclusive():
                # fp32 gradients were written for the convolution parameters too (model ran outside autocast): fold the
                # 16-bit ones into the fp32 symmetric buffer and exchange that
                if f.flags16:
                    rc = _lib.lib().sod_grad_merge16(f.grad.data_ptr(), g16, f.numel, f.flags16, _lib.stream_ptr())
                else:
                    rc = _lib.lib().sod_grad_merge_bf16(f.grad.data_ptr(), g16, f.numel, _lib.stream_ptr())
                _lib.check(rc, "sod_grad_merge")
                _lib.count_launch()
            self._launch_allreduce(segs, n, lr_dev, g16, s16, finf, scaler)
        _lib.count_launch()
        if scaler is not None and self._scaler_readback is not None and not torch.cuda.is_current_stream_capturing():
            self._scaler_readback()
        f.master_grads_seen = False
        self._grads_clean = True
        self._clean_version = self._grad_versions()
        self._stepped = True
        self.steps += 1

    def shard_bounds(self, rank: int, world: int) -> tuple[int, int]:
        """element range of the flat buffers rank `rank` owns in the world > 1 step kernels (csrc/sgd.cu: ceil(nvec/W)
        float4s)"""
        nvec = self.flat.numel // 4
        shard = (nvec + world - 1) // world
        return min(rank * shard, nvec) * 4, min((rank + 1) * shard, nvec) * 4

    @torch.no_grad()
    def gather_state(self) -> None:
        """world > 1: every rank only ever updates the optimizer state of the shard it owns (ZeRO-1 style); bring the
        full buffers up to date on every rank.  COLLECTIVE (torch.distributed broadcasts, not on the hot path) — called by
        `state_dict()`, so `state_dict()` must be entered by all ranks, like the reference's DDP/amp save path runs on
        every process before rank 0 writes the file (utils/pipeline_ops.py:46-78)."""
        f = self.flat
        if f.arena is None:
            return
        import torch.distributed as dist
        world = f.arena.world
        for buf in self._state_buffers():
            for r in range(world):
                lo, hi = self.shard_bounds(r, world)
                if hi > lo:
                    dist.broadcast(buf[lo:hi], src=dist.get_global_rank(f.arena.group, r), group=f.arena.group)

    # -- CUDA-graph capture: the warm-up iterations must not move the training state ------------------------
    def snapshot(self) -> dict:
        """copies of everything a step changes: parameters, optimizer state, the 16-bit shadow, the step counts, the loss
        scaler"""
        return dict(tensors=[t.clone() for t in self._snapshot_tensors()], steps=self.steps, stepped=self._stepped)

    @torch.no_grad()
    def restore(self, snap: dict) -> None:
        for t, old in zip(self._snapshot_tensors(), snap["tensors"]):
            t.copy_(old)
        self.steps, self._stepped = snap["steps"], snap["stepped"]

    def _snapshot_tensors(self) -> list[torch.Tensor]:
        f = self.flat
        return [f.param, *self._state_buffers()] + ([f.shadow16] if f.shadow16 is not None else []) + \
            ([f.scaler] if f.scaler is not None else [])


class FusedSGD(FusedOptimizer):
    """SGD with momentum / weight decay as one flat sm_90a kernel; gradient averaging folded in when
    distributed.  Arithmetic = torch.optim.SGD (torch/optim/sgd.py:343-380) with dampening 0, Nesterov per group."""

    def __init__(self, params, lr=1e-3, momentum=0.0, weight_decay=0.0, nesterov=False, model: nn.Module | None = None):
        if nesterov and momentum <= 0:
            raise ValueError("Nesterov momentum requires a momentum and zero dampening")     # torch.optim.SGD's rule
        defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=bool(nesterov), dampening=0)
        super().__init__(params, defaults, model)

    def _state_buffers(self):
        return [self.flat.mom]

    def _segment(self, b, e, g, flags):
        if g is None:
            return _lib.sod_sgd_segment(b, e, 0.0, 0.0, 0.0, flags)
        if g.get("nesterov"):
            flags |= _lib.SOD_SEG_NESTEROV
        return _lib.sod_sgd_segment(b, e, float(g["lr"]), float(g["weight_decay"]), float(g["momentum"]), flags)

    def _launch_local(self, segs, n, lr_dev, g16, s16, finf, scaler=None):
        f = self.flat
        flags = _lib.SOD_SGD_ZERO_GRAD | f.flags16
        if scaler is not None:
            rc = _lib.lib().sod_sgd_momentum_scaler(f.param.data_ptr(), f.mom.data_ptr(), f.grad.data_ptr(), g16, s16, f.numel,
                                                    segs, n, lr_dev, scaler, flags, _lib.stream_ptr())
        else:
            rc = _lib.lib().sod_sgd_momentum(f.param.data_ptr(), f.mom.data_ptr(), f.grad.data_ptr(), g16, s16, f.numel,
                                             segs, n, lr_dev, float(self.inv_scale), finf, flags, _lib.stream_ptr())
        _lib.check(rc, "sod_sgd_momentum")

    def _launch_allreduce(self, segs, n, lr_dev, g16, s16, finf, scaler=None):
        f = self.flat
        flags = _lib.SOD_SGD_ZERO_GRAD | f.flags16
        g16_off = f.grad16_off if g16 is not None else 0
        if scaler is not None:
            rc = _lib.lib().sod_allreduce_sgd_scaler(f.arena.ref, f.grad_off, g16_off, f.param_off, f.mom.data_ptr(), s16,
                                                     f.numel, segs, n, lr_dev, scaler, flags, _lib.stream_ptr())
        else:
            rc = _lib.lib().sod_allreduce_sgd(f.arena.ref, f.grad_off, g16_off, f.param_off, f.mom.data_ptr(), s16, f.numel,
                                              segs, n, lr_dev, float(self.inv_scale), finf, flags, _lib.stream_ptr())
        _lib.check(rc, "sod_allreduce_sgd")

    def gather_momentum(self) -> None:
        """world > 1: the full momentum buffer on every rank (collective; see `gather_state`)"""
        self.gather_state()

    # momentum lives in the flat buffer; expose torch.optim.SGD's state layout on demand
    def state_dict(self):
        self.gather_state()
        self.state.clear()
        if self._stepped:
            for g in self.param_groups:
                for p in g["params"]:
                    self.state[p] = {"momentum_buffer": self.flat.momentum_view(p).clone()}
        sd = super().state_dict()
        self.state.clear()
        return sd

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        loaded = False
        with torch.no_grad():
            for g in self.param_groups:
                for p in g["params"]:
                    buf = self.state.get(p, {}).get("momentum_buffer")
                    if buf is not None:
                        self.flat.momentum_view(p).copy_(buf)
                        loaded = True
        self.state.clear()
        self._stepped = self._stepped or loaded
        self.flat.refresh_shadow()

    def __repr__(self):
        return super().__repr__().replace("FusedSGD", "FusedSGD[sm_90a flat]", 1)


class FusedAdam(FusedOptimizer):
    """torch.optim.Adam (amsgrad=False, maximize=False, L2 weight decay) as one flat sm_90a kernel, gradient averaging
    folded in when distributed — the optimizer of the reference's optim "adam" (utils/pipeline_ops.py:287-294).
    `flat.mom` holds exp_avg, `exp_avg_sq` sits beside it; the step count of every segment lives on the device
    (`step_dev`) and is advanced by the kernel, so a captured iteration replays with the right bias correction and an
    amp-overflow skip leaves it alone."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False, *,
                 maximize=False, decoupled_weight_decay=False, model: nn.Module | None = None, **_ignored):
        if amsgrad or maximize or decoupled_weight_decay:
            raise _lib.SodError("FusedAdam implements Adam without amsgrad, maximize or decoupled weight decay "
                                "(the reference's optim 'adam' sets none of them)")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0 or eps < 0.0:
            raise ValueError(f"invalid betas {betas} or eps {eps}")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                        foreach=None, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False)
        super().__init__(params, defaults, model)
        self.exp_avg_sq = torch.zeros_like(self.flat.mom)
        # int32[SOD_ADAM_STEP_WORDS]: the step count of every segment of _segment_plan(), then the kernel's ticket word
        self.step_dev = torch.zeros(_lib.SOD_ADAM_STEP_WORDS, dtype=torch.int32, device=self.flat.device)

    @property
    def exp_avg(self) -> torch.Tensor:
        return self.flat.mom

    def _state_buffers(self):
        return [self.flat.mom, self.exp_avg_sq]

    def _snapshot_tensors(self):
        return super()._snapshot_tensors() + [self.step_dev]

    def _segment(self, b, e, g, flags):
        if g is None:
            return _lib.sod_adam_segment(b, e, 0.0, 0.0, 0.0, 0.0, 0.0, flags)
        b1, b2 = g["betas"]
        return _lib.sod_adam_segment(b, e, float(g["lr"]), float(g["weight_decay"]), float(b1), float(b2), float(g["eps"]),
                                     flags)

    def _launch_local(self, segs, n, lr_dev, g16, s16, finf, scaler=None):
        f = self.flat
        flags = _lib.SOD_SGD_ZERO_GRAD | f.flags16
        if scaler is not None:
            rc = _lib.lib().sod_adam_scaler(f.param.data_ptr(), f.mom.data_ptr(), self.exp_avg_sq.data_ptr(), f.grad.data_ptr(),
                                            g16, s16, f.numel, segs, n, lr_dev, self.step_dev.data_ptr(), scaler, flags,
                                            _lib.stream_ptr())
        else:
            rc = _lib.lib().sod_adam(f.param.data_ptr(), f.mom.data_ptr(), self.exp_avg_sq.data_ptr(), f.grad.data_ptr(), g16,
                                     s16, f.numel, segs, n, lr_dev, self.step_dev.data_ptr(), float(self.inv_scale), finf,
                                     flags, _lib.stream_ptr())
        _lib.check(rc, "sod_adam")

    def _launch_allreduce(self, segs, n, lr_dev, g16, s16, finf, scaler=None):
        f = self.flat
        flags = _lib.SOD_SGD_ZERO_GRAD | f.flags16
        g16_off = f.grad16_off if g16 is not None else 0
        if scaler is not None:
            rc = _lib.lib().sod_allreduce_adam_scaler(f.arena.ref, f.grad_off, g16_off, f.param_off, f.mom.data_ptr(),
                                                      self.exp_avg_sq.data_ptr(), s16, f.numel, segs, n, lr_dev,
                                                      self.step_dev.data_ptr(), scaler, flags, _lib.stream_ptr())
        else:
            rc = _lib.lib().sod_allreduce_adam(f.arena.ref, f.grad_off, g16_off, f.param_off, f.mom.data_ptr(),
                                               self.exp_avg_sq.data_ptr(), s16, f.numel, segs, n, lr_dev,
                                               self.step_dev.data_ptr(), float(self.inv_scale), finf, flags,
                                               _lib.stream_ptr())
        _lib.check(rc, "sod_allreduce_adam")

    def group_steps(self) -> list[int]:
        """the step count of every param_group (host sync)"""
        steps = self.step_dev.tolist()
        return [steps[idx[0]] if idx else 0 for idx in self._group_segments()]

    # the state lives in the flat buffers; expose torch.optim.Adam's layout on demand
    def state_dict(self):
        self.gather_state()
        self.state.clear()
        for g, t in zip(self.param_groups, self.group_steps()):
            if t == 0:
                continue                       # torch creates a parameter's state at its first step
            for p in g["params"]:
                self.state[p] = {"step": torch.tensor(float(t), dtype=torch.float32),
                                 "exp_avg": self.flat.momentum_view(p).clone(),
                                 "exp_avg_sq": FlatParams._view(self.exp_avg_sq, self.flat.offset_of(p), p.data).clone()}
        sd = super().state_dict()
        self.state.clear()
        return sd

    def load_state_dict(self, state_dict):
        """torch.optim.Adam's layout; `step` may be a tensor or (torch of 2020, which the reference ran) an int"""
        super().load_state_dict(state_dict)
        try:
            steps = []
            for g in self.param_groups:
                ts = {int(float(self.state[p]["step"])) if "step" in self.state.get(p, {}) else 0 for p in g["params"]}
                if len(ts) > 1:
                    raise _lib.SodError(f"the parameters of one group carry different Adam steps {sorted(ts)}: the fused "
                                        "step keeps one count per group")
                steps.append(ts.pop() if ts else 0)
            with torch.no_grad():
                for g in self.param_groups:
                    for p in g["params"]:
                        st = self.state.get(p, {})
                        if "exp_avg" in st:
                            self.flat.momentum_view(p).copy_(st["exp_avg"])
                            FlatParams._view(self.exp_avg_sq, self.flat.offset_of(p), p.data).copy_(st["exp_avg_sq"])
                counts = [0] * _lib.SOD_ADAM_STEP_WORDS
                for idx, t in zip(self._group_segments(), steps):
                    for n in idx:
                        counts[n] = t
                self.step_dev.copy_(torch.tensor(counts, dtype=torch.int32))
        finally:
            self.state.clear()
        self._stepped = self._stepped or any(steps)
        self.flat.refresh_shadow()

    def __repr__(self):
        return super().__repr__().replace("FusedAdam", "FusedAdam[sm_90a flat]", 1)


def make_optimizer(model: nn.Module, optimizer_type: str, optimizer_info: dict) -> Optimizer:
    """Parameter grouping rules of reference utils/pipeline_ops.py:235-316, FusedSGD underneath."""
    lr, mom = optimizer_info["lr"], optimizer_info["momentum"]
    wd, nest = optimizer_info["weight_decay"], optimizer_info.get("nesterov", False)
    named = list(model.named_parameters())
    if optimizer_type == "sgd_trick":
        is_light = lambda n: "bias" in n or "bn" in n                     # noqa: E731
        groups = [{"params": [p for n, p in named if is_light(n)], "weight_decay": 0},
                  {"params": [p for n, p in named if not is_light(n)]}]
        return FusedSGD(groups, lr=lr, momentum=mom, weight_decay=wd, nesterov=nest, model=model)
    if optimizer_type == "sgd_r3":
        groups = [{"params": [p for n, p in named if n[-4:] == "bias"], "lr": 2 * lr},
                  {"params": [p for n, p in named if n[-4:] != "bias"], "lr": lr, "weight_decay": wd}]
        return FusedSGD(groups, momentum=mom, model=model)
    if optimizer_type == "sgd_all":
        return FusedSGD([p for _, p in named], lr=lr, weight_decay=wd, momentum=mom, model=model)
    if optimizer_type == "adam":
        return FusedAdam(model.parameters(), lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd, model=model)
    if optimizer_type == "f3_trick":
        backbone = [p for n, p in named if n.startswith("div") and not n.startswith("div_2")]
        head = [p for n, p in named if not n.startswith("div")]
        groups = [{"params": backbone, "lr": 0.1 * lr}, {"params": head, "lr": lr}]
        return FusedSGD(groups, momentum=mom, weight_decay=wd, nesterov=nest, model=model)
    raise NotImplementedError(optimizer_type)


class CustomScheduler:
    """LR schedules of reference utils/pipeline_ops.py:185-232, including its quirk: the coefficient is
    evaluated once per param group and the warmup branches shrink `total_num` on every evaluation."""

    def __init__(self, optimizer: Optimizer, total_num: int, scheduler_type: str, scheduler_info: dict):
        self.lr_group = [g["lr"] for g in optimizer.param_groups]
        self.total_num, self.type, self.info = total_num, scheduler_type, scheduler_info

    def _coefficient(self, curr: int):
        kind, decay = self.type, self.info["lr_decay"]
        if kind == "poly":
            return pow(1 - float(curr) / self.total_num, decay)
        if kind in ("poly_warmup", "cosine_warmup"):
            turn = self.info["warmup_epoch"]
            if curr < turn:
                return 1 / turn * (1 + curr)
            curr -= turn - 1
            self.total_num -= turn - 1
            if kind == "poly_warmup":
                return pow(1 - float(curr) / self.total_num, decay)
            return (1 + np.cos(np.pi * curr / self.total_num)) / 2
        if kind == "f3_sche":
            return 1 - abs((curr + 1) / (self.total_num + 1) * 2 - 1)
        raise NotImplementedError(kind)

    def step(self, optimizer: Optimizer, curr_epoch: int):
        for i, g in enumerate(optimizer.param_groups):
            g["lr"] = self.lr_group[i] * self._coefficient(curr_epoch)

    def __str__(self):
        return f"Scheduler:\n\tType: {self.type}\n\tInfo: {self.info}\n"
