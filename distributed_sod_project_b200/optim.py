"""Optimizer seam: `make_optimizer`, `CustomScheduler`, and `FusedSGD` (csrc/sgd.cu underneath).

Reference surface kept (paths in the reference repo):
* `make_optimizer(model, optimizer_type, optimizer_info)`          — utils/pipeline_ops.py:235-316
  (`sgd_trick`, `sgd_r3`, `sgd_all`, `f3_trick` → FusedSGD; `adam` → torch.optim.Adam, not on the hot path)
* `CustomScheduler(optimizer, total_num, scheduler_type, scheduler_info).step(optimizer, curr_epoch)`
                                                                     — utils/pipeline_ops.py:185-232
* the `torch.optim.Optimizer` protocol the loop relies on: `.param_groups[i]["lr"]` mutated from outside,
  `.zero_grad()`, `.step()`, `.state_dict()/.load_state_dict()` with per-parameter `momentum_buffer`
  (utils/pipeline_ops.py:73,118), `str(optimizer)` (train.py:176).

FusedSGD keeps parameters, gradients and momentum in three flat fp32 buffers laid out group-major
([group 0 | group 1 | … | parameters in no group]); every `p.data` / `p.grad` is a view into them.  `step()`
is one kernel: world 1 → `sod_sgd_momentum`; world > 1 (after `DistributedDataParallel` has moved the flat
parameter and gradient buffers into symmetric memory) → `sod_allreduce_sgd`, which also does the
gradient averaging, so nothing else runs between backward and the next forward.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn
from torch.optim import Adam, Optimizer

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
            raise _lib.SodError("FusedSGD needs fp32 parameters on one device")
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
        self.shadow16: torch.Tensor | None = None   # bf16 copy of `param`, refreshed by the fused step (amp O1 shadow)
        self.grad16: torch.Tensor | None = None     # bf16 gradients autograd accumulates for the shadowed tensors
        # bf16 shadow leaves the convolutions consume (amp._install_shadow_weights): (leaf, element offset, steal)
        # steal=True: `.grad` is left None so that autograd hands over cuDNN's gradient tensor as it is (no accumulate
        # kernel per parameter); FusedSGD.step collects all of them into `grad16` with one sod_grad_gather16 launch
        self.shadow_leaves: list[tuple[torch.Tensor, int, bool]] = []
        # set by a hook on the fp32 masters of shadowed parameters (amp._install_shadow_weights) when a gradient reaches one
        # of them — the model ran outside autocast — and cleared by the step that has consumed it
        self.master_grads_seen = False
        self._bind(copy_from_params=True)

    # -- mixed precision: bf16 shadow of the fp32 master ---------------------------------------------------
    def enable_shadow(self, dtype: torch.dtype = torch.bfloat16) -> None:
        if dtype != torch.bfloat16:
            raise _lib.SodError("the shadow copy is bf16 (fp16 needs dynamic loss scaling: handled without a shadow)")
        if self.shadow16 is None:
            self.shadow16 = torch.zeros(self.numel, dtype=dtype, device=self.device)
            self.grad16 = torch.zeros(self.numel, dtype=dtype, device=self.device)
        self.refresh_shadow()

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


class FusedSGD(Optimizer):
    """SGD with momentum / weight decay as one flat sm_90a kernel; gradient averaging folded in when
    distributed.  Arithmetic = torch.optim.SGD (torch/optim/sgd.py:343-380) with dampening 0, nesterov False."""

    def __init__(self, params, lr=1e-3, momentum=0.0, weight_decay=0.0, nesterov=False, model: nn.Module | None = None):
        if nesterov:
            raise _lib.SodError("nesterov momentum is not on the reference's hot path (config.py:65 nesterov=False)")
        defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=False, dampening=0)
        super().__init__(params, defaults)
        if 2 * (len(self.param_groups) + 1) > _lib.SOD_MAX_SEGMENTS:
            raise _lib.SodError(f"at most {_lib.SOD_MAX_SEGMENTS // 2 - 1} parameter groups")
        grouped = {id(p) for g in self.param_groups for p in g["params"]}
        leftovers = [p for p in model.parameters() if id(p) not in grouped] if model is not None else []
        conv_ids = {id(p) for m in model.modules() if isinstance(m, nn.Conv2d) for p in (m.weight, m.bias) if p is not None} \
            if model is not None else set()
        self.flat = FlatParams([list(g["params"]) for g in self.param_groups], leftovers, bf16_grad_ids=conv_ids)
        for p, _ in self.flat.slots:
            flat_registry[id(p)] = self.flat
        self.inv_scale = 1.0                   # amp: 1/S for the coming step
        self.found_inf: torch.Tensor | None = None  # amp: device uint32 flag, or None
        self._grads_clean = True
        self._clean_version = self._grad_versions()
        self._stepped = False
        self.steps = 0
        # learning rates as the kernels read them: a device table, rewritten (tiny fill kernels, by value) only when a
        # param_group's lr has changed — so a captured iteration follows the scheduler without being re-captured
        self._lr_dev = torch.zeros(_lib.SOD_MAX_SEGMENTS, dtype=torch.float32, device=self.flat.device) \
            if self.flat.device.type == "cuda" else None
        self._lr_sent: list[float | None] = [None] * _lib.SOD_MAX_SEGMENTS

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

    def _gather_stolen(self) -> None:
        """bf16 gradients autograd left in their own tensors (shadow leaves with steal=True, or any leaf whose `.grad`
        was replaced) → flat `grad16`, one launch for all of them"""
        f = self.flat
        if not f.shadow_leaves:
            return
        base = f.grad16.data_ptr()
        items = []
        for leaf, off, _ in f.shadow_leaves:
            g = leaf.grad
            if g is None or g.data_ptr() == base + 2 * off:
                continue
            if g.dtype == f.grad16.dtype and g.is_cuda and g.numel() == leaf.numel() and _same_physical_order(g, leaf):
                items.append((g.data_ptr(), off, g.numel()))
            else:                                            # unusual layout / dtype: plain torch accumulate
                FlatParams._view(f.grad16, off, leaf).add_(g.to(f.grad16.dtype))
        if items:
            key = tuple(items)
            if getattr(self, "_gather_key", None) != key:    # eager steps see new addresses every time, graph capture once
                self._gather_key = key
                self._gather_arr = (_lib.sod_gather_item * len(items))(*[_lib.sod_gather_item(a, b, c) for a, b, c in items])
            arr = self._gather_arr
            rc = _lib.lib().sod_grad_gather16(arr, len(items), base, f.numel, _lib.stream_ptr())
            _lib.check(rc, "sod_grad_gather16")
            _lib.count_launch((len(items) + _lib.SOD_GATHER_MAX_ITEMS - 1) // _lib.SOD_GATHER_MAX_ITEMS)

    def _segments(self):
        plan = self._segment_plan()
        exclusive = self._bf16_exclusive()
        segs = (_lib.sod_sgd_segment * max(len(plan), 1))()
        for n, (b, e, g, bf16_part) in enumerate(plan):
            flags = _lib.SOD_SEG_GRAD16 if (bf16_part and exclusive) else 0
            if g is None:
                segs[n] = _lib.sod_sgd_segment(b, e, 0.0, 0.0, 0.0, flags | _lib.SOD_SEG_FROZEN)
            else:
                segs[n] = _lib.sod_sgd_segment(b, e, float(g["lr"]), float(g["weight_decay"]), float(g["momentum"]), flags)
        return segs, len(plan)

    @torch.no_grad()
    def step(self, closure=None):
        if closure is not None:
            raise _lib.SodError("closures are not supported by the fused step")
        f = self.flat
        if not f.param.is_cuda:
            raise _lib.SodError("FusedSGD.step needs CUDA parameters (no CPU fallback)")
        segs, n = self._segments()
        self.sync_lr()
        lr_dev = self._lr_dev.data_ptr()
        self._gather_stolen()
        finf = self.found_inf.data_ptr() if self.found_inf is not None else None
        g16 = f.grad16.data_ptr() if f.grad16 is not None else None
        s16 = f.shadow16.data_ptr() if f.shadow16 is not None else None
        if f.arena is None:
            rc = _lib.lib().sod_sgd_momentum(f.param.data_ptr(), f.mom.data_ptr(), f.grad.data_ptr(), g16, s16, f.numel,
                                             segs, n, lr_dev, float(self.inv_scale), finf, _lib.SOD_SGD_ZERO_GRAD,
                                             _lib.stream_ptr())
            _lib.check(rc, "sod_sgd_momentum")
        else:
            a = f.arena
            if g16 is not None and not self._bf16_exclusive():
                # fp32 gradients were written for the convolution parameters too (model ran outside autocast): fold the
                # bf16 ones into the fp32 symmetric buffer and exchange that
                rc = _lib.lib().sod_grad_merge_bf16(f.grad.data_ptr(), g16, f.numel, _lib.stream_ptr())
                _lib.check(rc, "sod_grad_merge_bf16")
                _lib.count_launch()
            rc = _lib.lib().sod_allreduce_sgd(a.ref, f.grad_off, f.grad16_off if g16 is not None else 0, f.param_off,
                                              f.mom.data_ptr(), s16, f.numel, segs, n, lr_dev, float(self.inv_scale), finf,
                                              _lib.SOD_SGD_ZERO_GRAD, _lib.stream_ptr())
            _lib.check(rc, "sod_allreduce_sgd")
        _lib.count_launch()
        f.master_grads_seen = False
        self._grads_clean = True
        self._clean_version = self._grad_versions()
        self._stepped = True
        self.steps += 1

    def shard_bounds(self, rank: int, world: int) -> tuple[int, int]:
        """element range of the flat buffers rank `rank` owns in `sod_allreduce_sgd` (csrc/sgd.cu: ceil(nvec/W) float4s)"""
        nvec = self.flat.numel // 4
        shard = (nvec + world - 1) // world
        return min(rank * shard, nvec) * 4, min((rank + 1) * shard, nvec) * 4

    @torch.no_grad()
    def gather_momentum(self) -> None:
        """world > 1: every rank only ever updates the momentum of the shard it owns (ZeRO-1 style); bring the full
        buffer up to date on every rank.  COLLECTIVE (torch.distributed broadcasts, not on the hot path) — called by
        `state_dict()`, so `state_dict()` must be entered by all ranks, like the reference's DDP/amp save path runs on
        every process before rank 0 writes the file (utils/pipeline_ops.py:46-78)."""
        f = self.flat
        if f.arena is None:
            return
        import torch.distributed as dist
        world = f.arena.world
        for r in range(world):
            lo, hi = self.shard_bounds(r, world)
            if hi > lo:
                dist.broadcast(f.mom[lo:hi], src=dist.get_global_rank(f.arena.group, r), group=f.arena.group)

    # momentum lives in the flat buffer; expose torch.optim.SGD's state layout on demand
    def state_dict(self):
        self.gather_momentum()
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
        return Adam(model.parameters(), lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
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
