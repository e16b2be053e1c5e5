"""One training iteration of the reference (train.py:284-310), wired onto the sm_90a kernels.

`Trainer` performs exactly the construction sequence of the reference's `main_worker` (train.py:141-207):
model factory → make_optimizer → convert_syncbn_model (+ convert_wsgn_model) → amp.initialize → DDP → loss list; and `step` is the
loop body: forward, get_total_loss, zero_grad, backward, step, loss mean.  It is what `train.py`, `bench.py`,
the parity tests and `__graft_entry__.smoke()` all drive, so the measured path is the shipped path.
"""
from __future__ import annotations

import os

import torch

from . import _lib, amp, comm, network, syncbn
from .loss import CEL, BCEWithLogitsLoss, _FusedLossFn, get_total_loss
from .optim import CustomScheduler, make_optimizer
from .parallel import DistributedDataParallel
from .syncbn import convert_syncbn_model
from .wsgn import convert_wsgn_model
from .utils import init_seed

# overlap the next batch's host→device copy with the running iteration (see Trainer._stage_inputs).
# SOD_E2E_PREFETCH=0 restores the serialized copy.
PREFETCH_H2D = os.environ.get("SOD_E2E_PREFETCH", "1") == "1"


class Trainer:
    def __init__(self, model_name: str = "res50", lr: float = 0.05, momentum: float = 0.9, weight_decay: float = 5e-4,
                 nesterov: bool = False, optim: str = "f3_trick", reduction: str = "mean", use_aux_loss: bool = True,
                 dtype: torch.dtype = torch.bfloat16, channels_last: bool = True, seed: int = 0,
                 device: torch.device | None = None, report_items: bool = True, use_graph: bool = False,
                 native_interpolate: bool = True, shadow_weights: bool = True):
        if not torch.cuda.is_available():
            raise RuntimeError("the engine needs a CUDA device")
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.world = comm.world_size()
        self.channels_last = channels_last
        self.report_items = report_items
        from . import resample as _resample
        from .network import blocks as _blocks
        _blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = bool(native_interpolate)
        _resample.ENABLED = bool(native_interpolate)
        init_seed(seed)                                                    # train.py:113
        model = getattr(network, model_name)().to(self.device)            # train.py:141
        if channels_last:
            model = model.to(memory_format=torch.channels_last)           # before the optimizer flattens storage
        self.optimizer = make_optimizer(model, optim, dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                                                           nesterov=nesterov))    # train.py:157
        model = convert_syncbn_model(model)                                # train.py:180 (also at world 1: fused BN)
        model = convert_wsgn_model(model)                                  # WS-GN backbone: GroupNorm / WS kernels
        self.use_amp = dtype != torch.float32
        if self.use_amp:
            model, self.optimizer = amp.initialize(model, self.optimizer, opt_level="O1", dtype=dtype,
                                                   shadow_weights=shadow_weights)                  # train.py:183
        if self.world > 1:
            model = DistributedDataParallel(model, delay_allreduce=True)   # train.py:185
        self.model = model
        self.loss_funcs = [BCEWithLogitsLoss(reduction=reduction)]         # train.py:203
        if use_aux_loss:
            self.loss_funcs.append(CEL())                                  # train.py:204-207
        self.model.train()
        self._pinned_loss = torch.zeros(1, dtype=torch.float32).pin_memory()
        self._loss_event: torch.cuda.Event | None = None
        # CUDA-graph replay of the whole iteration (SURVEY §8f.1): one cudaGraphLaunch instead of ~1500 launches.
        # One graph per input shape (multi-scale training, reference utils/dataset.py:125-132, cycles through three);
        # learning rates are read from a device table (FusedOptimizer.sync_lr), so the scheduler never forces a re-capture.
        # fp16's dynamic loss scale lives on the device (amp.py), so it replays too.
        from .optim import FusedOptimizer
        self.use_graph = use_graph and isinstance(self.optimizer, FusedOptimizer) and \
            (not amp._cfg["dynamic"] or self.optimizer.flat.scaler is not None)
        self._graphs: dict = {}
        self._cur = None

    @property
    def module(self):
        return self.model.module if hasattr(self.model, "module") else self.model

    def scheduler(self, total_num: int, lr_type: str = "poly", lr_decay: float = 0.9, warmup_epoch: int = 1):
        return CustomScheduler(self.optimizer, total_num, lr_type, dict(lr_decay=lr_decay, warmup_epoch=warmup_epoch))

    def check_errors(self) -> None:
        """raise if a device-side barrier / packet wait of either arena timed out (host sync: call it at log points)"""
        for arena in (getattr(self.model, "arena", None), comm.small_arena() if self.world > 1 else None):
            if arena is not None:
                arena.check_error()

    # ----------------------------------------------------------------------------------------------
    def _iteration(self, x: torch.Tensor, m: torch.Tensor, report: bool):
        if self.channels_last:
            x = x.contiguous(memory_format=torch.channels_last)
        amp.push()                                                         # host writes of the loss scale (fp16)
        preds = self.model(x)                                              # train.py:293
        unit = not amp._cfg["dynamic"]
        # fp16: the fused loss forms its gradient already multiplied by the device loss scale; scale_loss multiplies the
        # loss by the same tensor, so backward hands that gradient on untouched
        sdev = amp.scale_tensor() if self.use_amp and amp._cfg["dynamic"] else None
        extra = (sdev,) if sdev is not None else ()
        if len(self.loss_funcs) == 2 and not report:
            holder: list = []
            loss = _FusedLossFn.apply(preds, m, self.loss_funcs[0].reduction, 1.0, 1.0, 1e-6, unit, 0, holder, *extra)
            items = holder[0]                                              # device scalars [bce, cel, total, ...]
        else:
            loss, items = get_total_loss(preds, m, self.loss_funcs, unit_upstream=unit, scale_dev=sdev)   # train.py:295
        self.optimizer.zero_grad()                                         # train.py:297
        if self.use_amp:
            with amp.scale_loss(loss, self.optimizer) as scaled:           # train.py:299
                scaled.backward()
        else:
            loss.backward()                                                # train.py:302
        self.optimizer.step()                                              # train.py:303
        reduced = comm.allreduce_tensor(loss.detach()) if self.world > 1 else loss.detach()   # train.py:306
        return reduced, items, preds

    def _capture(self, x: torch.Tensor, m: torch.Tensor) -> dict:
        """warm up eagerly on a side stream, then record one whole iteration into a CUDA graph"""
        static_x, static_m = x.clone(), m.clone()
        amp.push()                                   # a pending host write of the loss scale belongs to the state kept
        # the warm-up iterations (allocator, cuDNN autotune, autograd thread) must not move the training state
        snap = self.optimizer.snapshot()             # parameters, optimizer state (Adam: its step counts), shadow, scaler
        buffers = [b.clone() for b in self.module.buffers()]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                self._iteration(static_x, static_m, report=False)
        torch.cuda.current_stream().wait_stream(side)
        self.optimizer.restore(snap)
        if amp._cfg["dynamic"]:
            amp.read_scaler()                        # the host mirror back to the restored scaler
        with torch.no_grad():
            for b, old in zip(self.module.buffers(), buffers):
                b.copy_(old)
        if self.world > 1:
            torch.distributed.barrier()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        launches0 = _lib.launches
        syncbn.begin_iteration(self.device, graph=True)
        try:
            with torch.cuda.graph(graph):
                red, items, preds = self._iteration(static_x, static_m, report=False)
                syncbn.end_iteration(self.device)
        finally:
            syncbn.begin_iteration(self.device, graph=False)
        # capturing records, it does not execute: the optimizer has not stepped
        self.optimizer.steps, self.optimizer._stepped = snap["steps"], snap["stepped"]
        return dict(graph=graph, x=static_x, m=static_m, out=(red, items, preds), launches=_lib.launches - launches0)

    def _graph_for(self, x: torch.Tensor, m: torch.Tensor) -> dict:
        key = (tuple(x.shape), tuple(m.shape), x.dtype)
        ent = self._graphs.get(key)
        if ent is None:                                       # first call with this input size
            ent = self._graphs[key] = self._capture(x, m)
        self._cur = ent
        return ent

    def _replay(self, ent: dict) -> None:
        self.optimizer.sync_lr()                              # param_groups[i]["lr"] → device table, only when it moved
        amp.push()                                            # host writes of the fp16 loss scale, only when there are any
        ent["graph"].replay()
        self.optimizer.steps += 1
        self.optimizer._stepped = True
        _lib.count_launch(ent["launches"])

    def forward_backward_update(self, x: torch.Tensor, m: torch.Tensor, report: bool | None = None):
        """device tensors in, device loss out; no host synchronisation unless report strings are requested"""
        report = self.report_items if report is None else report
        if not self.use_graph:
            return self._iteration(x, m, report)
        ent = self._graph_for(x, m)
        ent["x"].copy_(x, non_blocking=True)
        ent["m"].copy_(m, non_blocking=True)
        self._replay(ent)
        red, items, preds = ent["out"]
        if report:
            items = [f"{v:.5f}" for v in items[:2].tolist()]
        return red, items, preds

    def step(self, x: torch.Tensor, m: torch.Tensor) -> dict:
        """the loop body with the reference's reporting: returns python floats / strings (host sync)."""
        reduced, items, preds = self.forward_backward_update(x, m)
        return dict(loss=float(reduced.item()), items=items if isinstance(items, list) else
                    [f"{v:.5f}" for v in items[:2].tolist()], preds=preds.detach())

    def step_from_host(self, x_pinned: torch.Tensor, m_pinned: torch.Tensor):
        """end-to-end form: pinned host batch → device (train.py:291-292) → iteration → loss back to pinned host
        memory.  The D2H read is asynchronous; `last_loss()` waits for it."""
        key = (tuple(x_pinned.shape), tuple(m_pinned.shape), x_pinned.dtype)
        ent = self._graphs.get(key) if self.use_graph else None
        if ent is not None:
            if PREFETCH_H2D:
                self._stage_inputs(ent, x_pinned, m_pinned)
            else:
                # H2D straight into the graph's static inputs
                ent["x"].copy_(x_pinned, non_blocking=True)
                ent["m"].copy_(m_pinned, non_blocking=True)
            self._replay(ent)
            reduced = ent["out"][0]
        else:
            x = x_pinned.to(self.device, non_blocking=True)
            m = m_pinned.to(self.device, non_blocking=True)
            reduced, _, _ = self.forward_backward_update(x, m, report=False)
        self._pinned_loss.copy_(reduced.reshape(1), non_blocking=True)
        self._loss_event = torch.cuda.Event()
        self._loss_event.record()

    def _stage_inputs(self, ent: dict, x_pinned: torch.Tensor, m_pinned: torch.Tensor) -> None:
        """(PREFETCH_H2D, default on) the H2D copy of this call's batch runs on a copy
        stream into one of two staging buffers, so it overlaps the previous call's iteration (the host loop runs ahead:
        nothing in `step_from_host` blocks); the iteration's stream then only pays a device-to-device copy into the
        graph's static inputs.  Same contract as the plain path: every step's H2D and D2H stay inside the caller's
        timed region.  (The reference prefetches too: `BackgroundGenerator(tr_loader, max_prefetch=2)`, train.py:278-285.)"""
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        st = ent.get("stage")
        if st is None:                                   # two staging buffers per captured input size
            st = ent["stage"] = dict(buf=[(torch.empty_like(ent["x"]), torch.empty_like(ent["m"])) for _ in range(2)],
                                     ready=[torch.cuda.Event(), torch.cuda.Event()],     # H2D into stage k has finished
                                     free=[None, None],                                  # the D2D out of stage k has finished
                                     idx=0)
        k = st["idx"]
        st["idx"] ^= 1
        cs, main = self._copy_stream, torch.cuda.current_stream()
        if st["free"][k] is not None:
            cs.wait_event(st["free"][k])
        with torch.cuda.stream(cs):
            st["buf"][k][0].copy_(x_pinned, non_blocking=True)
            st["buf"][k][1].copy_(m_pinned, non_blocking=True)
            st["ready"][k].record(cs)
        main.wait_event(st["ready"][k])
        ent["x"].copy_(st["buf"][k][0])
        ent["m"].copy_(st["buf"][k][1])
        free = torch.cuda.Event()
        free.record(main)
        st["free"][k] = free

    def last_loss(self) -> float:
        if self._loss_event is not None:
            self._loss_event.synchronize()
        return float(self._pinned_loss[0])
