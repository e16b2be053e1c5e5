#!/usr/bin/env python
"""Training entry point with the reference's command line and configuration surface.

    python train.py [-n NODES] [-ng GPUS_PER_NODE] [--ip IP] [-p PORT]          (reference train.py:48-60)

Same process model as the reference (`torch.multiprocessing.spawn`, one process per GPU, env:// rendezvous,
train.py:84-101) and the same construction order in `main_worker` (train.py:104-223); the hot path is this repo's
engine (`distributed_sod_project_b200/engine.py`).  NCCL is still initialised — it bootstraps the symmetric-memory
rendezvous — but no NCCL collective runs inside an iteration.

Out of scope here (SURVEY §2): TensorBoard / xlsx recorders.  Evaluation (`test`, `_test_process`) runs distributed with
GPU metrics (distributed_sod_project_b200/evaluate.py, metrics.py): on synthetic test sets by default, on the configured
on-disk sets (`te_data_list`, `val_data_path`) with `"synthetic_eval": False` (distributed_sod_project_b200/data.py).
With `"synthetic": False` training reads `rgb_data.tr_data_path` (an `Image/` + `Mask/` folder or a list file, with
`prefix`): DataLoader workers (`num_workers`) only decode, and the GPU runs the reference's JointResize(`input_size`),
flip, RandomRotate(10), ColorJitter(0.1, 0.1, 0.1), ToTensor / Normalize and the `size_list` collate, bit for bit as
Pillow and torchvision compute them (distributed_sod_project_b200/pipeline.py `TrainPrefetcher`).  The random
parameters come from generators seeded by (epoch, rank) in the main process, so a run does not depend on
`num_workers`.  A missing `tr_data_path` is an error naming it.  With `"synthetic": True` (the default) training batches
come from `synthetic.synth_batch`, which honours the dataloader's output contract, incl. the multi-scale collate.
"""
from __future__ import annotations

import argparse
import os
import random
import time

import torch
import torch.distributed as dist

from config import user_config
from distributed_sod_project_b200 import amp
from distributed_sod_project_b200.checkpoint import resume_checkpoint, save_checkpoint
from distributed_sod_project_b200.data import open_test_set
from distributed_sod_project_b200.engine import Trainer
from distributed_sod_project_b200.evaluate import shard, test_process
from distributed_sod_project_b200.synthetic import synth_batch, synth_eval_set
from distributed_sod_project_b200.utils import (AvgMeter, check_mkdir, construct_exp_name, construct_path_dict, construct_print,
                                                init_cudnn, write_data_to_file)

parser = argparse.ArgumentParser(prog="main script", description="H100-native engine behind the Distributed-SOD-Project API.",
                                 allow_abbrev=False)
parser.version = "1.0.0"
parser.add_argument("-v", "--version", action="version")
parser.add_argument("-n", "--nodes", default=1, type=int, metavar="N")
parser.add_argument("-ng", "--ngpus_per_node", default=2, type=int)
parser.add_argument("--ip", default="127.0.0.1", type=str)
parser.add_argument("-p", "--port", default="8888", type=str)

_DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def init_process(ip, port, rank, world_size):
    os.environ["MASTER_ADDR"] = ip
    os.environ["MASTER_PORT"] = port
    dist.init_process_group(backend="nccl", init_method="env://", world_size=world_size, rank=rank,
                            device_id=torch.device("cuda", rank % torch.cuda.device_count()))


class SyntheticU8Loader:
    """what the reference's DataLoader workers produce BEFORE `ToTensor` (utils/dataset.py:104-116): 8-bit HWC images and
    8-bit masks at `in_size`, pinned; the tensor-side transforms and the multi-scale collate then run on the GPU
    (distributed_sod_project_b200/pipeline.py)"""

    def __init__(self, batch_size, iters, in_size, rank, epoch_seed=0):
        self.bs, self.iters, self.in_size, self.rank, self.epoch = batch_size, iters, in_size, rank, epoch_seed

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return self.iters

    def __iter__(self):
        for i in range(self.iters):
            seed = 1234 + self.rank + 1000 * (self.epoch * self.iters + i)
            g = torch.Generator().manual_seed(seed)
            img = torch.randint(0, 256, (self.bs, self.in_size, self.in_size, 3), generator=g, dtype=torch.uint8)
            _, m = synth_batch(seed, self.bs, self.in_size)
            mask = (m[:, 0] * 255).round().to(torch.uint8)
            yield img.pin_memory(), mask.pin_memory(), [f"synthetic_{self.epoch}_{i}_{k}" for k in range(self.bs)]


class SyntheticLoader:
    """stands in for `create_loader(ImageFolder(...))` (reference utils/dataset.py:72-156): yields
    (image[N,3,S,S] f32, mask[N,1,S,S] f32 in [0,1], names); with `size_list` one size per batch, shared by all ranks."""

    def __init__(self, batch_size, iters, in_size, size_list, rank, epoch_seed=0):
        self.bs, self.iters, self.in_size, self.size_list, self.rank = batch_size, iters, in_size, size_list, rank
        self.epoch = epoch_seed

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __len__(self):
        return self.iters

    def __iter__(self):
        sizes = random.Random(self.epoch)          # same choice on every rank (shared RNG)
        for i in range(self.iters):
            size = sizes.choice(self.size_list) if self.size_list else self.in_size
            x, m = synth_batch(1234 + self.rank + 1000 * (self.epoch * self.iters + i), self.bs, size)
            yield x.pin_memory(), m.pin_memory(), [f"synthetic_{self.epoch}_{i}_{k}" for k in range(self.bs)]


def main_worker(local_rank, ngpus_per_node, world_size, args, exp_name, path_config):
    cfg = user_config
    if local_rank == 0:
        construct_print(cfg)
    init_cudnn(benchmark=(cfg["size_list"] is None), deterministic=False)
    torch.cuda.set_device(local_rank)
    if cfg["is_distributed"] and world_size > 1:
        init_process(args.ip, args.port, local_rank, world_size)
    batch_size_single_gpu = cfg["batch_size"] // ngpus_per_node                        # reference train.py:119

    if not cfg.get("synthetic", True):
        # the reference's training set (train.py:121-138): workers decode, the GPU resizes, augments and normalises one
        # batch ahead; a missing tr_data_path is an error naming it
        from distributed_sod_project_b200.data import make_train_loader
        from distributed_sod_project_b200.pipeline import TrainPrefetcher
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist.is_initialized() else (0, 1)
        source = make_train_loader(cfg["rgb_data"]["tr_data_path"], batch_size_single_gpu, world, rank, cfg["num_workers"],
                                   cfg["prefix"])
        loader = TrainPrefetcher(source, cfg["input_size"], size_list=cfg["size_list"], seed=0, rank=rank,
                                 joint_transforms=cfg.get("joint_transforms"))
    elif cfg.get("synthetic_uint8", True):
        # SURVEY §8f.2: uint8 batches from the (here: synthetic) workers, pinned → H2D and ToTensor / Normalize / multi-scale
        # collate as one GPU kernel, one batch ahead of the iteration (reference: BackgroundGenerator, train.py:285)
        from distributed_sod_project_b200.pipeline import DevicePrefetcher
        source = SyntheticU8Loader(batch_size_single_gpu, cfg.get("synthetic_iters_per_epoch", 20), cfg["input_size"], local_rank)
        loader = DevicePrefetcher(source, size_list=cfg["size_list"], seed=0)
        loader.set_epoch = lambda e, _l=loader, _s=source: (_s.set_epoch(e), _l.rng.seed(e))
    else:
        loader = SyntheticLoader(batch_size_single_gpu, cfg.get("synthetic_iters_per_epoch", 20), cfg["input_size"],
                                 cfg["size_list"], local_rank)
    total_iter_num = cfg["epoch_num"] * len(loader)

    dtype = _DTYPES[cfg.get("dtype", "bf16")] if cfg["use_amp"] else torch.float32
    trainer = Trainer(model_name=cfg["model"], lr=cfg["lr"], momentum=cfg["momentum"], weight_decay=cfg["weight_decay"],
                      nesterov=cfg["nesterov"], optim=cfg["optim"], reduction=cfg["reduction"], use_aux_loss=cfg["use_aux_loss"],
                      dtype=dtype, channels_last=cfg.get("channels_last", True), report_items=True,
                      # one captured graph per input size; learning rates are read from a device table, so multi-scale
                      # batches and a per-iteration schedule (`sche_usebatch`) replay graphs too
                      use_graph=cfg.get("cuda_graph", False))
    scheduler = trainer.scheduler(total_iter_num if cfg["sche_usebatch"] else cfg["epoch_num"], cfg["lr_type"], cfg["lr_decay"],
                                  cfg["warmup_epoch"])
    if local_rank == 0:
        construct_print(f"optimizer = {trainer.optimizer}")
        construct_print(f"scheduler = {scheduler}")

    def test(mode="test"):
        """reference train.py:338-369: every data set of `te_data_list` (mode "val": `val_data_path`) through the model;
        here every rank evaluates its shard and the metrics are reduced over the ranks (evaluate.py)"""
        names = cfg["rgb_data"]["val_data_path"] if mode == "val" else cfg["rgb_data"]["te_data_list"]
        total_results = {}
        if not cfg.get("synthetic_eval", True):
            # the reference's on-disk sets (train.py:346-376), every rank its shard, six metrics as the reference reports
            for data_name, data_path in names.items():
                loader, n_img = open_test_set(data_name, data_path, batch_size_single_gpu, cfg["num_workers"], cfg["prefix"])
                save_dir = os.path.join(path_config["save"], data_name) if cfg.get("save_pre", True) else None
                results = test_process(trainer.model, loader, length=n_img, wfm=cfg.get("wfm_impl", "gpu"),
                                       input_size=cfg["input_size"], save_dir=save_dir)
                msg = f"Results on the {mode}set({data_name}:'{data_path}', {n_img} images over {max(world_size, 1)} rank(s)):\n{results}"
                if local_rank == 0:
                    write_data_to_file(msg, path_config["te_log"])
                    construct_print(msg)
                total_results[data_name.upper()] = results
            return total_results
        for data_name in names:
            n_img = cfg.get("synthetic_eval_images", 32)
            mine = list(shard(n_img))
            batches = synth_eval_set(data_name, mine, batch_size_single_gpu, cfg["input_size"])
            results = test_process(trainer.model, batches, length=n_img)
            msg = f"Results on the {mode}set({data_name}: synthetic, {n_img} images over {max(world_size, 1)} rank(s)):\n{results}"
            if local_rank == 0:
                write_data_to_file(msg, path_config["te_log"])
                construct_print(msg)
            total_results[data_name.upper()] = results
        return total_results

    if cfg["resume_mode"] == "test":                                  # reference train.py:160-172: load the weights, evaluate, stop
        resume_checkpoint(model=trainer.model, load_path=path_config["final_full_net"], mode="onlynet", local_rank=local_rank)
        test(mode="test")
        if dist.is_initialized():
            dist.destroy_process_group()
        return

    start_epoch = 0
    if cfg["resume_mode"] == "train":
        # reference train.py:188-198 resumes on rank 0 only (SURVEY Q5: the other ranks keep their initial weights and the
        # first all-reduce mixes them); here every rank loads the same file
        start_epoch = resume_checkpoint(model=trainer.model, optimizer=trainer.optimizer, amp=amp if cfg["use_amp"] else None,
                                        exp_name=exp_name, load_path=path_config["final_full_net"], mode="all",
                                        local_rank=local_rank)

    for curr_epoch in range(start_epoch, cfg["epoch_num"]):
        loader.set_epoch(curr_epoch)
        if not cfg["sche_usebatch"]:
            scheduler.step(optimizer=trainer.optimizer, curr_epoch=curr_epoch)
        trainer.model.train()
        record = AvgMeter()
        loss_acc, seen = torch.zeros((), device="cuda"), 0      # Σ loss·n of this epoch accumulated on the device, Σ n on the host
        t0 = time.time()
        for batch_id, (inputs, masks, names) in enumerate(loader):
            curr_iter = curr_epoch * len(loader) + batch_id
            if cfg["sche_usebatch"]:
                scheduler.step(trainer.optimizer, curr_epoch=curr_iter)
            inputs = inputs.cuda(non_blocking=True)                                      # train.py:291-292 (no-ops on the
            masks = masks.cuda(non_blocking=True)                                        # pipeline path: already on the device)
            want_log = local_rank == 0 and cfg["print_freq"] > 0 and (curr_iter + 1) % cfg["print_freq"] == 0
            reduced, items, _ = trainer.forward_backward_update(inputs, masks, report=want_log)
            # reference train.py:311 updates the running average every iteration; here that costs no host sync
            loss_acc.add_(reduced.detach().reshape(()), alpha=float(inputs.size(0)))
            seen += inputs.size(0)
            if want_log:                                                                 # host sync only when printing
                loss_val = float(reduced.item())
                record.val, record.sum, record.count = loss_val, float(loss_acc.item()), seen
                record.avg = record.sum / max(seen, 1)
                trainer.check_errors()                                                   # device-side barrier / packet timeouts
                lr_str = ",".join(f"{g['lr']:.7f}" for g in trainer.optimizer.param_groups)
                log = (f"[I:{batch_id}/{len(loader)}/{curr_iter}/{total_iter_num}][E:{curr_epoch}:{cfg['epoch_num']}]>[{exp_name}]"
                       f"[Lr:{lr_str}][Avg:{record.avg:.5f}|Cur:{loss_val:.5f}|{items}]")
                print(log)
                write_data_to_file(log, path_config["tr_log"])
        torch.cuda.synchronize()
        trainer.check_errors()
        if local_rank == 0:
            n_img = len(loader) * batch_size_single_gpu * max(world_size, 1)
            construct_print(f"epoch {curr_epoch}: {time.time() - t0:.2f}s, {n_img / (time.time() - t0):.1f} img/s")
        if cfg["val_freq"] > 0 and (curr_epoch + 1) % cfg["val_freq"] == 0:      # train.py:254-255 (there: rank 0 only)
            test(mode="val")
        if (cfg["save_freq"] > 0 and (curr_epoch + 1) % cfg["save_freq"] == 0) or curr_epoch == cfg["epoch_num"] - 1:
            # every rank enters (the sharded momentum is gathered collectively), rank 0 writes, all leave through a barrier
            save_checkpoint(model=trainer.model, optimizer=trainer.optimizer, amp=amp if cfg["use_amp"] else None,
                            exp_name=exp_name, current_epoch=curr_epoch + 1, full_net_path=path_config["final_full_net"],
                            state_net_path=path_config["final_state_net"], write=local_rank == 0)   # utils/pipeline_ops.py:46-78
    if cfg.get("final_test", True):
        test(mode="test")                                                      # train.py:273-275
    construct_print("End Training...")
    trainer.check_errors()
    if dist.is_initialized():
        dist.destroy_process_group()


def main():
    args = parser.parse_args()
    assert torch.cuda.is_available(), "only on GPUs (reference train.py:63)"
    exp_name = construct_exp_name(user_config)
    path_config = construct_path_dict(proj_root=user_config["proj_root"], exp_name=exp_name, xlsx_name=user_config["xlsx_name"])
    check_mkdir(path_config["save"])
    check_mkdir(path_config["pth"])
    if user_config["is_distributed"]:
        construct_print("We will use the distributed training.")
        world_size = args.ngpus_per_node * args.nodes
        torch.multiprocessing.spawn(main_worker, nprocs=args.ngpus_per_node,
                                    args=(args.ngpus_per_node, world_size, args, exp_name, path_config))
    else:
        construct_print("We will not use the distributed training.")
        main_worker(0, 1, 1, args, exp_name, path_config)


if __name__ == "__main__":
    main()
