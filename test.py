#!/usr/bin/env python
"""Evaluation entry point with the reference's surface (`python test.py`, reference test.py:38-48): build
`user_config["model"]`, load the weights of the final checkpoint (`resume_checkpoint(..., mode="onlynet")`), evaluate
every set of `te_data_list`.  One process evaluates everything, or — launched with `torchrun --nproc-per-node N test.py` —
every rank evaluates its shard and the metrics are reduced over the ranks (the reference's author lists multi-GPU
evaluation as an open issue, readme.md:67-69).  Metrics run on the GPU (distributed_sod_project_b200/metrics.py).

Data sets are synthetic by default (`synthetic_eval_images` images per configured set name); with
`"synthetic_eval": False` the `te_data_list` sets are read from disk (distributed_sod_project_b200/data.py) and all six of
the reference's metrics are reported, predictions resized to each ground truth's size exactly as Pillow does.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

from config import user_config
from distributed_sod_project_b200 import network
from distributed_sod_project_b200.checkpoint import resume_checkpoint
from distributed_sod_project_b200.data import open_test_set
from distributed_sod_project_b200.evaluate import shard, test_process
from distributed_sod_project_b200.syncbn import convert_syncbn_model
from distributed_sod_project_b200.synthetic import synth_eval_set
from distributed_sod_project_b200.utils import check_mkdir, construct_exp_name, construct_path_dict, construct_print, write_data_to_file

TEST_SETTING = dict(save_results=False, batch_size=24)       # reference test.py:30


def main():
    assert torch.cuda.is_available(), "only on GPUs (reference test.py:28)"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    exp_name = construct_exp_name(user_config)
    path_config = construct_path_dict(proj_root=user_config["proj_root"], exp_name=exp_name, xlsx_name=user_config["xlsx_name"])
    check_mkdir(path_config["save"])
    construct_print(f"We will test the model on {world} GPU(s).")
    model = getattr(network, user_config["model"])().cuda().to(memory_format=torch.channels_last)      # reference test.py:40
    model = convert_syncbn_model(model)                        # eval-mode BatchNorm through the same kernels as training
    resume_checkpoint(model=model, load_path=path_config["final_full_net"], mode="onlynet", local_rank=local)
    total_results = {}
    if not user_config.get("synthetic_eval", True):
        # the on-disk sets (reference test.py:51-75 with utils/dataset.py:72-122), six metrics per set
        for data_name, data_path in user_config["rgb_data"]["te_data_list"].items():
            loader, n_img = open_test_set(data_name, data_path, TEST_SETTING["batch_size"], user_config["num_workers"],
                                          user_config["prefix"])
            save_dir = os.path.join(path_config["save"], data_name) if user_config.get("save_pre", True) else None
            results = test_process(model, loader, length=n_img, wfm=user_config.get("wfm_impl", "gpu"),
                                   input_size=user_config["input_size"], save_dir=save_dir)
            msg = f"Results on the testset({data_name}:'{data_path}', {n_img} images over {world} rank(s)):\n{results}"
            if local == 0:
                write_data_to_file(msg, path_config["te_log"])
                construct_print(msg)
            total_results[data_name.upper()] = results
        if world > 1:
            dist.destroy_process_group()
        return total_results
    for data_name in user_config["rgb_data"]["te_data_list"]:  # reference test.py:51-75
        n_img = user_config.get("synthetic_eval_images", 32)
        batches = synth_eval_set(data_name, list(shard(n_img)), TEST_SETTING["batch_size"], user_config["input_size"])
        results = test_process(model, batches, length=n_img)
        msg = f"Results on the testset({data_name}: synthetic, {n_img} images over {world} rank(s)):\n{results}"
        if local == 0:
            write_data_to_file(msg, path_config["te_log"])
            construct_print(msg)
        total_results[data_name.upper()] = results
    if world > 1:
        dist.destroy_process_group()
    return total_results


if __name__ == "__main__":
    main()
