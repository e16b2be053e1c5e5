"""Experiment configuration — same keys and semantics as the reference's `config.py:25-76`.

Two DEFAULTS differ from the reference on purpose: `use_amp` is True (the reference ships False; bf16 autocast is the benchmark
configuration) and `resume_mode` is "" (the reference ships "test", which evaluates an existing checkpoint and
exits — a fresh checkout has none).  Every other default is the reference's.

Extra keys (all optional, defaults reproduce the benchmark configuration):
  dtype           "bf16" | "fp16" | "fp32": autocast dtype used when `use_amp` is True
  channels_last   run the network in NHWC (what cuDNN's tensor-core kernels and the SyncBN kernels want)
  synthetic       train on synthetic batches of the dataloader's output contract; False: train on
                  `rgb_data.tr_data_path` with the reference's resize and augmentation run on the GPU (train.py)
  joint_transforms  with `synthetic` False: the reference's joint transforms (utils/joint_transforms.py) to train with,
                  a list of [name, *args] entries in application order, with the reference's constructor arguments:
                  ["JointResize", size], ["ScaleCenterCrop", input_size], ["PaddingSquare", pad_size],
                  ["RandomScaleCrop", input_size, scale_factor], ["RandomHorizontallyFlip"], ["RandomRotate", degree],
                  ["RandomGaussianBlur"].  Accepted order: exactly one size step first (JointResize, ScaleCenterCrop
                  or PaddingSquare), then optionally RandomScaleCrop (its input_size is the size step's side), then
                  RandomHorizontallyFlip, RandomRotate and RandomGaussianBlur, each optional, in that order; the chain
                  must make `input_size`² samples.  Anything else is a ValueError naming the entry.  ColorJitter(0.1,
                  0.1, 0.1) always follows.  Absent or None: the reference's [["JointResize", input_size],
                  ["RandomHorizontallyFlip"], ["RandomRotate", 10]].  Evaluation is not affected.
  cuda_graph      capture one iteration per (shape, lr) and replay it: one launch instead of ~700 kernel launches
  synthetic_eval  evaluate on synthetic sets of `synthetic_eval_images` images named after the configured sets; False:
                  read `te_data_list` / `val_data_path` from disk (a missing path is an error naming the set) and report
                  all six metrics, with the reference's Pillow resizes reproduced bit for bit on the GPU.
                  `save_pre` then writes each rank's predictions under
                  `<output>/<exp>/pre/<set>/`.
  wfm_impl        where the on-disk evaluation computes the weighted F-measure: "gpu" (scipy's distance transform, tie
                  rule included, and the weighting as CUDA kernels) or "host" (scipy itself on each rank's images).  Both
                  compute the same metric and agree to 1e-10 per image; "gpu" keeps evaluation about as fast as without it.
"""
import os
from collections import OrderedDict

__all__ = ["user_config"]

proj_root = os.path.dirname(os.path.abspath(__file__))
datasets_root = os.environ.get("SOD_DATASETS_ROOT", "/home/lart/Datasets/")

_rgb = os.path.join(datasets_root, "Saliency/RGBSOD")
ecssd_path = os.path.join(_rgb, "ECSSD")
dutomron_path = os.path.join(_rgb, "DUT-OMRON")
hkuis_path = os.path.join(_rgb, "HKU-IS")
pascals_path = os.path.join(_rgb, "PASCAL-S")
soc_path = os.path.join(_rgb, "SOC/Test")
dutstr_path = os.path.join(_rgb, "DUTS/Train")
dutste_path = os.path.join(_rgb, "DUTS/Test")

user_config = {
    "model": "cp_res50",
    "resume_mode": "",            # ['train', 'test', '']
    "version": "0.2",
    "use_aux_loss": True,
    "save_pre": True,
    "epoch_num": 30,
    "lr": 0.05,
    "xlsx_name": "result_full.xlsx",
    "output_name": "output",
    "is_distributed": True,
    "use_amp": True,
    "rgb_data": {
        "tr_data_path": dutstr_path,
        "val_data_path": {"pascal-s": pascals_path},
        "te_data_list": OrderedDict({"pascal-s": pascals_path, "ecssd": ecssd_path, "dut-omron": dutomron_path,
                                     "hku-is": hkuis_path, "duts": dutste_path, "soc": soc_path}),
    },
    "record_freq": 100,
    "print_freq": 10,
    "val_freq": 5,
    "save_freq": 5,
    "prefix": (".jpg", ".png"),
    "size_list": None,            # e.g. [256, 320, 384] for multi-scale training
    "reduction": "mean",
    "optim": "f3_trick",
    "weight_decay": 5e-4,
    "momentum": 0.9,
    "nesterov": False,
    "sche_usebatch": False,
    "lr_type": "poly",
    "warmup_epoch": 1,
    "lr_decay": 0.9,
    "batch_size": 48,
    "num_workers": 4,
    "input_size": 320,
    "proj_root": proj_root,
    # --- engine extras ---
    "dtype": "bf16",
    "channels_last": True,
    "synthetic": True,
    "synthetic_iters_per_epoch": 20,
    "synthetic_uint8": True,      # synthetic batches as 8-bit images + GPU pre-processing kernel (pipeline.py); False: fp32 tensors from the host
    "cuda_graph": True,           # replay each iteration as one CUDA graph (one graph per input size; lr read from a device table)
    "synthetic_eval": True,       # evaluate on synthetic sets; False: the on-disk te_data_list / val_data_path sets
    "synthetic_eval_images": 32,  # images per synthetic evaluation set (te_data_list / val_data_path names are kept as labels)
    "wfm_impl": "gpu",            # on-disk evaluation's weighted F-measure: "gpu" kernels or "host" scipy; same metric, within 1e-10 per image
    "final_test": True,           # evaluate every test set after training, as reference train.py:273-275
}

# test hook: SOD_CONFIG_JSON='{"epoch_num": 1, ...}' overrides keys without editing this file
if os.environ.get("SOD_CONFIG_JSON"):
    import json as _json
    user_config.update(_json.loads(os.environ["SOD_CONFIG_JSON"]))
