#!/usr/bin/env python
"""Generate the golden vectors of `vgg16` by running the UNMODIFIED reference on CPU.

    SOD_REFERENCE=/path/to/Distributed-SOD-Project python tools/make_golden_vgg.py

The reference ships `Backbone_VGG16_in3` (backbone/origin/from_origin.py:18-25) but no TestModel on it, and its
TestModel cannot take it by a one-import swap: the slices carry 64, 128, 256, 512 and 512 channels, and the first one
is at full resolution.  So the model is composed here, from the reference's own `Backbone_VGG16_in3`, `SIM`,
`BasicConv2d`, `upsample_add` and `cus_sample`, in the reference TestModel's construction order (backbone, trans32 …
trans2, sim32 … sim2, upconv32 … upconv2, upconv1, classifier) with trans32 … trans2 taking 512, 512, 256, 128, 64
channels and the head `classifier(upconv1(d2))` (no ×2 up-sample).  It is registered as `network.vgg16` in the
reference's `network` module, so `step_vectors` / `model_init_vectors` of tools/make_golden.py run it as they run `res50`.

The shims of tools/make_golden.py stand in for the missing packages; `load_state_dict_from_url` returns {}, so
`vgg16_bn(pretrained=True)` keeps the init it was built with.  `pretrained=True` also passes `init_weights=False`, so
`VGG._initialize_weights` never runs: the convolutions keep torch's default init (kaiming-uniform weights, uniform
non-zero biases).

Writes tests/golden/model_vgg16_init.npz, the fp32 trajectories step_vgg16_w1_s64 / _w1_s128 / _w2_s64 and the float64
runs of their first two iterations (`_fp64`) (W=2 by the concatenated-batch construction of tools/make_golden.py).

The reference's own fp32 distance from its float64 run, |loss| and max |logits| difference (the trajectory tests
derive their iteration-1 allowance from it):

    vector      iteration 0: loss, logits       iteration 1: loss, logits
    w1_s64      4.4e-08, 6.8e-05                3.3e-04, —
    w1_s128     1.8e-07, 1.0e-04                5.3e-05, 1.8e-02
    w2_s64      1.8e-07, 9.1e-05 (worst rank)   5.9e-05, — (worst rank)

Iteration 0 sits far inside 1e-3.  One SGD step amplifies fp32 rounding to 3.3e-4 on the 64² loss (2.3e-4 relative) and
1.8e-2 on the 128² logits (0.8 % of their largest magnitude, 2.33).
"""
from __future__ import annotations

import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402


def _probe_params(model):
    """small fixed probes of the post-step parameters (the res50 probe keys do not exist in this model)"""
    sd = dict(model.named_parameters())
    keys = ["div_2.0.weight", "div_2.0.bias", "div_4.1.weight", "div_32.8.weight", "div_32.7.bias", "trans32.weight",
            "sim2.bnh_2.bias", "upconv1.basicconv.0.weight", "classifier.weight", "classifier.bias"]
    return {k: sd[k].detach().reshape(-1)[:64].numpy().copy() for k in keys}


def install_vgg_model():
    mg.install_reference()
    import network
    from backbone.origin.from_origin import Backbone_VGG16_in3
    from module.BaseBlocks import BasicConv2d
    from module.MyLightModule import SIM
    from utils.tensor_ops import cus_sample, upsample_add

    class vgg16(nn.Module):
        def __init__(self):
            super().__init__()
            self.upsample_add = upsample_add
            self.upsample = cus_sample
            self.div_2, self.div_4, self.div_8, self.div_16, self.div_32 = Backbone_VGG16_in3()
            self.trans32 = nn.Conv2d(512, 64, 1, 1)
            self.trans16 = nn.Conv2d(512, 64, 1, 1)
            self.trans8 = nn.Conv2d(256, 64, 1, 1)
            self.trans4 = nn.Conv2d(128, 64, 1, 1)
            self.trans2 = nn.Conv2d(64, 64, 1, 1)
            self.sim32 = SIM(64, 32)
            self.sim16 = SIM(64, 32)
            self.sim8 = SIM(64, 32)
            self.sim4 = SIM(64, 32)
            self.sim2 = SIM(64, 32)
            self.upconv32 = BasicConv2d(64, 64, kernel_size=3, stride=1, padding=1)
            self.upconv16 = BasicConv2d(64, 64, kernel_size=3, stride=1, padding=1)
            self.upconv8 = BasicConv2d(64, 64, kernel_size=3, stride=1, padding=1)
            self.upconv4 = BasicConv2d(64, 64, kernel_size=3, stride=1, padding=1)
            self.upconv2 = BasicConv2d(64, 32, kernel_size=3, stride=1, padding=1)
            self.upconv1 = BasicConv2d(32, 32, kernel_size=3, stride=1, padding=1)
            self.classifier = nn.Conv2d(32, 1, 1)

        def forward(self, in_data):
            in_data_2 = self.div_2(in_data)
            in_data_4 = self.div_4(in_data_2)
            in_data_8 = self.div_8(in_data_4)
            in_data_16 = self.div_16(in_data_8)
            in_data_32 = self.div_32(in_data_16)
            in_data_32 = self.trans32(in_data_32)
            in_data_16 = self.trans16(in_data_16)
            in_data_8 = self.trans8(in_data_8)
            in_data_4 = self.trans4(in_data_4)
            in_data_2 = self.trans2(in_data_2)
            out_data_32 = self.upconv32(self.sim32(in_data_32) + in_data_32)
            out_data_16 = self.upsample_add(out_data_32, in_data_16)
            out_data_16 = self.upconv16(self.sim16(out_data_16) + out_data_16)
            out_data_8 = self.upsample_add(out_data_16, in_data_8)
            out_data_8 = self.upconv8(self.sim8(out_data_8) + out_data_8)
            out_data_4 = self.upsample_add(out_data_8, in_data_4)
            out_data_4 = self.upconv4(self.sim4(out_data_4) + out_data_4)
            out_data_2 = self.upsample_add(out_data_4, in_data_2)
            out_data_2 = self.upconv2(self.sim2(out_data_2) + out_data_2)
            return self.classifier(self.upconv1(out_data_2))

    network.vgg16 = vgg16
    mg._probe_params = _probe_params


def main():
    os.makedirs(mg.OUT, exist_ok=True)
    install_vgg_model()
    torch.set_num_threads(8)
    mg.model_init_vectors("vgg16")
    mg.step_vectors("vgg16", 1, 2, 64, 3, "vgg16_w1_s64", keep_logits=(0,))
    mg.step_vectors("vgg16", 1, 4, 128, 3, "vgg16_w1_s128", keep_logits=(0, 1))
    mg.step_vectors("vgg16", 2, 2, 64, 3, "vgg16_w2_s64", keep_logits=(0,))
    mg.step_vectors("vgg16", 1, 2, 64, 2, "vgg16_w1_s64_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors("vgg16", 1, 4, 128, 2, "vgg16_w1_s128_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors("vgg16", 2, 2, 64, 2, "vgg16_w2_s64_fp64", keep_logits=(0,), dtype=torch.float64)


if __name__ == "__main__":
    main()
