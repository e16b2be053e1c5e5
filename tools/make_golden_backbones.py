#!/usr/bin/env python
"""Generate the golden vectors of one backbone plugin by running the UNMODIFIED reference on CPU.

    SOD_REFERENCE=/path/to/Distributed-SOD-Project python tools/make_golden_backbones.py {vgg16|wsgn_res50|wsgn_resnext50|aim_res50}

Writes tests/golden/model_<backbone>_init.npz, the fp32 trajectories step_<backbone>_w1_s64 / _w1_s128 / _w2_s64 and
the float64 runs of their first two iterations (`_fp64`).  W=2 is the concatenated-batch construction of
tools/make_golden.py: GroupNorm is per sample, and the decoder's SyncBN over two ranks is BatchNorm over the
concatenated batch.  The float64 runs are what the fp32 vectors are rounding noise around: one SGD step amplifies the
reference's own fp32 rounding (to ~1e-2 on WS-GN ResNet-50's 64² loss and ~4e-2 on its 128² logits), so the trajectory
tests hold later iterations to twice that distance where it exceeds 1e-3 (tests/test_gpu_backbones.py).

The shims of tools/make_golden.py stand in for the missing packages.  Each installer below makes the reference build
the backbone; one backbone is built per run, because the installers patch `sys.modules` and the reference's `network`.
"""
from __future__ import annotations

import functools
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402


def _vgg_probe_params(model):
    """small fixed probes of the post-step parameters (the res50 probe keys do not exist in this model)"""
    sd = dict(model.named_parameters())
    keys = ["div_2.0.weight", "div_2.0.bias", "div_4.1.weight", "div_32.8.weight", "div_32.7.bias", "trans32.weight",
            "sim2.bnh_2.bias", "upconv1.basicconv.0.weight", "classifier.weight", "classifier.bias"]
    return {k: sd[k].detach().reshape(-1)[:64].numpy().copy() for k in keys}


def install_vgg_model():
    """The reference ships `Backbone_VGG16_in3` (backbone/origin/from_origin.py:18-25) but no TestModel on it, and its
    TestModel cannot take it by a one-import swap: the slices carry 64, 128, 256, 512 and 512 channels, and the first
    one is at full resolution.  So the model is composed here, from the reference's own `Backbone_VGG16_in3`, `SIM`,
    `BasicConv2d`, `upsample_add` and `cus_sample`, in the reference TestModel's construction order (backbone, trans32
    … trans2, sim32 … sim2, upconv32 … upconv2, upconv1, classifier) with trans32 … trans2 taking 512, 512, 256, 128,
    64 channels and the head `classifier(upconv1(d2))` (no ×2 up-sample).  It is registered as `network.vgg16` in the
    reference's `network` module, so `step_vectors` / `model_init_vectors` of tools/make_golden.py run it as they run
    `res50`.

    `load_state_dict_from_url` returns {}, so `vgg16_bn(pretrained=True)` keeps the init it was built with.
    `pretrained=True` also passes `init_weights=False`, so `VGG._initialize_weights` never runs: the convolutions keep
    torch's default init (kaiming-uniform weights, uniform non-zero biases).

    The reference's own fp32 distance from its float64 run, |loss| and max |logits| difference (the trajectory tests
    derive their iteration-1 allowance from it):

        vector      iteration 0: loss, logits       iteration 1: loss, logits
        w1_s64      4.4e-08, 6.8e-05                3.3e-04, —
        w1_s128     1.8e-07, 1.0e-04                5.3e-05, 1.8e-02
        w2_s64      1.8e-07, 9.1e-05 (worst rank)   5.9e-05, — (worst rank)

    Iteration 0 sits far inside 1e-3.  One SGD step amplifies fp32 rounding to 3.3e-4 on the 64² loss (2.3e-4
    relative) and 1.8e-2 on the 128² logits (0.8 % of their largest magnitude, 2.33)."""
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
    mg._probe_params = _vgg_probe_params
    return "vgg16"


def install_wsgn_backbone():
    """The reference's TestModel takes its backbone from `backbone.origin.from_origin` (network/TestModel.py:11); a
    user switches to the weight-standardised GroupNorm ResNet-50 by importing `backbone.wsgn.from_wsgn.
    Backbone_ResNet50_in3` instead.  Here that one-import swap is a `sys.modules` entry: `backbone.origin.from_origin`
    is the `from_wsgn` module, so the reference's `res50` is built on the WS-GN backbone.  The release download
    (`model_zoo.load_url` in backbone/wsgn/customized_func.py:32-43) returns a one-entry `module.`-prefixed dict whose
    only key the reference's filter drops, so the seeded random init is kept (an empty dict would fail on its
    `keys()[0]`)."""
    mg.install_reference()
    import torch.utils.model_zoo as mz
    mz.load_url = lambda *a, **k: {"module.__no_such_parameter__": torch.zeros(1)}
    import backbone.wsgn.from_wsgn as from_wsgn
    sys.modules["backbone.origin.from_origin"] = from_wsgn
    return "res50"


def install_wsgn_resnext_backbone():
    """The WS-GN backbone swap, with `Backbone_ResNeXt50_in3` in place of `Backbone_ResNet50_in3`.  The reference's
    builder calls `l_resnext50(pretrained=True)` without the `baseWidth` / `cardinality` its signature requires (a
    TypeError); the release it loads (X-50-GN-WS.pth.tar) is ResNeXt-50 32×4d, so `from_wsgn`'s `l_resnext50` name is
    pointed at `functools.partial(l_resnext50, baseWidth=4, cardinality=32)`."""
    install_wsgn_backbone()
    import backbone.wsgn.from_wsgn as from_wsgn
    from_wsgn.l_resnext50 = functools.partial(from_wsgn.l_resnext50, baseWidth=4, cardinality=32)
    from_wsgn.Backbone_ResNet50_in3 = from_wsgn.Backbone_ResNeXt50_in3
    return "res50"


def _aim_probe_params(model):
    """small fixed probes of the post-step parameters (`trans32` does not exist in this model)"""
    sd = dict(model.named_parameters())
    keys = ["div_2.0.weight", "div_4.1.0.conv1.weight", "div_32.2.bn3.weight", "div_32.2.conv3.weight",
            "trans.conv0.h2h_0.weight", "trans.conv2.bnm_1.bias", "trans.conv4.identity.bias", "sim2.bnh_2.bias",
            "upconv1.basicconv.0.weight", "classifier.weight", "classifier.bias"]
    return {k: sd[k].detach().reshape(-1)[:64].numpy().copy() for k in keys}


def install_aim_model():
    """The reference ships MINet's `LightAIM` neck (module/MyLightModule.py:216-236) but no network on it.  MINet_Res50
    puts it between the ResNet-50 and the SIM decoder, so the model is composed here, from the reference's own
    `Backbone_ResNet50_in3`, `LightAIM`, `SIM`, `BasicConv2d`, `upsample_add` and `cus_sample`, in the order backbone,
    trans (= LightAIM((64, 256, 512, 1024, 2048), (64,) * 5)), sim32 … sim2, upconv32 … upconv2, upconv1, classifier;
    forward is the reference `res50`'s with `trans(...)` giving the five laterals.  It is registered as
    `network.aim_res50`.  The neck keeps torch's default conv and BN init, as the reference's module does.

    The reference's own fp32 distance from its float64 run, |loss| and max |logits| difference:

        vector      iteration 0: loss, logits       iteration 1: loss, logits
        w1_s64      9.8e-07, 9.5e-04                2.2e-04, —
        w1_s128     1.4e-07, 2.9e-04                1.8e-05, 1.2e-01
        w2_s64      9.7e-07, 2.1e-04 (worst rank)   5.6e-04, — (worst rank)

    The 64² iteration-0 logits are already 6.7e-4 of their largest magnitude (1.42) from the float64 run, so the
    trajectory test allows the reference's noise from iteration 0 on.  One SGD step amplifies the 128² logits' fp32
    rounding to 1.2e-1 (7 % of their largest magnitude, 1.63): the neck's 91 M parameters take the same step size."""
    mg.install_reference()
    import network
    from backbone.origin.from_origin import Backbone_ResNet50_in3
    from module.BaseBlocks import BasicConv2d
    from module.MyLightModule import SIM, LightAIM
    from utils.tensor_ops import cus_sample, upsample_add

    class aim_res50(nn.Module):
        def __init__(self):
            super().__init__()
            self.upsample_add = upsample_add
            self.upsample = cus_sample
            self.div_2, self.div_4, self.div_8, self.div_16, self.div_32 = Backbone_ResNet50_in3()
            self.trans = LightAIM(iC_list=(64, 256, 512, 1024, 2048), oC_list=(64, 64, 64, 64, 64))
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
            in_data_2, in_data_4, in_data_8, in_data_16, in_data_32 = self.trans(
                in_data_2, in_data_4, in_data_8, in_data_16, in_data_32)
            out_data_32 = self.upconv32(self.sim32(in_data_32) + in_data_32)
            out_data_16 = self.upsample_add(out_data_32, in_data_16)
            out_data_16 = self.upconv16(self.sim16(out_data_16) + out_data_16)
            out_data_8 = self.upsample_add(out_data_16, in_data_8)
            out_data_8 = self.upconv8(self.sim8(out_data_8) + out_data_8)
            out_data_4 = self.upsample_add(out_data_8, in_data_4)
            out_data_4 = self.upconv4(self.sim4(out_data_4) + out_data_4)
            out_data_2 = self.upsample_add(out_data_4, in_data_2)
            out_data_2 = self.upconv2(self.sim2(out_data_2) + out_data_2)
            return self.classifier(self.upconv1(self.upsample(out_data_2, scale_factor=2)))

    network.aim_res50 = aim_res50
    mg._probe_params = _aim_probe_params
    return "aim_res50"


INSTALLERS = {"vgg16": install_vgg_model, "wsgn_res50": install_wsgn_backbone,
              "wsgn_resnext50": install_wsgn_resnext_backbone, "aim_res50": install_aim_model}


def main():
    if len(sys.argv) != 2 or sys.argv[1] not in INSTALLERS:
        raise SystemExit(f"usage: {sys.argv[0]} {{{'|'.join(INSTALLERS)}}}")
    tag = sys.argv[1]
    os.makedirs(mg.OUT, exist_ok=True)
    model = INSTALLERS[tag]()                       # the reference `network` name the backbone is built under
    torch.set_num_threads(8)
    mg.model_init_vectors(model, tag=tag)
    mg.step_vectors(model, 1, 2, 64, 3, f"{tag}_w1_s64", keep_logits=(0,))
    mg.step_vectors(model, 1, 4, 128, 3, f"{tag}_w1_s128", keep_logits=(0, 1))
    mg.step_vectors(model, 2, 2, 64, 3, f"{tag}_w2_s64", keep_logits=(0,))
    mg.step_vectors(model, 1, 2, 64, 2, f"{tag}_w1_s64_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors(model, 1, 4, 128, 2, f"{tag}_w1_s128_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors(model, 2, 2, 64, 2, f"{tag}_w2_s64_fp64", keep_logits=(0,), dtype=torch.float64)


if __name__ == "__main__":
    main()
