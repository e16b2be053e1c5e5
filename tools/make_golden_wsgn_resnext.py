#!/usr/bin/env python
"""Generate the golden vectors of `wsgn_resnext50` by running the UNMODIFIED reference on CPU.

    SOD_REFERENCE=/path/to/Distributed-SOD-Project python tools/make_golden_wsgn_resnext.py

The WS-GN backbone swap of tools/make_golden_wsgn.py, with `Backbone_ResNeXt50_in3` in place of
`Backbone_ResNet50_in3`.  The reference's builder calls `l_resnext50(pretrained=True)` without the `baseWidth` /
`cardinality` its signature requires (a TypeError); the release it loads (X-50-GN-WS.pth.tar) is ResNeXt-50 32×4d, so
`from_wsgn`'s `l_resnext50` name is pointed at `functools.partial(l_resnext50, baseWidth=4, cardinality=32)`.

Writes tests/golden/model_wsgn_resnext50_init.npz, the fp32 trajectories step_wsgn_resnext50_w1_s64 / _w1_s128 /
_w2_s64 and the float64 runs of their first two iterations (`_fp64`).
"""
from __future__ import annotations

import functools
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
import make_golden_wsgn as mgw  # noqa: E402


def install_wsgn_resnext_backbone():
    mgw.install_wsgn_backbone()
    import backbone.wsgn.from_wsgn as from_wsgn
    from_wsgn.l_resnext50 = functools.partial(from_wsgn.l_resnext50, baseWidth=4, cardinality=32)
    from_wsgn.Backbone_ResNet50_in3 = from_wsgn.Backbone_ResNeXt50_in3


def main():
    os.makedirs(mg.OUT, exist_ok=True)
    install_wsgn_resnext_backbone()
    torch.set_num_threads(8)
    tag = "wsgn_resnext50"
    mg.model_init_vectors("res50", tag=tag)
    mg.step_vectors("res50", 1, 2, 64, 3, f"{tag}_w1_s64", keep_logits=(0,))
    mg.step_vectors("res50", 1, 4, 128, 3, f"{tag}_w1_s128", keep_logits=(0, 1))
    mg.step_vectors("res50", 2, 2, 64, 3, f"{tag}_w2_s64", keep_logits=(0,))
    mg.step_vectors("res50", 1, 2, 64, 2, f"{tag}_w1_s64_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors("res50", 1, 4, 128, 2, f"{tag}_w1_s128_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors("res50", 2, 2, 64, 2, f"{tag}_w2_s64_fp64", keep_logits=(0,), dtype=torch.float64)


if __name__ == "__main__":
    main()
