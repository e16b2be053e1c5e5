#!/usr/bin/env python
"""Generate the golden vectors of `wsgn_res50` by running the UNMODIFIED reference on CPU.

    SOD_REFERENCE=/path/to/Distributed-SOD-Project python tools/make_golden_wsgn.py

The reference's TestModel takes its backbone from `backbone.origin.from_origin` (network/TestModel.py:11); a user
switches to the weight-standardised GroupNorm ResNet-50 by importing `backbone.wsgn.from_wsgn.Backbone_ResNet50_in3`
instead.  Here that one-import swap is a `sys.modules` entry: `backbone.origin.from_origin` is the `from_wsgn` module,
so the reference's `res50` / `cp_res50` are built on the WS-GN backbone.  The shims of tools/make_golden.py stand in for
the missing packages; the release download (`model_zoo.load_url` in backbone/wsgn/customized_func.py:32-43) returns a
one-entry `module.`-prefixed dict whose only key the reference's filter drops, so the seeded random init is kept
(an empty dict would fail on its `keys()[0]`).

Writes tests/golden/model_wsgn_res50_init.npz, the fp32 trajectories step_wsgn_res50_w1_s64 / _w1_s128 /
_w2_s64 and the float64 runs of the first two iterations of each (`_fp64`) (W=2 by the concatenated-batch construction of tools/make_golden.py: GroupNorm is per sample, and the
decoder's SyncBN over two ranks is BatchNorm over the concatenated batch).
"""
from __future__ import annotations

import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402


def install_wsgn_backbone():
    mg.install_reference()
    import torch.utils.model_zoo as mz
    mz.load_url = lambda *a, **k: {"module.__no_such_parameter__": torch.zeros(1)}
    import backbone.wsgn.from_wsgn as from_wsgn
    sys.modules["backbone.origin.from_origin"] = from_wsgn


def main():
    os.makedirs(mg.OUT, exist_ok=True)
    install_wsgn_backbone()
    torch.set_num_threads(8)
    mg.model_init_vectors("res50", tag="wsgn_res50")
    mg.step_vectors("res50", 1, 2, 64, 3, "wsgn_res50_w1_s64", keep_logits=(0,))
    mg.step_vectors("res50", 1, 4, 128, 3, "wsgn_res50_w1_s128", keep_logits=(0, 1))
    mg.step_vectors("res50", 2, 2, 64, 3, "wsgn_res50_w2_s64", keep_logits=(0,))
    # the same two W=1 runs in float64: what the fp32 vectors are rounding noise around.  One SGD step of this model
    # already amplifies fp32 rounding to ~1e-2 on the 64² loss and ~4e-2 on the 128² logits, so iteration 1 is held to
    # that noise level (tests/test_gpu_wsgn_model.py)
    mg.step_vectors("res50", 1, 2, 64, 2, "wsgn_res50_w1_s64_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors("res50", 1, 4, 128, 2, "wsgn_res50_w1_s128_fp64", keep_logits=(0, 1), dtype=torch.float64)
    mg.step_vectors("res50", 2, 2, 64, 2, "wsgn_res50_w2_s64_fp64", keep_logits=(0,), dtype=torch.float64)


if __name__ == "__main__":
    main()
