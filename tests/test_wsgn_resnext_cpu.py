"""CPU checks of the ResNeXt WS-GN plugins (`wsgn_resnext50`, `cp_wsgn_resnext50`): bit-identity with the reference's
weight-standardised GroupNorm ResNeXt-50 32×4d TestModel, names, counts and optimizer groups, the release's pretrained
file format, the grouped convolutions' exclusion from the 16-bit shadow and gradient ranges, the launch-geometry model
of csrc/gconv.cu and its C ABI."""
from __future__ import annotations

import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import gconv_geometry as geo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(name="wsgn_resnext50"):
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return getattr(network, name)()


@pytest.mark.parametrize("name", ["wsgn_resnext50", "cp_wsgn_resnext50"])
def test_plugin_is_bit_identical_to_reference(golden, name):
    """init_seed(0) + the plugin against the reference TestModel on `Backbone_ResNeXt50_in3`
    (tests/golden/model_wsgn_resnext50_init.npz, tools/make_golden_wsgn_resnext.py): keys, shapes, values at fixed
    positions, per-tensor sums and one training-mode forward at 8 threads"""
    g = golden("model_wsgn_resnext50_init.npz")
    m = _model(name)
    sd = m.state_dict()
    assert "\n".join(sd) == str(g["keys"])
    for i, v in enumerate(sd.values()):
        assert list(v.shape) == [d for d in g["shapes"][i] if d >= 0]
        a = v.detach().reshape(-1).double()
        idx = torch.from_numpy(np.linspace(0, a.numel() - 1, g["values"].shape[1]).astype(np.int64))
        np.testing.assert_array_equal(a[idx].numpy(), g["values"][i])
        np.testing.assert_allclose([a.sum().item(), (a * a).sum().item()], g["moments"][i], rtol=1e-12, atol=0)
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    try:
        y = m(torch.from_numpy(g["x"])).detach().numpy()
    finally:
        torch.set_num_threads(threads)
    np.testing.assert_array_equal(y, g["y"])


def test_names_counts_and_f3_trick_groups():
    from distributed_sod_project_b200.network.blocks import WSConv2d
    from distributed_sod_project_b200.optim import is_plain_conv, make_optimizer
    m = _model()
    assert sum(isinstance(x, nn.GroupNorm) for x in m.modules()) == 53
    assert sum(isinstance(x, WSConv2d) for x in m.modules()) == 53
    grouped = [(n, x) for n, x in m.named_modules() if isinstance(x, WSConv2d) and x.groups > 1]
    assert len(grouped) == 16 and all(n.endswith(".conv2") and x.groups == 32 for n, x in grouped)
    assert sorted({x.in_channels // 32 for _, x in grouped}) == [4, 8, 16, 32]
    assert not any(is_plain_conv(x) for _, x in grouped)
    assert sum(p.numel() for n, p in m.named_parameters() if n.startswith("div")) == 22_979_904
    names = [n for n, _ in m.named_parameters()]
    assert "div_4.1.0.downsample.0.weight" in names and "div_32.2.conv3.weight" in names
    assert tuple(m.state_dict()["div_8.0.conv2.weight"].shape) == (256, 8, 3, 3)
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    groups = [[n for n, p in m.named_parameters() if any(p is q for q in g["params"])] for g in opt.param_groups]
    assert all(n.startswith("div") and not n.startswith("div_2") for n in groups[0])
    assert all(not n.startswith("div") for n in groups[1])
    assert set(names) - set(groups[0]) - set(groups[1]) == {"div_2.0.weight", "div_2.1.weight", "div_2.1.bias"}
    f = opt.flat
    ids = {id(x.weight) for _, x in grouped}
    for p, off in f.slots:
        if id(p) in ids:
            bucket = next(i for i, (b, e) in enumerate(f.ranges) if b <= off < e)
            assert off >= f.splits[bucket], "a grouped WS weight sits in the 16-bit gradient range"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=str)
def test_grouped_convolutions_get_no_shadow(dtype):
    from distributed_sod_project_b200 import amp
    from distributed_sod_project_b200.optim import make_optimizer
    m = _model()
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    opt.flat.enable_shadow(dtype)
    amp._install_shadow_weights(m, opt.flat)
    assert not any(hasattr(x, "_sod_w16") for x in m.modules() if isinstance(x, nn.Conv2d) and x.groups > 1)
    assert any(hasattr(x, "_sod_w16") for x in m.modules())


def test_res50_builds_as_before(golden):
    """the generalised Bottleneck keeps res50 and wsgn_res50 (names and random draws) unchanged"""
    for name, vec in (("res50", "model_res50_init.npz"), ("wsgn_res50", "model_wsgn_res50_init.npz")):
        g = golden(vec)
        sd = _model(name).state_dict()
        assert "\n".join(sd) == str(g["keys"])
        for i, v in enumerate(sd.values()):
            np.testing.assert_allclose([v.double().sum().item()], [g["moments"][i][0]], rtol=1e-12, atol=0)


def test_load_pretrained_backbone_reads_the_resnext_release_format(tmp_path):
    """X-50-GN-WS.pth.tar's layout: tensors under "state_dict", `module.` prefix, the ResNeXt names (the grouped
    `conv2` weights are [D·C, D, 3, 3])"""
    from distributed_sod_project_b200.network import load_pretrained_backbone
    m = _model()
    sd = m.state_dict()
    g = torch.Generator().manual_seed(5)
    src = {"module.conv1.weight": torch.randn(sd["div_2.0.weight"].shape, generator=g),
           "module.layer2.0.conv2.weight": torch.randn(256, 8, 3, 3, generator=g),
           "module.layer4.0.downsample.1.bias": torch.rand(2048, generator=g),
           "module.layer1.0.conv2.weight": torch.randn(128, 128, 3, 3),           # a dense 3x3: ignored
           "module.fc.weight": torch.zeros(1000, 2048)}
    path = tmp_path / "X-50-GN-WS.pth.tar"
    torch.save({"epoch": 100, "arch": "l_resnext50", "state_dict": src}, path)
    loaded = load_pretrained_backbone(m, str(path))
    assert loaded == sorted(["div_2.0.weight", "div_8.0.conv2.weight", "div_32.0.downsample.1.bias"])
    now = m.state_dict()
    torch.testing.assert_close(now["div_8.0.conv2.weight"], src["module.layer2.0.conv2.weight"], rtol=0, atol=0)
    torch.testing.assert_close(now["div_4.1.0.conv2.weight"], sd["div_4.1.0.conv2.weight"], rtol=0, atol=0)


def test_geometry_model_regimes_and_library_agree():
    """every cell of the geometry model is reached for every channels-per-group value and stride, and the library's
    wgrad split and workspace size are the model's (they need no device)"""
    from distributed_sod_project_b200 import _lib
    cases = geo.regime_cases()
    for cpg in geo.CPG:
        for stride in (1, 2):
            cells = {c[-1] for c in cases if c[3:5] == (cpg, stride)}
            assert {"single", "split"} <= {c[0] for c in cells}
            assert {"even", "short"} == {c[1] for c in cells}
            assert {"whole", "tail"} == {c[2] for c in cells}
            assert {"full", "partial"} == {c[3] for c in cells}
    assert any(c[-1][0] == "capped" for c in cases)
    lib = _lib.lib()
    for n, h, w, cpg, stride, _ in cases + [(16, 80, 80, 4, 1, None), (16, 20, 20, 32, 2, None)]:
        p = n * geo.out_size(h, stride) * geo.out_size(w, stride)
        s, pc = geo.wgrad_geometry(p)
        assert (s - 1) * pc < p <= s * pc and pc % geo.WG_PIXELS == 0 and 1 <= s <= geo.WG_MAX_SPLIT
        c = 32 * cpg
        assert lib.sod_gconv3x3_wgrad_splits(n, h, w, c, 32, stride) == s
        assert lib.sod_gconv3x3_wgrad_workspace_bytes(n, h, w, c, 32, stride) == s * c * 9 * cpg * 4
    assert geo.wgrad_geometry(16 * 80 * 80)[0] == geo.WG_MAX_SPLIT


def test_gconv_abi_is_declared_bound_and_refuses_bad_arguments():
    from distributed_sod_project_b200 import _lib
    header = open(os.path.join(ROOT, "include", "sod_b200.h")).read()
    for name in ("sod_gconv3x3_fwd", "sod_gconv3x3_dgrad", "sod_gconv3x3_wgrad", "sod_gconv3x3_wgrad_splits",
                 "sod_gconv3x3_wgrad_workspace_bytes"):
        assert f" {name}(" in header and name in _lib.EXPORTS
    assert "#define SOD_GCONV_GROUPS 32" in header and _lib.SOD_GCONV_GROUPS == 32
    h = _lib.lib()
    assert h.sod_version() == 7
    assert h.sod_gconv3x3_fwd(None, None, None, 1, 1, 8, 8, 256, 32, 1, None) == -1
    assert h.sod_gconv3x3_dgrad(None, None, None, 1, 1, 8, 8, 256, 32, 1, None) == -1
    assert h.sod_gconv3x3_wgrad(None, None, None, 1, 1, 8, 8, 256, 32, 1, None, 0, None) == -1
    assert h.sod_gconv3x3_wgrad_splits(1, 8, 8, 256, 16, 1) == 0          # 16 groups
    assert h.sod_gconv3x3_wgrad_splits(1, 8, 8, 2048, 32, 1) == 0         # 64 channels per group
    assert h.sod_gconv3x3_wgrad_splits(1, 8, 8, 256, 32, 3) == 0          # stride 3
    assert h.sod_gconv3x3_wgrad_workspace_bytes(0, 8, 8, 256, 32, 1) == 0


def test_cpu_tensors_are_refused_by_the_grouped_seam():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.wsgn import FusedWSConv2d
    m = FusedWSConv2d(128, 128, 3, 1, 1, groups=32, bias=False)
    with pytest.raises(_lib.SodError):
        m(torch.randn(1, 128, 4, 4))
