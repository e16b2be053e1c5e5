"""CPU checks of the VGG16-BN plugins (`vgg16`, `cp_vgg16`): bit-identity with the reference's TestModel composed on
`Backbone_VGG16_in3`, names, counts and optimizer groups, torchvision's `vgg16_bn` file format, the CPU routing of the
2×2 pools, and the C ABI of the 2×2 max-pool entries."""
from __future__ import annotations

import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(name="vgg16"):
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return getattr(network, name)()


@pytest.mark.parametrize("name", ["vgg16", "cp_vgg16"])
def test_plugin_is_bit_identical_to_reference(golden, name):
    """init_seed(0) + the plugin against the reference composition (tests/golden/model_vgg16_init.npz,
    tools/make_golden_vgg.py): keys in order, shapes, values at fixed positions, per-tensor sums and one training-mode
    forward at 8 threads.  The first convolution's biases are torch's default uniform init, not zero"""
    g = golden("model_vgg16_init.npz")
    m = _model(name)
    sd = m.state_dict()
    assert "\n".join(sd) == str(g["keys"])
    for i, v in enumerate(sd.values()):
        assert list(v.shape) == [d for d in g["shapes"][i] if d >= 0]
        a = v.detach().reshape(-1).double()
        idx = torch.from_numpy(np.linspace(0, a.numel() - 1, g["values"].shape[1]).astype(np.int64))
        np.testing.assert_array_equal(a[idx].numpy(), g["values"][i])
        np.testing.assert_allclose([a.sum().item(), (a * a).sum().item()], g["moments"][i], rtol=1e-12, atol=0)
    assert 0.05 < float(m.div_2[0].bias.detach().abs().mean()) < 0.15
    threads = torch.get_num_threads()
    torch.set_num_threads(8)
    try:
        y = m(torch.from_numpy(g["x"])).detach().numpy()
    finally:
        torch.set_num_threads(threads)
    assert y.shape == g["x"].shape[:1] + (1,) + g["x"].shape[2:]          # full resolution: no ×2 head up-sample
    np.testing.assert_array_equal(y, g["y"])


def test_names_counts_and_f3_trick_groups():
    from distributed_sod_project_b200.network.blocks import _VGGPool
    from distributed_sod_project_b200.optim import make_optimizer
    m = _model()
    backbone = [m.div_2, m.div_4, m.div_8, m.div_16, m.div_32]
    assert [len(s) for s in backbone] == [6, 7, 10, 10, 10]
    convs = [x for s in backbone for x in s.modules() if isinstance(x, nn.Conv2d)]
    assert len(convs) == 13 and all(c.kernel_size == (3, 3) and c.padding == (1, 1) and c.bias is not None for c in convs)
    assert sum(isinstance(x, nn.BatchNorm2d) for s in backbone for x in s.modules()) == 13
    pools = [x for s in backbone for x in s.modules() if isinstance(x, nn.MaxPool2d)]
    assert len(pools) == 4 and all(isinstance(p, _VGGPool) for p in pools)
    assert all(isinstance(s[0], _VGGPool) for s in backbone[1:])
    assert [c.out_channels for c in convs] == [64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512]
    assert [m.get_submodule(f"trans{s}").in_channels for s in (32, 16, 8, 4, 2)] == [512, 512, 256, 128, 64]
    assert sum(p.numel() for n, p in m.named_parameters() if n.startswith("div")) == 14_723_136
    sd = m.state_dict()
    assert "div_4.1.weight" in sd and "div_4.2.running_var" in sd and "div_32.8.bias" in sd and "div_32.10.weight" not in sd
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    names = [n for n, _ in m.named_parameters()]
    groups = [[n for n, p in m.named_parameters() if any(p is q for q in g["params"])] for g in opt.param_groups]
    assert all(n.startswith("div") and not n.startswith("div_2") for n in groups[0])
    assert all(not n.startswith("div") for n in groups[1])
    assert set(names) - set(groups[0]) - set(groups[1]) == {f"div_2.{i}.{k}" for i in (0, 1, 3, 4) for k in ("weight", "bias")}


def test_cpu_forward_keeps_the_torch_pool():
    """on CPU tensors the pools and conv-BN-ReLU triples are the reference's torch ops"""
    m = _model().eval()
    x = torch.randn(1, 3, 16, 18)
    with torch.no_grad():
        feats = [x]
        for s in (m.div_2, m.div_4, m.div_8, m.div_16, m.div_32):
            feats.append(s(feats[-1]))
        ref = F.relu(m.div_4[2](m.div_4[1](F.max_pool2d(feats[1], 2, 2))))
        ref = F.relu(m.div_4[5](m.div_4[4](ref)))
    assert [tuple(f.shape[2:]) for f in feats[1:]] == [(16, 18), (8, 9), (4, 4), (2, 2), (1, 1)]
    assert torch.equal(feats[2], ref)


def test_load_pretrained_backbone_reads_torchvision_vgg16_bn(tmp_path):
    """a torchvision-format file made here from `torchvision.models.vgg16_bn(weights=None)`: every `features.*` tensor
    (weights, biases, BN statistics, num_batches_tracked) lands in its slice, `classifier.*` is ignored"""
    import torchvision
    from distributed_sod_project_b200.network import load_pretrained_backbone
    from distributed_sod_project_b200.network.blocks import VGG16_SLICES
    torch.manual_seed(3)
    tv = torchvision.models.vgg16_bn(weights=None)
    src = tv.state_dict()
    with torch.no_grad():
        for k, v in src.items():
            if k.startswith("features.") and v.is_floating_point():
                v.add_(torch.rand_like(v))                              # running_var / BN weights away from 1 / 0
    path = tmp_path / "vgg16_bn-6c64b313.pth"
    torch.save(src, path)
    m = _model()
    head_before = {k: v.clone() for k, v in m.state_dict().items() if not k.startswith("div")}
    loaded = load_pretrained_backbone(m, str(path))
    feats = [k for k in src if k.startswith("features.")]
    assert len(loaded) == len(feats) == 13 * 7
    own = m.state_dict()
    names = ("div_2", "div_4", "div_8", "div_16", "div_32")
    for k in feats:
        i = int(k.split(".")[1])
        s = next(j for j, (a, b) in enumerate(VGG16_SLICES) if a <= i < b)
        nk = f"{names[s]}.{i - VGG16_SLICES[s][0]}.{k.split('.', 2)[2]}"
        assert nk in loaded and torch.equal(own[nk], src[k]), k
    assert not any("classifier" in k and k.startswith("div") for k in loaded)
    for k, v in head_before.items():
        assert torch.equal(own[k], v), k


def test_maxpool2x2_abi_is_declared_bound_and_refuses_bad_arguments():
    """both entries are in the header and the ctypes table with the 3×3 entries' argument list; refusals return before
    anything is launched (the pointers below are never dereferenced)"""
    from distributed_sod_project_b200 import _lib
    header = open(os.path.join(ROOT, "include", "sod_b200.h")).read()
    for name in ("sod_maxpool2x2s2_fwd", "sod_maxpool2x2s2_bwd"):
        assert f" {name}(" in header and name in _lib.EXPORTS
        assert _lib._PROTOTYPES[name] == _lib._PROTOTYPES[name.replace("2x2", "3x3")]
    h = _lib.lib()
    assert h.sod_version() == 7
    a, b, c = 1 << 20, 2 << 20, 3 << 20
    for fn in (h.sod_maxpool2x2s2_fwd, h.sod_maxpool2x2s2_bwd):
        assert fn(None, b, c, 1, 4, 4, 8, 0, None) == -1                           # SOD_EINVAL
        assert fn(a + 8, b, c, 1, 4, 4, 8, 0, None) == -2                          # SOD_EALIGN
        assert fn(a, b, c + 4, 1, 4, 4, 8, 0, None) == -2
        assert fn(a, b, c, 1, 1, 4, 8, 0, None) == -4                              # h < 2: SOD_EUNSUPPORTED
        assert fn(a, b, c, 1, 4, 1, 8, 0, None) == -4                              # w < 2
        assert fn(a, b, c, 1, 4, 4, 12, 0, None) == -4                             # C % 8 != 0
        assert fn(a, b, c, 0, 4, 4, 8, 0, None) == -1
