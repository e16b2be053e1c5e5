"""CPU checks of the WS-GN plugins (`wsgn_res50`, `cp_wsgn_res50`): bit-identity with the reference's weight-standardised
GroupNorm ResNet-50 TestModel, names and optimizer groups, the WS-GN release's pretrained file format, the fp64 oracle
of csrc/wsgn.cu, its launch-geometry model and the C ABI of the new entries."""
from __future__ import annotations

import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import wsgn as owsgn
from oracle import wsgn_geometry as geo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(name="wsgn_res50"):
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return getattr(network, name)()


@pytest.mark.parametrize("name", ["wsgn_res50", "cp_wsgn_res50"])
def test_wsgn_plugin_is_bit_identical_to_reference(golden, name):
    """init_seed(0) + the plugin against the reference TestModel on backbone.wsgn (tests/golden/model_wsgn_res50_init.npz,
    tools/make_golden_wsgn.py): same keys and shapes, the same values at fixed positions and per-tensor sums, and the
    same output of one training-mode forward at the 8 threads the vectors were made with"""
    g = golden("model_wsgn_res50_init.npz")
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


def test_wsgn_names_norms_and_f3_trick_groups():
    from distributed_sod_project_b200.network.blocks import WSConv2d
    from distributed_sod_project_b200.optim import make_optimizer
    m = _model()
    names = [n for n, _ in m.named_parameters()]
    assert names[:3] == ["div_2.0.weight", "div_2.1.weight", "div_2.1.bias"] and names[-1] == "classifier.bias"
    assert sum(isinstance(x, nn.GroupNorm) for x in m.modules()) == 53
    assert sum(isinstance(x, WSConv2d) for x in m.modules()) == 53
    assert all(x.num_groups == 32 and x.eps == 1e-5 for x in m.modules() if isinstance(x, nn.GroupNorm))
    # GroupNorm keeps no running statistics: the only buffers are the decoder's BatchNorm ones
    assert all(not b.startswith("div") for b, _ in m.named_buffers())
    assert sum(isinstance(x, nn.BatchNorm2d) for x in m.modules()) == 84 - 53
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    grouped = [[n for n, p in m.named_parameters() if any(p is q for q in g["params"])] for g in opt.param_groups]
    assert [g["lr"] for g in opt.param_groups] == pytest.approx([0.005, 0.05])
    assert all(n.startswith("div") and not n.startswith("div_2") for n in grouped[0])
    assert all(not n.startswith("div") for n in grouped[1])
    frozen = set(names) - set(grouped[0]) - set(grouped[1])
    assert frozen == {"div_2.0.weight", "div_2.1.weight", "div_2.1.bias"}
    # no WS convolution's parameters are in the optimizer's 16-bit gradient part of the flat buffer
    ws_ids = {id(x.weight) for x in m.modules() if isinstance(x, WSConv2d)}
    f = opt.flat
    for p, off in f.slots:
        if id(p) in ws_ids:
            bucket = next(i for i, (b, e) in enumerate(f.ranges) if b <= off < e)
            assert off >= f.splits[bucket], "a WS weight sits in the 16-bit gradient range"


def test_res50_flat_layout_is_unchanged_by_the_ws_exclusion():
    """the optimizer's 16-bit / fp32 split of res50 is exactly the one every plain convolution gives"""
    from distributed_sod_project_b200.optim import make_optimizer
    m = _model("res50")
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    conv = {id(p) for x in m.modules() if isinstance(x, nn.Conv2d) for p in (x.weight, x.bias) if p is not None}
    f = opt.flat
    for p, off in f.slots:
        bucket = next(i for i, (b, e) in enumerate(f.ranges) if b <= off < e)
        assert (off < f.splits[bucket]) == (id(p) in conv)


def test_load_pretrained_backbone_reads_the_wsgn_release_format(tmp_path):
    """the WS-GN release's file: tensors under "state_dict", keys `module.`-prefixed, torchvision naming; unknown and
    mis-shaped keys ignored"""
    from distributed_sod_project_b200.network import load_pretrained_backbone
    m = _model()
    sd = m.state_dict()
    g = torch.Generator().manual_seed(5)
    src = {"module.conv1.weight": torch.randn(sd["div_2.0.weight"].shape, generator=g),
           "module.bn1.weight": torch.rand(64, generator=g), "module.bn1.bias": torch.rand(64, generator=g),
           "module.layer3.5.conv2.weight": torch.randn(sd["div_16.5.conv2.weight"].shape, generator=g),
           "module.layer4.2.bn3.bias": torch.rand(2048, generator=g),
           "module.fc.weight": torch.zeros(1000, 2048), "module.layer1.0.conv1.weight": torch.zeros(3, 3)}
    path = tmp_path / "R-50-GN-WS.pth.tar"
    torch.save({"epoch": 90, "arch": "l_resnet50", "state_dict": src}, path)
    loaded = load_pretrained_backbone(m, str(path))
    assert loaded == sorted(["div_2.0.weight", "div_2.1.weight", "div_2.1.bias", "div_16.5.conv2.weight",
                             "div_32.2.bn3.bias"])
    now = m.state_dict()
    torch.testing.assert_close(now["div_2.0.weight"], src["module.conv1.weight"], rtol=0, atol=0)
    torch.testing.assert_close(now["div_32.2.bn3.bias"], src["module.layer4.2.bn3.bias"], rtol=0, atol=0)
    torch.testing.assert_close(now["div_4.1.0.conv1.weight"], sd["div_4.1.0.conv1.weight"], rtol=0, atol=0)


@pytest.mark.parametrize("relu,res", [(False, False), (True, False), (True, True)])
def test_group_norm_oracle_matches_torch_fp64(relu, res):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(2, 64, 5, 3, generator=g, dtype=torch.float64) * 3 + 7).requires_grad_(True)
    gamma = (torch.rand(64, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True)
    beta = torch.randn(64, generator=g, dtype=torch.float64).requires_grad_(True)
    r = torch.randn(2, 64, 5, 3, generator=g, dtype=torch.float64).requires_grad_(True) if res else None
    y = torch.nn.functional.group_norm(x, 32, gamma, beta, 1e-5)
    if r is not None:
        y = y + r
    if relu:
        y = torch.relu(y)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(dy)
    o = owsgn.group_norm_forward(x.detach().numpy(), gamma.detach().numpy(), beta.detach().numpy(),
                                 None if r is None else r.detach().numpy(), relu)
    np.testing.assert_allclose(o["y"], y.detach().numpy(), rtol=1e-12, atol=1e-12)
    b = owsgn.group_norm_backward(dy.numpy(), x.detach().numpy(), gamma.detach().numpy(), beta.detach().numpy(),
                                  None if r is None else r.detach().numpy(), relu)
    np.testing.assert_allclose(b["dx"], x.grad.numpy(), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(b["dgamma"], gamma.grad.numpy(), rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(b["dbeta"], beta.grad.numpy(), rtol=1e-10, atol=1e-10)
    if r is not None:
        np.testing.assert_allclose(b["dres"], r.grad.numpy(), rtol=0, atol=0)


def test_ws_oracle_matches_the_reference_expression_in_fp64():
    """the oracle's Ŵ and hand-derived dW against float64 autograd of the plugin's (= the reference's) expression, on
    the golden init weights of every filter shape of the backbone"""
    from distributed_sod_project_b200.network.blocks import WSConv2d
    m = _model()
    seen = set()
    g = torch.Generator().manual_seed(2)
    for mod in m.modules():
        if not isinstance(mod, WSConv2d) or tuple(mod.weight.shape) in seen:
            continue
        seen.add(tuple(mod.weight.shape))
        w = mod.weight.detach().double().clone().requires_grad_(True)
        ref = WSConv2d.standardized_weight(type("P", (), {"weight": w, "eps": 1e-5})())
        up = torch.randn(w.shape, generator=g, dtype=torch.float64)
        ref.backward(up)
        np.testing.assert_allclose(owsgn.ws_forward(w.detach().numpy()), ref.detach().numpy(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(owsgn.ws_backward(w.detach().numpy(), up.numpy()), w.grad.numpy(),
                                   rtol=1e-9, atol=1e-9 * float(w.grad.abs().max()))
    assert len(seen) == 20


def test_geometry_model_regimes():
    """every split / tail / phase / lane cell the kernels have is reachable on a 132-SM H100 and on other SM counts,
    the stem of the benched workload (16 × 160² × 64) splits across CTAs, and no CTA is empty"""
    for sms in (132, 114, 148):
        cells = {c[-1] for c in geo.regime_cases(sms)}
        assert {"one", "many"} == {c[0] for c in cells}
        assert {"even", "short"} == {c[1] for c in cells}
        assert {"idle", "full"} == {c[2] for c in cells}
        assert {"multi", "single"} == {c[3] for c in cells}
    g = geo.make_geom(16, 160 * 160, 64, 132)
    assert g.S > 1 and g.S * 16 <= 2 * 132 + 16
    for n in (1, 2, 16):
        for hw in (1, 7, 100, 25600, 36864):
            for c in geo.CHANNELS:
                g = geo.make_geom(n, hw, c, 132)
                assert 1 <= g.S <= geo.MAX_SPLIT and (g.S - 1) * g.rc < hw <= g.S * g.rc


def test_wsgn_abi_is_declared_and_bound():
    """the new entries are in the header and bound with matching prototypes (argument kinds are checked for every
    entry by tests/test_host_cpu.py); the version stays 7; shape and argument refusals need no device"""
    from distributed_sod_project_b200 import _lib
    header = open(os.path.join(ROOT, "include", "sod_b200.h")).read()
    for name in ("sod_groupnorm_workspace_bytes", "sod_groupnorm_splits", "sod_groupnorm_fwd", "sod_groupnorm_bwd",
                 "sod_ws_fwd", "sod_ws_bwd"):
        assert f" {name}(" in header and name in _lib.EXPORTS
    assert "#define SOD_GN_GROUPS 32" in header and _lib.SOD_GN_GROUPS == 32
    h = _lib.lib()
    assert h.sod_version() == 7
    assert h.sod_ws_fwd(None, None, 0, 1, 9, ctypes.c_float(1e-5), None) == -1
    assert h.sod_groupnorm_fwd(None, None, None, 0, None, None, None, 1, 1, 64, 32, ctypes.c_float(1e-5), 0, None, 0,
                               None) == -1


class _RefStyleWSConv(nn.Conv2d):
    """the reference's backbone/wsgn/customized_func.Conv2d pattern: an nn.Conv2d subclass whose forward standardises"""

    def forward(self, x):
        w = self.weight - self.weight.mean(dim=(1, 2, 3), keepdim=True)
        w = w / (w.reshape(w.size(0), -1).std(dim=1).view(-1, 1, 1, 1) + 1e-5)
        return torch.nn.functional.conv2d(x, w, self.bias, self.stride, self.padding, self.dilation, self.groups)


class _OwnConvForward(nn.Conv2d):
    def _conv_forward(self, x, weight, bias):
        return super()._conv_forward(x, weight * 2.0, bias)


class _KeepsForward(nn.Conv2d):
    """a subclass that changes nothing about the convolution"""


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=str)
def test_amp_and_optimizer_leave_every_convolution_with_its_own_forward_alone(dtype):
    """a Conv2d subclass with its own forward or _conv_forward (a weight-standardised convolution of any origin) gets no
    16-bit shadow, keeps its forward, and its parameters sit in the fp32-gradient part of the flat buffer; plain
    convolutions and subclasses that keep nn.Conv2d's forward are shadowed as before"""
    from distributed_sod_project_b200 import amp
    from distributed_sod_project_b200.network.blocks import WSConv2d
    from distributed_sod_project_b200.optim import FusedSGD, is_plain_conv
    net = nn.Sequential(nn.Conv2d(3, 8, 3, padding=1), _RefStyleWSConv(8, 8, 3, padding=1, bias=False),
                        _OwnConvForward(8, 8, 1), _KeepsForward(8, 8, 1), WSConv2d(8, 4, 3, bias=False))
    assert [is_plain_conv(m) for m in net] == [True, False, False, True, False]
    opt = FusedSGD(net.parameters(), lr=0.1, momentum=0.9, model=net)
    f = opt.flat
    f.enable_shadow(dtype)
    assert amp._install_shadow_weights(net, f) == 2
    for m, plain in zip(net, [True, False, False, True, False]):
        assert hasattr(m, "_sod_w16") == plain
        assert ("forward" in vars(m)) == plain                 # the instance forward is only patched on plain ones
        for p in (m.weight, m.bias):
            if p is None:
                continue
            off = f.offset_of(p)
            bucket = next(i for i, (b, e) in enumerate(f.ranges) if b <= off < e)
            assert (off < f.splits[bucket]) == plain
    x = torch.randn(1, 3, 6, 6)
    ref = x
    for m in net:
        ref = type(m).forward(m, ref)
    with torch.no_grad():
        assert torch.equal(net(x), ref)
