"""CPU checks of the `aim_res50` / `cp_aim_res50` plugins (ResNet-50, MINet's LightAIM neck, the TestModel decoder):
init and forward bit for bit against the reference's modules, the neck's names, order and sizes, f3_trick's groups, the
input-size check, and the C entries and oracle of the nearest ×2 kernels the neck runs on."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

from _nearest import upsample2x_nearest_bwd, upsample2x_nearest_bwd64, upsample2x_nearest_fwd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# registration order of the reference's conv_2nV1 / conv_3nV1 (module/MyLightModule.py:57-213)
_2N_HEAD = ["h2h_0", "l2l_0", "bnh_0", "bnl_0", "h2h_1", "h2l_1", "l2h_1", "l2l_1", "bnl_1", "bnh_1"]
_2N = {0: _2N_HEAD + ["h2h_2", "l2h_2", "bnh_2", "h2h_3", "bnh_3", "identity"],
       1: _2N_HEAD + ["h2l_2", "l2l_2", "bnl_2", "l2l_3", "bnl_3", "identity"]}
_3N = ["h2h_0", "m2m_0", "l2l_0", "bnh_0", "bnm_0", "bnl_0", "h2h_1", "h2m_1", "m2h_1", "m2m_1", "m2l_1", "l2m_1", "l2l_1",
       "bnh_1", "bnm_1", "bnl_1", "h2m_2", "l2m_2", "m2m_2", "bnm_2", "m2m_3", "bnm_3", "identity"]


def _model(name):
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return getattr(network, name)()


@pytest.mark.parametrize("name", ["aim_res50", "cp_aim_res50"])
def test_aim_plugin_is_bit_identical_to_reference(golden, name):
    """after init_seed(0), against the reference's modules composed as MINet_Res50 (tests/golden/model_aim_res50_init.npz,
    `tools/make_golden_backbones.py aim_res50`): state_dict keys and shapes, 32 fixed values and the moments of every
    tensor, and one training-mode forward at the 8 intra-op threads the vectors were made with"""
    g = golden("model_aim_res50_init.npz")
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


def test_neck_names_order_and_sizes():
    """`trans.conv{0..4}.<name>` in the reference's registration order; 91 035 072 neck parameters (85 674 240 of them in
    conv4, whose mid_c is min(1024, 2048)), 65 convolutions and 36 BatchNorms; the rest of the model is res50's minus the
    trans convolutions; cp_aim_res50 has the same parameters"""
    m = _model("aim_res50")
    neck = m.trans
    for i, layout in enumerate((_2N[0], _3N, _3N, _3N, _2N[1])):
        block = getattr(neck, f"conv{i}")
        assert [n for n, c in block.named_children() if isinstance(c, (nn.Conv2d, nn.BatchNorm2d))] == layout
    names = [n for n, _ in m.named_parameters()]
    assert sum(p.numel() for n, p in m.named_parameters() if n.startswith("trans.")) == 91_035_072
    assert sum(p.numel() for n, p in m.named_parameters() if n.startswith("trans.conv4.")) == 85_674_240
    assert sum(isinstance(x, nn.Conv2d) for x in neck.modules()) == 65
    assert sum(isinstance(x, nn.BatchNorm2d) for x in neck.modules()) == 36
    r = _model("res50")
    rest = [n for n, _ in r.named_parameters() if not n.startswith("trans")]
    assert [n for n in names if not n.startswith("trans.")] == rest
    ni = names.index("trans.conv0.h2h_0.weight")
    assert names[ni - 1].startswith("div_32.") and names[ni + 2 * 65 + 2 * 36] == "sim32.h2l_0.weight"
    cp = _model("cp_aim_res50")
    assert [(n, p.shape) for n, p in cp.named_parameters()] == [(n, p.shape) for n, p in m.named_parameters()]
    assert all(torch.equal(a, b) for a, b in zip(cp.state_dict().values(), m.state_dict().values()))


def test_f3_trick_groups_put_the_neck_in_the_head():
    from distributed_sod_project_b200.optim import make_optimizer
    m = _model("aim_res50")
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    groups = [[n for n, p in m.named_parameters() if any(p is q for q in g["params"])] for g in opt.param_groups]
    assert [g["lr"] for g in opt.param_groups] == pytest.approx([0.005, 0.05])
    assert all(n.startswith("div") and not n.startswith("div_2") for n in groups[0])
    neck = {n for n, _ in m.named_parameters() if n.startswith("trans.")}
    assert neck <= set(groups[1]) and len(neck) == 2 * 65 + 2 * 36
    assert {n for n, _ in m.named_parameters()} - set(groups[0]) - set(groups[1]) == \
        {"div_2.0.weight", "div_2.1.weight", "div_2.1.bias"}


@pytest.mark.parametrize("hw", [(80, 64), (64, 48), (100, 100)])
def test_input_sides_must_be_multiples_of_32(hw):
    """the plugin refuses a side the neck's nearest ×2 cannot line up with the ResNet maps, naming it, before any
    layer runs"""
    m = _model("aim_res50")
    calls = []
    m.div_2.register_forward_pre_hook(lambda *a: calls.append(1))
    with pytest.raises(ValueError, match=re.escape(str(hw))):
        m(torch.zeros(1, 3, *hw))
    assert not calls


def test_nearest_entries_are_declared_and_bound():
    from distributed_sod_project_b200 import _lib
    header = open(os.path.join(ROOT, "include", "sod_b200.h")).read()
    for name in ("sod_upsample2x_nearest_fwd", "sod_upsample2x_nearest_bwd"):
        proto = re.search(rf"int {name}\(([^)]*)\);", header)
        assert proto, name
        assert proto.group(1).replace(" ", "").startswith(("constvoid*x,void*y", "constvoid*dy,void*dx"))
        assert name in _lib.EXPORTS and len(_lib._PROTOTYPES[name][1]) == 8


@pytest.mark.parametrize("shape", [(2, 8, 5, 7), (1, 64, 4, 4), (3, 16, 1, 9)])
def test_nearest_oracle_matches_torch(shape):
    """the restated kernels against `nn.Upsample(scale_factor=2, mode="nearest")` on the CPU: the forward equal; the
    fp32 backward within one rounding per add of the float64 sum, which equals float64 autograd's gradient"""
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(*shape, generator=g, dtype=torch.float64, requires_grad=True)
    y = nn.Upsample(scale_factor=2, mode="nearest")(x)
    assert torch.equal(upsample2x_nearest_fwd(x.detach()), y.detach())
    assert torch.equal(upsample2x_nearest_fwd(x.detach().float()), y.detach().float())
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (ref,) = torch.autograd.grad(y, x, dy)
    exact = upsample2x_nearest_bwd64(dy)
    torch.testing.assert_close(exact, ref, rtol=1e-15, atol=1e-15)
    dy32 = dy.float()
    got = upsample2x_nearest_bwd(dy32)
    assert got.dtype == torch.float32 and got.shape == x.shape
    bound = 3 * torch.finfo(torch.float32).eps * upsample2x_nearest_bwd64(dy32.abs())
    assert bool(((got.double() - upsample2x_nearest_bwd64(dy32)).abs() <= bound).all())
    assert torch.equal(got[0, 0, 0, 0], ((dy32[0, 0, 0, 0] + dy32[0, 0, 0, 1]) + dy32[0, 0, 1, 0]) + dy32[0, 0, 1, 1])
