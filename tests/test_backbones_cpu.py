"""CPU checks shared by every backbone of tests/_backbones.py: each model plugin's init and forward bit for bit against
the reference's TestModel on that backbone, and f3_trick's optimizer groups."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from _backbones import PLUGINS


def _model(name):
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return getattr(network, name)()


@pytest.mark.parametrize("name", ["res50", "cp_res50"] + [n for r in PLUGINS for n in (r.name, r.cp)])
def test_model_plugin_is_bit_identical_to_reference(golden, name):
    """the plugin after init_seed(0) against the reference's model (tests/golden/model_<backbone>_init.npz, written by
    `tools/make_golden.py --only-model-init` for res50 and `tools/make_golden_backbones.py` for the others): same
    state_dict keys and shapes, the same values at 32 fixed positions of every tensor, the same per-tensor sums, and the
    same full-resolution output of one training-mode forward pass.  The forward runs at the 8 intra-op threads the
    vectors were made with: the CPU batch-norm reductions are split by thread count."""
    g = golden(f"model_{name.removeprefix('cp_')}_init.npz")
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
    assert y.shape == g["x"].shape[:1] + (1,) + g["x"].shape[2:]
    np.testing.assert_array_equal(y, g["y"])


@pytest.mark.parametrize("row", PLUGINS, ids=lambda r: r.name)
def test_f3_trick_groups(row):
    """group 0 is the backbone without div_2 at 0.1·lr, group 1 everything outside the backbone at lr, and the row's
    div_2 parameters are in neither"""
    from distributed_sod_project_b200.optim import make_optimizer
    m = _model(row.name)
    opt = make_optimizer(m, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    names = [n for n, _ in m.named_parameters()]
    groups = [[n for n, p in m.named_parameters() if any(p is q for q in g["params"])] for g in opt.param_groups]
    assert [g["lr"] for g in opt.param_groups] == pytest.approx([0.005, 0.05])
    assert all(n.startswith("div") and not n.startswith("div_2") for n in groups[0])
    assert all(not n.startswith("div") for n in groups[1])
    assert set(names) - set(groups[0]) - set(groups[1]) == row.frozen
