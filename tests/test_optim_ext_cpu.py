"""CPU checks of the fused Adam and of Nesterov SGD: ABI layout, the reference's `make_optimizer` groupings for optim
"adam" and `nesterov: True`, the Adam oracle against the reference's trajectory (tests/golden/optim_ext_kat.npz, written
by tools/make_golden_optim.py), and `FusedAdam`'s torch.optim.Adam state_dict layout."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import adam as oadam


class _Tiny(torch.nn.Module):
    """the module the golden vectors were recorded with (tools/make_golden.py)"""

    def __init__(self):
        super().__init__()
        self.div_2 = torch.nn.Linear(5, 7); self.div_4 = torch.nn.Linear(7, 6)
        self.div_16 = torch.nn.Linear(6, 3, bias=False); self.head = torch.nn.Linear(3, 2)
        self.classifier = torch.nn.Linear(2, 1)


def _info(nesterov=False):
    return dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=nesterov)


def _tiny_from(flat):
    net = _Tiny()
    off = 0
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(torch.from_numpy(flat[off:off + p.numel()]).view_as(p)); off += p.numel()
    return net


def test_adam_segment_layout_and_entry_points():
    from distributed_sod_project_b200 import _lib
    assert ctypes.sizeof(_lib.sod_adam_segment) == 40 and ctypes.sizeof(_lib.sod_sgd_segment) == 32
    assert _lib.SOD_SEG_NESTEROV == 4 and _lib.SOD_ADAM_STEP_WORDS == _lib.SOD_MAX_SEGMENTS + 1
    assert {"sod_adam", "sod_allreduce_adam"} <= set(_lib.EXPORTS)


def test_make_optimizer_adam_matches_reference_groups(golden):
    from distributed_sod_project_b200.optim import FusedAdam, make_optimizer
    g = golden("optim_ext_kat.npz")
    net = _Tiny()
    opt = make_optimizer(net, "adam", _info())
    assert isinstance(opt, FusedAdam) and "FusedAdam" in str(opt)
    assert [n for n, _ in net.named_parameters()] == list(g["adam/names"])
    of = [next((gi for gi, gr in enumerate(opt.param_groups) if any(p is q for q in gr["params"])), -1)
          for _, p in net.named_parameters()]
    np.testing.assert_array_equal(of, g["adam/group_of"])
    np.testing.assert_array_equal([gr["lr"] for gr in opt.param_groups], g["adam/group_lr"])
    np.testing.assert_array_equal([gr["weight_decay"] for gr in opt.param_groups], g["adam/group_wd"])
    np.testing.assert_array_equal([gr["betas"] for gr in opt.param_groups], g["adam/group_betas"])
    np.testing.assert_array_equal([gr["eps"] for gr in opt.param_groups], g["adam/group_eps"])
    # one group over every parameter: no frozen segment; exp_avg_sq beside exp_avg
    segs, n = opt._segments()
    assert n == 1 and segs[0].flags == 0 and segs[0].end == opt.flat.numel
    assert abs(segs[0].beta1 - 0.9) < 1e-7 and abs(segs[0].beta2 - 0.999) < 1e-7 and abs(segs[0].eps - 1e-8) < 1e-15
    assert opt.exp_avg is opt.flat.mom and opt.exp_avg_sq.shape == opt.flat.mom.shape


@pytest.mark.parametrize("kind", ["sgd_trick", "f3_trick"])
def test_make_optimizer_nesterov_matches_reference_groups(golden, kind):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.optim import FusedSGD, make_optimizer
    g = golden("optim_ext_kat.npz")
    tag = f"{kind}_nesterov"
    net = _Tiny()
    opt = make_optimizer(net, kind, _info(nesterov=True))
    assert isinstance(opt, FusedSGD)
    of = [next((gi for gi, gr in enumerate(opt.param_groups) if any(p is q for q in gr["params"])), -1)
          for _, p in net.named_parameters()]
    np.testing.assert_array_equal(of, g[f"{tag}/group_of"])
    np.testing.assert_allclose([gr["lr"] for gr in opt.param_groups], g[f"{tag}/group_lr"], rtol=1e-12)
    np.testing.assert_array_equal([gr["weight_decay"] for gr in opt.param_groups], g[f"{tag}/group_wd"])
    np.testing.assert_array_equal([gr["nesterov"] for gr in opt.param_groups], g[f"{tag}/group_nesterov"])
    segs, n = opt._segments()
    for i in range(n):
        frozen = bool(segs[i].flags & _lib.SOD_SEG_FROZEN)
        assert bool(segs[i].flags & _lib.SOD_SEG_NESTEROV) == (not frozen)
    # without nesterov the flag stays off (the default configuration is unchanged)
    segs, n = make_optimizer(_Tiny(), kind, _info())._segments()
    assert not any(segs[i].flags & _lib.SOD_SEG_NESTEROV for i in range(n))


def test_nesterov_needs_momentum_and_adam_refuses_what_it_does_not_implement():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.optim import FusedAdam, FusedSGD, make_optimizer
    with pytest.raises(ValueError):
        make_optimizer(_Tiny(), "f3_trick", dict(lr=0.05, momentum=0.0, weight_decay=5e-4, nesterov=True))
    with pytest.raises(ValueError):
        FusedSGD(_Tiny().parameters(), lr=0.1, momentum=0.0, nesterov=True)
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(decoupled_weight_decay=True)):
        with pytest.raises(_lib.SodError):
            FusedAdam(_Tiny().parameters(), lr=1e-3, **kw)


def _adam_segments(g, it):
    """the golden Adam run as oracle segments: one group over the whole (unpadded) flat vector"""
    n = g["adam/p0"].size
    b1, b2 = g["adam/group_betas"][0]
    return [oadam.Segment(0, n, float(g[f"adam/lr{it}"][0]), float(g["adam/group_wd"][0]), float(b1), float(b2),
                          float(g["adam/group_eps"][0]))]


def test_adam_oracle_follows_reference_trajectory(golden):
    g = golden("optim_ext_kat.npz")
    p = g["adam/p0"].astype(np.float32).copy()
    m = np.zeros_like(p); v = np.zeros_like(p); steps = [0]
    p64, m64, v64, steps64 = p.astype(np.float64), np.zeros(p.size), np.zeros(p.size), [0]
    for it in range(4):
        segs = _adam_segments(g, it)
        grad = g[f"adam/g{it}"].astype(np.float32)
        assert oadam.adam_step(p, m, v, grad, segs, steps)
        p64, m64, v64, steps64 = oadam.adam_step_f64(p64, m64, v64, grad, segs, steps64)
        want = g[f"adam/p{it + 1}"]
        np.testing.assert_allclose(p, want, rtol=3e-6, atol=2e-7)
        np.testing.assert_allclose(p64, want, rtol=3e-6, atol=2e-7)
        # fp32 oracle, fp64 oracle and torch agree; fp64 sits within fp32 rounding of torch's fp32 result
        assert np.abs(p64 - want).max() <= np.abs(p.astype(np.float64) - want).max() + 1e-7
    assert steps == steps64 == [4]
    np.testing.assert_allclose(m, g["adam/state_exp_avg"], rtol=3e-6, atol=1e-8)
    np.testing.assert_allclose(v, g["adam/state_exp_avg_sq"], rtol=3e-6, atol=1e-12)
    np.testing.assert_array_equal(g["adam/state_step"], 4.0)
    # the overflow skip touches nothing
    before = p.copy()
    bad = g["adam/g0"].astype(np.float32).copy(); bad[3] = np.inf
    assert not oadam.adam_step(p, m, v, bad, _adam_segments(g, 0), steps)
    assert steps == [4] and np.array_equal(p, before)


def _torch_adam_state(g):
    """torch.optim.Adam (CPU) stepped 4 times over the golden gradients: the state_dict a reference checkpoint holds"""
    net = _tiny_from(g["adam/p0"])
    ref = torch.optim.Adam(net.parameters(), lr=0.05, betas=(0.9, 0.999), eps=1e-8, weight_decay=5e-4)
    for it in range(4):
        ref.param_groups[0]["lr"] = float(g[f"adam/lr{it}"][0])          # the golden run's poly schedule
        off = 0
        for p in net.parameters():
            p.grad = torch.from_numpy(g[f"adam/g{it}"][off:off + p.numel()]).view_as(p).clone(); off += p.numel()
        ref.step()
    return net, ref.state_dict()


def test_torch_adam_state_dict_round_trips_through_fused_adam(golden):
    from distributed_sod_project_b200.optim import make_optimizer
    g = golden("optim_ext_kat.npz")
    net_ref, sd = _torch_adam_state(g)
    net = _tiny_from(g["adam/p0"])
    opt = make_optimizer(net, "adam", _info())
    assert opt.state_dict()["state"] == {}                         # no state before the first step, as torch
    opt.load_state_dict(sd)
    assert opt.group_steps() == [4] and opt.step_dev.tolist()[:1] == [4]
    for p, (i, st) in zip(net.parameters(), sorted(sd["state"].items())):
        assert torch.equal(opt.flat.momentum_view(p), st["exp_avg"])
    back = opt.state_dict()
    assert set(back["state"]) == set(sd["state"])
    for i, st in sd["state"].items():
        got = back["state"][i]
        assert got["step"].dtype == torch.float32 and got["step"].dim() == 0 and float(got["step"]) == float(st["step"])
        assert torch.equal(got["exp_avg"], st["exp_avg"]) and torch.equal(got["exp_avg_sq"], st["exp_avg_sq"])
    assert back["param_groups"][0]["betas"] == (0.9, 0.999) and back["param_groups"][0]["lr"] == sd["param_groups"][0]["lr"]
    # torch of 2020 (the reference's) wrote `step` as an int
    old = {"state": {i: dict(st, step=int(st["step"])) for i, st in sd["state"].items()}, "param_groups": sd["param_groups"]}
    opt2 = make_optimizer(_tiny_from(g["adam/p0"]), "adam", _info())
    opt2.load_state_dict(old)
    assert opt2.group_steps() == [4] and torch.equal(opt2.exp_avg_sq, opt.exp_avg_sq)
    # the golden state after step 4 is what torch.optim.Adam holds here as well
    for key in ("exp_avg", "exp_avg_sq"):
        np.testing.assert_allclose(torch.cat([s[key].reshape(-1) for _, s in sorted(sd["state"].items())]).numpy(),
                                   g[f"adam/state_{key}"], rtol=1e-6, atol=1e-12)


def test_mismatched_steps_within_a_group_raise(golden):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.optim import make_optimizer
    g = golden("optim_ext_kat.npz")
    _, sd = _torch_adam_state(g)
    sd["state"][2]["step"] = torch.tensor(3.0)
    opt = make_optimizer(_tiny_from(g["adam/p0"]), "adam", _info())
    with pytest.raises(_lib.SodError):
        opt.load_state_dict(sd)
    assert opt.group_steps() == [0] and float(opt.exp_avg_sq.abs().max()) == 0.0     # nothing half-loaded
    del sd["state"][5]                                                                 # a parameter without state: step 0
    sd["state"][2]["step"] = torch.tensor(4.0)
    with pytest.raises(_lib.SodError):
        opt.load_state_dict(sd)
