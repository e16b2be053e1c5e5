"""Parity of the fused SGD-momentum kernel with the oracle / the reference optimizer's golden trajectory."""
import numpy as np
import pytest
import torch

from oracle import optim_replay as rp
from oracle import sgd as osgd

pytestmark = pytest.mark.gpu


def _segs(spec):
    from distributed_sod_project_b200 import _lib
    arr = (_lib.sod_sgd_segment * len(spec))()
    for i, (b, e, lr, wd, mu, fl) in enumerate(spec):
        arr[i] = _lib.sod_sgd_segment(b, e, lr, wd, mu, fl)
    return arr


def _call(p, v, g, spec, inv_scale=1.0, found=None, flags=1, lr_dev=None):
    from distributed_sod_project_b200 import _lib
    rc = _lib.lib().sod_sgd_momentum(p.data_ptr(), v.data_ptr(), g.data_ptr(), None, None, p.numel(), _segs(spec), len(spec),
                                     lr_dev.data_ptr() if lr_dev is not None else None,
                                     inv_scale, found.data_ptr() if found is not None else None, flags,
                                     torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rc


@pytest.mark.parametrize("n", [4, 64, 4096 + 64, 1_000_000 + 4, 24_912_000])
def test_flat_kernel_vs_oracle(n):
    rng = np.random.default_rng(n)
    p0 = rng.standard_normal(n).astype(np.float32); v0 = rng.standard_normal(n).astype(np.float32)
    g0 = rng.standard_normal(n).astype(np.float32)
    a = (n // 3) // 4 * 4; b = (2 * n // 3) // 4 * 4
    spec = [(0, a, 0.005, 5e-4, 0.9, 0), (a, b, 0.05, 5e-4, 0.9, 0), (b, n, 0.0, 0.0, 0.0, 1)]
    segs = [osgd.Segment(0, a, 0.005, 5e-4, 0.9), osgd.Segment(a, b, 0.05, 5e-4, 0.9), osgd.Segment(b, n, 0, 0, frozen=True)]
    p, v, g = (torch.tensor(t, device="cuda") for t in (p0, v0, g0))
    assert _call(p, v, g, spec, inv_scale=0.5) == 0
    # the kernel's own operation order, FMAs included (oracle/optim_replay.py): bit for bit
    table = [dict(begin=s[0], end=s[1], lr=s[2], wd=s[3], mu=s[4], flags=s[5]) for s in spec]
    pe, (ve,), _, _, _ = rp.step("sgd", p0, [v0], g0, None, table, inv_scale=0.5)
    np.testing.assert_array_equal(p.cpu().numpy().view(np.uint32), pe.view(np.uint32))
    np.testing.assert_array_equal(v.cpu().numpy().view(np.uint32), ve.view(np.uint32))
    np.testing.assert_array_equal(p.cpu().numpy()[b:], p0[b:])       # frozen range untouched
    assert float(g.abs().max()) == 0.0                                  # SOD_SGD_ZERO_GRAD
    p64, v64 = osgd.sgd_step_f64(p0, v0, g0, segs, inv_scale=0.5)
    np.testing.assert_allclose(p.cpu().numpy(), p64, rtol=1e-5, atol=1e-6)


def test_overflow_skip_keeps_state_and_clears_grads():
    n = 4096
    p = torch.ones(n, device="cuda"); v = torch.full((n,), 2.0, device="cuda"); g = torch.ones(n, device="cuda")
    found = torch.ones(1, dtype=torch.int32, device="cuda")
    assert _call(p, v, g, [(0, n, 0.1, 0.0, 0.9, 0)], found=found) == 0
    assert float(p.min()) == 1.0 and float(v.min()) == 2.0 and float(g.abs().max()) == 0.0
    found.zero_(); g.fill_(1.0)
    assert _call(p, v, g, [(0, n, 0.1, 0.0, 0.9, 0)], found=found, flags=0) == 0
    assert float(p.max()) == pytest.approx(1.0 - 0.1 * 2.8) and float(g.min()) == 1.0
    pe, (ve,), _, _, _ = rp.step("sgd", np.ones(n, np.float32), [np.full(n, 2.0, np.float32)], np.ones(n, np.float32), None,
                                 [dict(begin=0, end=n, lr=0.1, wd=0.0, mu=0.9, flags=0)], zero_grad=False)
    assert np.array_equal(p.cpu().numpy(), pe) and np.array_equal(v.cpu().numpy(), ve)


def test_grad_nonfinite():
    from distributed_sod_project_b200 import _lib
    g = torch.zeros(1 << 20, device="cuda"); f = torch.zeros(1, dtype=torch.int32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert _lib.lib().sod_grad_nonfinite(g.data_ptr(), g.numel(), f.data_ptr(), s) == 0
    assert int(f.item()) == 0
    g[777_777] = float("nan")
    assert _lib.lib().sod_grad_nonfinite(g.data_ptr(), g.numel(), f.data_ptr(), s) == 0
    assert int(f.item()) == 1


def test_argument_contract():
    from distributed_sod_project_b200 import _lib
    p = torch.zeros(64, device="cuda")
    assert _call(p, p.clone(), p.clone(), [(0, 62, 0.1, 0, 0.9, 0)]) == -2          # SOD_EALIGN
    assert _call(p, p.clone(), p.clone(), [(32, 64, 0.1, 0, 0.9, 0), (0, 32, 0.1, 0, 0.9, 0)]) == -1   # unsorted
    assert b"aligned" in _lib.lib().sod_strerror(-2)


class _Tiny(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.div_2 = torch.nn.Linear(5, 7); self.div_4 = torch.nn.Linear(7, 6)
        self.div_16 = torch.nn.Linear(6, 3, bias=False); self.head = torch.nn.Linear(3, 2)
        self.classifier = torch.nn.Linear(2, 1)


@pytest.mark.parametrize("kind", ["f3_trick", "sgd_trick", "sgd_all"])
def test_fused_optimizer_follows_reference_trajectory(golden, kind):
    """FusedSGD built by OUR make_optimizer vs parameters produced by the reference's make_optimizer +
    torch.optim.SGD + CustomScheduler(poly) over 4 steps (tests/golden/sgd_kat.npz)."""
    from distributed_sod_project_b200.optim import CustomScheduler, make_optimizer
    g = golden("sgd_kat.npz")
    net = _Tiny().cuda()
    flat0 = torch.tensor(g[f"{kind}/p0"], device="cuda")
    off = 0
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(flat0[off:off + p.numel()].view_as(p)); off += p.numel()
    opt = make_optimizer(net, kind, dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    sched = CustomScheduler(opt, total_num=4, scheduler_type="poly", scheduler_info=dict(lr_decay=0.9, warmup_epoch=1))
    for it in range(4):
        sched.step(opt, curr_epoch=it)
        np.testing.assert_allclose([gr["lr"] for gr in opt.param_groups], g[f"{kind}/lr{it}"], rtol=1e-12)
        opt.zero_grad()
        gflat = torch.tensor(g[f"{kind}/g{it}"], device="cuda"); off = 0
        for p in net.parameters():
            p.grad.copy_(gflat[off:off + p.numel()].view_as(p)); off += p.numel()
        opt.step()
        got = torch.cat([p.detach().reshape(-1) for p in net.parameters()]).cpu().numpy()
        np.testing.assert_allclose(got, g[f"{kind}/p{it + 1}"], rtol=3e-6, atol=2e-7)
    # state_dict round trip keeps torch.optim.SGD's layout
    sd = opt.state_dict()
    assert all("momentum_buffer" in s for s in sd["state"].values()) and len(sd["state"]) == sum(len(gr["params"]) for gr in sd["param_groups"])
    net2 = _Tiny().cuda(); net2.load_state_dict(net.state_dict())
    opt2 = make_optimizer(net2, kind, dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    opt2.load_state_dict(sd)
    assert torch.equal(opt2.flat.mom, opt.flat.mom)
    assert "FusedSGD" in str(opt)


def test_learning_rate_table_on_the_device_overrides_the_segment_values():
    """ABI v6: with `lr_dev` the kernel reads each segment's learning rate from device memory at execution time — a
    captured CUDA graph then follows CustomScheduler (reference utils/pipeline_ops.py:225-229) without re-capture."""
    n = 8192
    p0 = torch.linspace(-1, 1, n, device="cuda"); g0 = torch.full((n,), 0.5, device="cuda")
    spec = [(0, n // 2, 123.0, 0.0, 0.0, 0), (n // 2, n, 456.0, 0.0, 0.0, 0)]     # by-value lrs must be ignored
    lr = torch.tensor([0.1, 0.01] + [0.0] * 14, device="cuda")
    p, v, g = p0.clone(), torch.zeros(n, device="cuda"), g0.clone()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        assert _call(p, v, g, spec, flags=0, lr_dev=lr) == 0        # warm-up launch
        p.copy_(p0); v.zero_()
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=s):
            from distributed_sod_project_b200 import _lib
            rc = _lib.lib().sod_sgd_momentum(p.data_ptr(), v.data_ptr(), g.data_ptr(), None, None, n, _segs(spec), 2, lr.data_ptr(),
                                             1.0, None, 0, torch.cuda.current_stream().cuda_stream)
            assert rc == 0
    graph.replay(); torch.cuda.synchronize()
    want = p0.clone(); want[:n // 2] -= 0.1 * 0.5; want[n // 2:] -= 0.01 * 0.5
    assert torch.allclose(p, want, rtol=0, atol=1e-6)
    lr[0].fill_(0.2); lr[1].fill_(0.0)                                # the scheduler moved: same graph, new rates
    p.copy_(p0); v.zero_()
    graph.replay(); torch.cuda.synchronize()
    want = p0.clone(); want[:n // 2] -= 0.2 * 0.5
    assert torch.allclose(p, want, rtol=0, atol=1e-6)


def test_multi_tensor_gather_of_bf16_gradients():
    """sod_grad_gather16: scattered dense bf16 tensors → their slots of the flat bf16 gradient buffer, bit-exact, incl.
    sizes that are not multiples of 8, a misaligned source and more items than one launch carries."""
    from distributed_sod_project_b200 import _lib
    g = torch.Generator().manual_seed(3)
    sizes = [1, 7, 8, 64, 4097, 8192, 8193, 147456, 2359296 + 3] + [33] * 170
    flat_n = sum((s + 63) // 64 * 64 for s in sizes) + 64
    flat = torch.full((flat_n,), -7.0, dtype=torch.bfloat16, device="cuda")
    srcs, items, off = [], [], 64
    for i, sz in enumerate(sizes):
        t = torch.randn(sz + 1, generator=g).to(torch.bfloat16).cuda()
        t = t[1:] if i % 5 == 4 else t[:sz]                  # every fifth source starts 2 bytes off a 16-byte boundary
        srcs.append(t)
        items.append(_lib.sod_gather_item(t.data_ptr(), off, sz))
        off += (sz + 63) // 64 * 64
    arr = (_lib.sod_gather_item * len(items))(*items)
    rc = _lib.lib().sod_grad_gather16(arr, len(items), flat.data_ptr(), flat_n, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    off = 64
    for t, sz in zip(srcs, sizes):
        assert torch.equal(flat[off:off + sz], t), sz
        pad = (sz + 63) // 64 * 64
        assert bool((flat[off + sz:off + pad] == -7.0).all())           # nothing written outside the item
        off += pad
    bad = (_lib.sod_gather_item * 1)(_lib.sod_gather_item(srcs[0].data_ptr(), 4, 1))
    assert _lib.lib().sod_grad_gather16(bad, 1, flat.data_ptr(), flat_n, torch.cuda.current_stream().cuda_stream) == -2


def test_bf16_only_gradient_segments():
    """SOD_SEG_GRAD16 (ABI v7): in such a range the gradient is taken from the bf16 buffer alone — the fp32 buffer is neither
    read (garbage there must not matter) nor cleared; other ranges keep adding both buffers."""
    from distributed_sod_project_b200 import _lib
    n = 4096 + 64
    a = 2048
    g = torch.Generator().manual_seed(9)
    p0 = torch.randn(n, generator=g).cuda(); v0 = torch.randn(n, generator=g).cuda()
    g32 = torch.randn(n, generator=g).cuda(); g16 = torch.randn(n, generator=g).to(torch.bfloat16).cuda()
    p, v, gg, hh = p0.clone(), v0.clone(), g32.clone(), g16.clone()
    shadow = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
    segs = (_lib.sod_sgd_segment * 2)(_lib.sod_sgd_segment(0, a, 0.1, 5e-4, 0.9, _lib.SOD_SEG_GRAD16), _lib.sod_sgd_segment(a, n, 0.01, 0.0, 0.9, 0))
    rc = _lib.lib().sod_sgd_momentum(p.data_ptr(), v.data_ptr(), gg.data_ptr(), hh.data_ptr(), shadow.data_ptr(), n, segs, 2, None, 1.0, None,
                                     _lib.SOD_SGD_ZERO_GRAD, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    eff = torch.cat([g16[:a].float(), g32[a:] + g16[a:].float()])
    wd = torch.cat([torch.full((a,), 5e-4), torch.zeros(n - a)]).cuda(); lr = torch.cat([torch.full((a,), 0.1), torch.full((n - a,), 0.01)]).cuda()
    ev = 0.9 * v0 + (eff + wd * p0)
    ep = p0 - lr * ev
    assert torch.allclose(v, ev, rtol=3e-6, atol=1e-6) and torch.allclose(p, ep, rtol=3e-6, atol=1e-6)
    assert torch.equal(gg[:a], g32[:a]) and float(gg[a:].abs().max()) == 0.0          # fp32 buffer untouched in the bf16-only range
    assert float(hh.float().abs().max()) == 0.0
    assert torch.equal(shadow, p.to(torch.bfloat16))
