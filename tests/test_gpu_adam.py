"""The fused Adam step (`sod_adam`, csrc/sgd.cu) against the Adam oracle and the reference optimizer's golden
trajectory, its device step counter under amp overflow skips and CUDA-graph replay, Nesterov SGD against the reference,
and the `Trainer` with optim "adam" end to end."""
import numpy as np
import pytest
import torch

from oracle import adam as oadam
from oracle import optim_replay as rp

pytestmark = pytest.mark.gpu

B1, B2, EPS = 0.9, 0.999, 1e-8


def _segs(spec):
    from distributed_sod_project_b200 import _lib
    arr = (_lib.sod_adam_segment * len(spec))()
    for i, (b, e, lr, wd, fl) in enumerate(spec):
        arr[i] = _lib.sod_adam_segment(b, e, lr, wd, B1, B2, EPS, fl)
    return arr


def _call(p, m, v, g, spec, step_dev, g16=None, shadow=None, inv_scale=1.0, found=None, flags=1, lr_dev=None):
    from distributed_sod_project_b200 import _lib
    ptr = lambda t: t.data_ptr() if t is not None else None       # noqa: E731
    return _lib.lib().sod_adam(p.data_ptr(), m.data_ptr(), v.data_ptr(), g.data_ptr(), ptr(g16), ptr(shadow), p.numel(),
                               _segs(spec), len(spec), ptr(lr_dev), step_dev.data_ptr(), inv_scale, ptr(found), flags,
                               torch.cuda.current_stream().cuda_stream)


def _steps(counts):
    from distributed_sod_project_b200 import _lib
    t = torch.zeros(_lib.SOD_ADAM_STEP_WORDS, dtype=torch.int32, device="cuda")
    t[:len(counts)] = torch.tensor(counts, dtype=torch.int32)
    return t


@pytest.mark.parametrize("n", [4, 64, 4096 + 64, 1_000_000 + 4, 24_912_000])
def test_flat_kernel_vs_oracle(n):
    """three segments — bf16-only gradient (SOD_SEG_GRAD16), fp32 + bf16 gradient, frozen — with different step counts"""
    from distributed_sod_project_b200 import _lib
    rng = np.random.default_rng(n)
    p0 = rng.standard_normal(n).astype(np.float32)
    m0 = (0.1 * rng.standard_normal(n)).astype(np.float32)
    v0 = (0.01 * np.abs(rng.standard_normal(n)) + 1e-4).astype(np.float32)
    g32 = rng.standard_normal(n).astype(np.float32)
    g16 = torch.tensor(rng.standard_normal(n).astype(np.float32)).to(torch.bfloat16)
    a = (n // 3) // 4 * 4; b = (2 * n // 3) // 4 * 4
    spec = [(0, a, 1e-3, 5e-4, _lib.SOD_SEG_GRAD16), (a, b, 3e-3, 0.0, 0), (b, n, 0.0, 0.0, _lib.SOD_SEG_FROZEN)]
    segs = [oadam.Segment(0, a, 1e-3, 5e-4, B1, B2, EPS), oadam.Segment(a, b, 3e-3, 0.0, B1, B2, EPS),
            oadam.Segment(b, n, 0.0, 0.0, frozen=True)]
    p, m, v, g = (torch.tensor(t, device="cuda") for t in (p0, m0, v0, g32))
    h = g16.cuda()
    shadow = p.to(torch.bfloat16)
    step_dev = _steps([0, 6, 9])
    assert _call(p, m, v, g, spec, step_dev, g16=h, shadow=shadow, inv_scale=0.5) == 0
    torch.cuda.synchronize()
    eff = np.concatenate([g16[:a].float().numpy(), g32[a:] + g16[a:].float().numpy()])   # what the kernel must consume
    pe, me, ve, steps = p0.copy(), m0.copy(), v0.copy(), [0, 6, 9]
    assert oadam.adam_step(pe, me, ve, eff, segs, steps, inv_scale=0.5)
    assert step_dev.tolist()[:4] == steps + [0] == [1, 7, 9, 0]         # frozen count kept; ticket re-armed
    got = p.cpu().numpy()
    # the kernel's own operation order, FMAs included (oracle/optim_replay.py): bit for bit
    table = [dict(begin=s[0], end=s[1], lr=s[2], wd=s[3], beta1=B1, beta2=B2, eps=EPS, flags=s[4]) for s in spec]
    rpe, (rme, rve), _, _, _ = rp.step("adam", p0, [m0, v0], g32, g16.float().numpy(), table, inv_scale=0.5, steps=[0, 6, 9])
    for x, w in ((got, rpe), (m.cpu().numpy(), rme), (v.cpu().numpy(), rve)):
        np.testing.assert_array_equal(x.view(np.uint32), w.view(np.uint32))
    np.testing.assert_array_equal(got[b:], p0[b:])                      # frozen range untouched, bit for bit
    np.testing.assert_array_equal(m.cpu().numpy()[b:], m0[b:])
    np.testing.assert_array_equal(v.cpu().numpy()[b:], v0[b:])
    p64, _, _, _ = oadam.adam_step_f64(p0, m0, v0, eff, segs, [0, 6, 9], inv_scale=0.5)
    np.testing.assert_allclose(got, p64, rtol=1e-5, atol=1e-6)
    gc = g.cpu().numpy()
    np.testing.assert_array_equal(gc[:a], g32[:a])                      # GRAD16 range: fp32 buffer neither read nor cleared
    assert (n - a == 0) or float(np.abs(gc[a:]).max()) == 0.0
    assert float(h.float().abs().max()) == 0.0
    assert torch.equal(shadow, p.to(torch.bfloat16))


def test_overflow_skip_keeps_state_and_step_and_clears_grads():
    n = 4096
    p0 = torch.linspace(-1, 1, n, device="cuda")
    p, m, v = p0.clone(), torch.full((n,), 0.5, device="cuda"), torch.full((n,), 2.0, device="cuda")
    g = torch.ones(n, device="cuda")
    step_dev = _steps([0])
    found = torch.ones(1, dtype=torch.int32, device="cuda")
    assert _call(p, m, v, g, [(0, n, 0.1, 0.0, 0)], step_dev, found=found) == 0
    torch.cuda.synchronize()
    assert torch.equal(p, p0) and float(m.min()) == float(m.max()) == 0.5 and float(v.min()) == float(v.max()) == 2.0
    assert float(g.abs().max()) == 0.0 and step_dev.tolist()[:2] == [0, 0]
    # the next clean step is step 1 (bias correction with t = 1)
    found.zero_(); g.fill_(1.0); m.zero_(); v.zero_()
    assert _call(p, m, v, g, [(0, n, 0.1, 0.0, 0)], step_dev, found=found, flags=0) == 0
    torch.cuda.synchronize()
    assert step_dev.tolist()[:2] == [1, 0] and float(g.min()) == 1.0
    pe, me, ve, st = p0.cpu().numpy().copy(), np.zeros(n, np.float32), np.zeros(n, np.float32), [0]
    assert oadam.adam_step(pe, me, ve, np.ones(n, np.float32), [oadam.Segment(0, n, 0.1, 0.0, B1, B2, EPS)], st)
    np.testing.assert_allclose(p.cpu().numpy(), pe, rtol=3e-6, atol=1e-6)
    rpe, _, _, _, _ = rp.step("adam", p0.cpu().numpy(), [np.zeros(n, np.float32)] * 2, np.ones(n, np.float32), None,
                              [dict(begin=0, end=n, lr=0.1, wd=0.0, beta1=B1, beta2=B2, eps=EPS, flags=0)], zero_grad=False,
                              steps=[0])
    np.testing.assert_array_equal(p.cpu().numpy().view(np.uint32), rpe.view(np.uint32))
    assert float((p0 - p).min()) == pytest.approx(0.1, rel=1e-5)              # t = 1: the first Adam step moves by ≈ lr


def test_graph_replay_follows_the_device_step_count_and_learning_rate():
    """captured once, replayed three times: the three eager steps, bias corrections at t = 1, 2, 3 included; a new
    learning rate in the device table takes effect without re-capture"""
    n = 8192
    gen = torch.Generator().manual_seed(4)
    p0 = torch.randn(n, generator=gen).cuda(); g0 = torch.randn(n, generator=gen).cuda()
    spec = [(0, n // 2, 123.0, 5e-4, 0), (n // 2, n, 456.0, 0.0, 0)]        # by-value lrs must be ignored
    lr = torch.zeros(16, device="cuda"); lr[0], lr[1] = 1e-2, 1e-3

    eager = []
    p, m, v = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    step_dev = _steps([0, 0])
    for _ in range(3):
        assert _call(p, m, v, g0.clone(), spec, step_dev, flags=0, lr_dev=lr) == 0
        eager.append((p.clone(), m.clone(), v.clone()))
    assert step_dev.tolist()[:2] == [3, 3]

    p, m, v, g = p0.clone(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), g0.clone()
    step_dev = _steps([0, 0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        assert _call(p, m, v, g, spec, step_dev, flags=0, lr_dev=lr) == 0         # warm-up launch
        p.copy_(p0); m.zero_(); v.zero_(); step_dev.zero_()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        assert _call(p, m, v, g, spec, step_dev, flags=0, lr_dev=lr) == 0
    for k in range(3):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(p, eager[k][0]) and torch.equal(m, eager[k][1]) and torch.equal(v, eager[k][2]), k
    assert step_dev.tolist()[:2] == [3, 3]
    # the scheduler moved: same graph, new rate (segment 1 frozen at lr 0 this time)
    lr[0].fill_(2e-2); lr[1].fill_(0.0)
    before = p.clone()
    graph.replay(); torch.cuda.synchronize()
    pe, me, ve, st = before.cpu().numpy().copy(), eager[2][1].cpu().numpy().copy(), eager[2][2].cpu().numpy().copy(), [3, 3]
    segs = [oadam.Segment(0, n // 2, 2e-2, 5e-4, B1, B2, EPS), oadam.Segment(n // 2, n, 0.0, 0.0, B1, B2, EPS)]
    assert oadam.adam_step(pe, me, ve, g0.cpu().numpy(), segs, st)
    np.testing.assert_allclose(p.cpu().numpy(), pe, rtol=3e-6, atol=1e-6)
    assert torch.equal(p[n // 2:], before[n // 2:]) and step_dev.tolist()[:2] == [4, 4]


def test_argument_contract():
    from distributed_sod_project_b200 import _lib
    p = torch.zeros(64, device="cuda")
    sd = _steps([0, 0])
    assert _call(p, p.clone(), p.clone(), p.clone(), [(0, 62, 0.1, 0, 0)], sd) == -2                       # SOD_EALIGN
    assert _call(p, p.clone(), p.clone(), p.clone(), [(32, 64, 0.1, 0, 0), (0, 32, 0.1, 0, 0)], sd) == -1   # unsorted
    assert _call(p, p.clone(), p.clone(), p.clone(), [(0, 64, 0.1, 0, _lib.SOD_SEG_NESTEROV)], sd) == -1  # SGD-only flag
    rc = _lib.lib().sod_adam(p.data_ptr(), p.data_ptr(), p.data_ptr(), p.data_ptr(), None, None, 64, _segs([(0, 64, 0.1, 0, 0)]),
                             1, None, None, 1.0, None, 0, torch.cuda.current_stream().cuda_stream)
    assert rc == -1                                                                                          # no step counter
    torch.cuda.synchronize()
    assert sd.tolist() == [0] * _lib.SOD_ADAM_STEP_WORDS


class _Tiny(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.div_2 = torch.nn.Linear(5, 7); self.div_4 = torch.nn.Linear(7, 6)
        self.div_16 = torch.nn.Linear(6, 3, bias=False); self.head = torch.nn.Linear(3, 2)
        self.classifier = torch.nn.Linear(2, 1)


@pytest.mark.parametrize("tag,kind,nesterov", [("adam", "adam", False), ("sgd_trick_nesterov", "sgd_trick", True),
                                                ("f3_trick_nesterov", "f3_trick", True)])
def test_fused_optimizer_follows_reference_trajectory(golden, tag, kind, nesterov):
    """FusedAdam / Nesterov FusedSGD built by OUR make_optimizer vs the reference's make_optimizer + torch optimizer +
    CustomScheduler(poly) over 4 steps (tests/golden/optim_ext_kat.npz)"""
    from distributed_sod_project_b200.optim import CustomScheduler, make_optimizer
    g = golden("optim_ext_kat.npz")
    net = _Tiny().cuda()
    flat0 = torch.tensor(g[f"{tag}/p0"], device="cuda")
    off = 0
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(flat0[off:off + p.numel()].view_as(p)); off += p.numel()
    info = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=nesterov)
    opt = make_optimizer(net, kind, info)
    sched = CustomScheduler(opt, total_num=4, scheduler_type="poly", scheduler_info=dict(lr_decay=0.9, warmup_epoch=1))
    for it in range(4):
        sched.step(opt, curr_epoch=it)
        np.testing.assert_allclose([gr["lr"] for gr in opt.param_groups], g[f"{tag}/lr{it}"], rtol=1e-12)
        opt.zero_grad()
        gflat = torch.tensor(g[f"{tag}/g{it}"], device="cuda"); off = 0
        for p in net.parameters():
            p.grad.copy_(gflat[off:off + p.numel()].view_as(p)); off += p.numel()
        opt.step()
        got = torch.cat([p.detach().reshape(-1) for p in net.parameters()]).cpu().numpy()
        np.testing.assert_allclose(got, g[f"{tag}/p{it + 1}"], rtol=3e-6, atol=2e-7)
    if kind != "adam":
        return
    assert opt.group_steps() == [4]
    sd = opt.state_dict()
    st = [sd["state"][i] for i in range(len(g["adam/names"]))]
    np.testing.assert_array_equal([float(s["step"]) for s in st], g["adam/state_step"])
    np.testing.assert_allclose(torch.cat([s["exp_avg"].reshape(-1) for s in st]).cpu().numpy(), g["adam/state_exp_avg"],
                               rtol=3e-6, atol=1e-8)
    np.testing.assert_allclose(torch.cat([s["exp_avg_sq"].reshape(-1) for s in st]).cpu().numpy(),
                               g["adam/state_exp_avg_sq"], rtol=3e-6, atol=1e-12)
    # round trip into a fresh optimizer
    net2 = _Tiny().cuda(); net2.load_state_dict(net.state_dict())
    opt2 = make_optimizer(net2, kind, info)
    opt2.load_state_dict(sd)
    assert torch.equal(opt2.flat.mom, opt.flat.mom) and torch.equal(opt2.exp_avg_sq, opt.exp_avg_sq)
    assert opt2.group_steps() == [4]


def _trainer(**kw):
    from distributed_sod_project_b200.engine import Trainer
    return Trainer(model_name="res50", lr=1e-4, momentum=0.9, weight_decay=5e-4, optim="adam", channels_last=True,
                   report_items=False, **kw)


def test_trainer_adam_captures_a_graph_with_shadow_weights():
    from distributed_sod_project_b200.optim import FusedAdam
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(dtype=torch.bfloat16, use_graph=True)
    assert isinstance(tr.optimizer, FusedAdam) and tr.use_graph
    flat = tr.optimizer.flat
    assert flat.shadow16 is not None and len(flat.shadow_leaves) > 0        # bf16 shadow weights installed
    p0 = flat.param.clone()
    for it in range(3):
        x, m = synth_batch(700 + it, 2, 64)
        red, _, _ = tr.forward_backward_update(x.cuda(), m.cuda())
        assert np.isfinite(float(red))
    assert len(tr._graphs) >= 1
    assert tr.optimizer.group_steps() == [3] and tr.optimizer.steps == 3
    assert not torch.equal(p0, flat.param)
    assert torch.equal(flat.shadow16, flat.param.to(torch.bfloat16))


def test_adam_graph_follows_the_scheduler_like_the_eager_run():
    """multi-scale batches with a per-iteration schedule: one captured graph per input size reproduces the eager Adam run
    (tolerances of test_gpu_step.py's SGD version of this test)"""
    from distributed_sod_project_b200.synthetic import synth_batch
    sizes = [64, 96, 64, 128, 96, 64, 128]
    runs = {}
    for use_graph in (False, True):
        tr = _trainer(dtype=torch.bfloat16, use_graph=use_graph)
        sched = tr.scheduler(total_num=len(sizes), lr_type="poly")
        losses = []
        for it, size in enumerate(sizes):
            sched.step(tr.optimizer, curr_epoch=it)
            x, m = synth_batch(500 + it, 4, size)
            red, _, _ = tr.forward_backward_update(x.cuda(), m.cuda())
            losses.append(float(red))
        runs[use_graph] = (losses, tr.optimizer.steps, tr.optimizer.group_steps())
        if use_graph:
            assert len(tr._graphs) == 3
    assert runs[True][1] == runs[False][1] == len(sizes)
    assert runs[True][2] == runs[False][2] == [len(sizes)]
    assert runs[True][0][:2] == pytest.approx(runs[False][0][:2], rel=2e-3)
    assert runs[True][0] == pytest.approx(runs[False][0], rel=5e-2)


def test_fp16_adam_overflow_skip_halve_recover():
    """fp16 amp with optim "adam": an overflowing scale skips the update (parameters, both moments and the step count
    unchanged, gradients cleared) and halves the scale until it fits; the step count advances on clean steps only"""
    from distributed_sod_project_b200 import amp
    from distributed_sod_project_b200.synthetic import synth_batch
    tr = _trainer(dtype=torch.float16)
    assert amp._cfg["dynamic"] and not tr.use_graph
    amp._cfg["scale"] = 2.0 ** 40
    opt, flat = tr.optimizer, tr.optimizer.flat
    history = []
    try:
        for it in range(40):
            scale = amp._cfg["scale"]
            p0, m0, v0, t0 = flat.param.clone(), flat.mom.clone(), opt.exp_avg_sq.clone(), opt.group_steps()[0]
            x, m = synth_batch(3000 + it, 2, 64)
            red, _, _ = tr.forward_backward_update(x.cuda(), m.cuda())
            skipped = bool(int(opt.found_inf.item()))
            history.append(skipped)
            assert float(flat.grad.abs().max()) == 0.0
            if skipped:
                assert torch.equal(p0, flat.param) and torch.equal(m0, flat.mom) and torch.equal(v0, opt.exp_avg_sq)
                assert opt.group_steps()[0] == t0 and amp._cfg["scale"] == scale / 2
            else:
                assert not torch.equal(p0, flat.param) and np.isfinite(float(red))
                assert opt.group_steps()[0] == t0 + 1
            if sum(1 for s in history if not s) >= 3:
                break
    finally:
        amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, found_inf=None)
    assert history[0] and not history[-1]
    first_ok = history.index(False)
    assert all(history[:first_ok])
    assert opt.group_steps()[0] == sum(1 for s in history if not s)
