"""fp16 mixed precision (apex amp O1, reference train.py:183,299) on the device: fp16 gradient and shadow buffers in the step
kernels, the device-resident dynamic loss scaler, the overflow checks folded into the gradient gather, the loss gradient
scaled before it is rounded, and the Trainer on CUDA graphs.

Oracles: the fp64 step of oracle/sgd.py and oracle/adam.py (the tolerance of tests/test_gpu_virtual_world.py: 1e-5 of
|p| + |Δp|), the same kernel on the fp32 gradient (bit for bit: both call the same update on the same operands), a host
model of the scaler's rules, and the fp64 loss gradient with the bounds derived in tests/test_gpu_loss_regimes.py."""
import os

import numpy as np
import pytest
import torch

from oracle import adam as oadam
from oracle import sgd as osgd

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def L():
    from distributed_sod_project_b200 import _lib
    return _lib.lib()


def lib():
    from distributed_sod_project_b200 import _lib
    return _lib


def sp():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return t.data_ptr() if t is not None else None


def bits(t):
    return t.detach().contiguous().cpu().view(torch.int32 if t.element_size() == 4 else torch.int16)


def scaler_dev(scale, growth_interval, unskipped=0, found=0):
    s = torch.zeros(lib().SOD_LOSS_SCALER_WORDS, dtype=torch.int32)
    s[0], s[2], s[3] = found, unskipped, growth_interval
    s.view(torch.float32)[1] = scale
    return s.cuda()


def scaler_state(s):
    w = s.cpu()
    return float(w.view(torch.float32)[1]), int(w[2]), int(w[0]), int(w[4])


def model_step(scale, unskipped, gi, overflow):
    """the rules the device scaler must follow (apex O1 dynamic scaling as amp.py applied them on the host)"""
    if overflow:
        return max(scale / 2.0, 1.0), 0
    unskipped += 1
    return (scale * 2.0 if unskipped % gi == 0 else scale), unskipped


# -- segments: [GRAD16 | fp32 | frozen | fp32]; sizes not multiples of the CTA tile ------------------------------------
def layout(n):
    q = (n // 16) * 4
    return [(0, 2 * q, "g16"), (2 * q, 3 * q, "f32"), (3 * q, 3 * q + 64, "frozen"), (3 * q + 64, n, "f32")]


def sgd_segs(n, nesterov=False):
    l = lib()
    out = []
    for i, (b, e, kind) in enumerate(layout(n)):
        f = (l.SOD_SEG_GRAD16 if kind == "g16" else 0) | (l.SOD_SEG_FROZEN if kind == "frozen" else 0)
        if nesterov and i % 2 == 0:
            f |= l.SOD_SEG_NESTEROV
        out.append(l.sod_sgd_segment(b, e, (0.05, 0.01, 0.0, 0.2)[i], (5e-4, 0.0, 0.0, 1e-2)[i], (0.9, 0.5, 0.0, 0.9)[i], f))
    return (l.sod_sgd_segment * len(out))(*out)


def adam_segs(n):
    l = lib()
    out = []
    for i, (b, e, kind) in enumerate(layout(n)):
        f = (l.SOD_SEG_GRAD16 if kind == "g16" else 0) | (l.SOD_SEG_FROZEN if kind == "frozen" else 0)
        out.append(l.sod_adam_segment(b, e, (1e-3, 5e-3, 0.0, 2e-3)[i], (5e-4, 0.0, 0.0, 1e-2)[i], 0.9, 0.999, 1e-8, f))
    return (l.sod_adam_segment * len(out))(*out)


def oracle_segments(rule, n, nesterov=False):
    segs = sgd_segs(n, nesterov) if rule != "adam" else adam_segs(n)
    out = []
    for s in segs:
        fz = bool(s.flags & lib().SOD_SEG_FROZEN)
        f32 = lambda v: float(np.float32(v))                      # noqa: E731
        if rule == "adam":
            out.append(oadam.Segment(s.begin, s.end, f32(s.lr), f32(s.weight_decay), 0.9, 0.999, f32(s.eps), fz))
        else:
            out.append(osgd.Segment(s.begin, s.end, f32(s.lr), f32(s.weight_decay), f32(s.momentum), fz,
                                    bool(s.flags & lib().SOD_SEG_NESTEROV)))
    return out


class Buffers:
    """flat fp32 state + 16-bit gradient/shadow buffers of one run"""

    def __init__(self, rule, p0, st0, g32, g16, dt16, step0=None):
        self.rule = rule
        self.p = torch.from_numpy(p0).cuda()
        self.st = [torch.from_numpy(s).cuda() for s in st0]
        self.g = torch.from_numpy(g32).cuda()
        self.g16 = g16.cuda() if g16 is not None else None
        n = p0.size
        self.sh = torch.full((n,), 0x7BFF if dt16 == torch.float16 else 0x7F7F, dtype=torch.int16).view(dt16).cuda()
        self.steps = torch.from_numpy(step0 if step0 is not None else np.zeros(lib().SOD_ADAM_STEP_WORDS, np.int32)).cuda()
        self.flags = lib().SOD_SGD_ZERO_GRAD | (lib().SOD_GRAD16_F16 if dt16 == torch.float16 else 0)

    def step(self, inv_scale=1.0, found=None, scaler=None, nesterov=False, use16=True, shadow=True):
        n = self.p.numel()
        g16, sh = (ptr(self.g16) if use16 else None), (ptr(self.sh) if shadow else None)
        if self.rule == "adam":
            segs = adam_segs(n)
            if scaler is not None:
                return L().sod_adam_scaler(ptr(self.p), ptr(self.st[0]), ptr(self.st[1]), ptr(self.g), g16, sh, n, segs,
                                           len(segs), None, ptr(self.steps), ptr(scaler), self.flags, sp())
            return L().sod_adam(ptr(self.p), ptr(self.st[0]), ptr(self.st[1]), ptr(self.g), g16, sh, n, segs, len(segs), None,
                                ptr(self.steps), inv_scale, ptr(found), self.flags, sp())
        segs = sgd_segs(n, nesterov)
        if scaler is not None:
            return L().sod_sgd_momentum_scaler(ptr(self.p), ptr(self.st[0]), ptr(self.g), g16, sh, n, segs, len(segs), None,
                                               ptr(scaler), self.flags, sp())
        return L().sod_sgd_momentum(ptr(self.p), ptr(self.st[0]), ptr(self.g), g16, sh, n, segs, len(segs), None, inv_scale,
                                    ptr(found), self.flags, sp())


def inputs(rule, n, seed, g16_dtype=torch.float16, both_formats=False):
    rng = np.random.default_rng(seed)
    p0 = (rng.standard_normal(n) * np.exp2(rng.integers(-3, 3, n))).astype(np.float32)
    st0 = [(rng.standard_normal(n) * 0.1).astype(np.float32)]
    if rule == "adam":
        st0.append(np.abs(rng.standard_normal(n) * 1e-4).astype(np.float32))
    g32 = (rng.standard_normal(n) * np.exp2(rng.integers(-6, 2, n))).astype(np.float32)
    if both_formats:          # k·2^-e with |k| < 256: exact in bf16 and in fp16
        g16 = torch.from_numpy((rng.integers(-255, 256, n) * np.exp2(-rng.integers(6, 12, n))).astype(np.float32))
    else:
        g16 = torch.from_numpy((rng.standard_normal(n) * np.exp2(rng.integers(-8, 4, n))).astype(np.float32))
    return p0, st0, g32, g16.to(g16_dtype)


def effective_grad(n, g32, g16):
    """what the world-1 kernel feeds the rule: grad16 alone in GRAD16 ranges, grad + grad16 elsewhere"""
    h = g16.float().numpy()
    g = g32 + h
    for b, e, kind in layout(n):
        if kind == "g16":
            g[b:e] = h[b:e]
    return g


# ---------------------------------------------------------------------------------------------------------------------
# 1. step kernels with fp16 grad16 / shadow16
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rule", ["sgd", "nesterov", "adam"])
@pytest.mark.parametrize("n", [4 * 1021, 4 * 98317])
def test_fp16_buffers_step_matches_fp32_step_and_fp64_oracle(rule, n):
    nest = rule == "nesterov"
    r = "adam" if rule == "adam" else "sgd"
    p0, st0, g32, g16 = inputs(r, n, n + len(rule))
    inv = 0.5
    a = Buffers(r, p0, st0, g32, g16, torch.float16)
    assert a.step(inv_scale=inv, nesterov=nest) == 0
    geff = effective_grad(n, g32, g16)
    # the same kernel, fp32 gradient only, no 16-bit buffers: the same update on the same operands
    b = Buffers(r, p0, st0, geff, None, torch.float16)
    b.flags = lib().SOD_SGD_ZERO_GRAD
    assert b.step(inv_scale=inv, nesterov=nest, use16=False, shadow=False) == 0
    torch.cuda.synchronize()
    assert torch.equal(bits(a.p), bits(b.p))
    for x, y in zip(a.st, b.st):
        assert torch.equal(bits(x), bits(y))
    # shadow: round-to-nearest of every updated parameter, = param.half(); untouched where frozen
    upd = torch.ones(n, dtype=torch.bool)
    for bb, e, kind in layout(n):
        if kind == "frozen":
            upd[bb:e] = False
    sh = bits(a.sh)
    assert torch.equal(sh[upd], bits(a.p.half())[upd])
    assert bool((sh[~upd] == 0x7BFF).all())
    # gradients cleared: fp32 outside GRAD16 ranges, grad16 everywhere
    assert not a.g16.float().any()
    g = a.g.cpu().numpy()
    for bb, e, kind in layout(n):
        if kind == "g16":
            assert np.array_equal(g[bb:e], g32[bb:e])
        else:
            assert not g[bb:e].any()
    # fp64 oracle
    segs = oracle_segments(rule, n, nest)
    if r == "adam":
        p64, *_ = oadam.adam_step_f64(p0, st0[0], st0[1], geff, segs, [0] * len(segs), inv_scale=inv)
    else:
        p64, _ = osgd.sgd_step_f64(p0, st0[0], geff, segs, inv_scale=inv)
    pg = a.p.double().cpu().numpy()
    tol = 1e-5 * (np.abs(p64) + np.abs(p64 - p0)) + 1e-30
    assert bool((np.abs(pg - p64) <= tol).all())


@pytest.mark.parametrize("rule", ["sgd", "adam"])
def test_fp16_and_bf16_buffers_give_identical_parameters_on_common_values(rule):
    n = 4 * 5003
    p0, st0, g32, g16 = inputs(rule, n, 11, torch.float32, both_formats=True)
    runs = {}
    for dt in (torch.float16, torch.bfloat16):
        assert torch.equal(g16.to(dt).float(), g16)
        b = Buffers(rule, p0, st0, g32, g16.to(dt), dt)
        for _ in range(2):
            b.g16.copy_(g16.to(dt))
            assert b.step(inv_scale=0.25) == 0
        runs[dt] = b
    torch.cuda.synchronize()
    assert torch.equal(bits(runs[torch.float16].p), bits(runs[torch.bfloat16].p))
    for x, y in zip(runs[torch.float16].st, runs[torch.bfloat16].st):
        assert torch.equal(bits(x), bits(y))
    upd = torch.ones(n, dtype=torch.bool)
    for bb, e, kind in layout(n):
        upd[bb:e] = kind != "frozen"
    assert torch.equal(bits(runs[torch.float16].sh)[upd], bits(runs[torch.float16].p.half())[upd])
    assert torch.equal(bits(runs[torch.bfloat16].sh)[upd], bits(runs[torch.bfloat16].p.bfloat16())[upd])


def test_grad_merge16_fp16():
    n = 4 * 777
    g = torch.randn(n, device="cuda")
    h = torch.randn(n, device="cuda").half()
    h[: n // 2] = 0
    want = g + h.float()
    assert L().sod_grad_merge16(ptr(g), ptr(h), n, lib().SOD_GRAD16_F16, sp()) == 0
    torch.cuda.synchronize()
    assert torch.equal(g, want) and not h.float().any()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the scaler state machine
# ---------------------------------------------------------------------------------------------------------------------
PATTERN = [1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 1, 0, 0, 0]


@pytest.mark.parametrize("rule", ["sgd", "nesterov", "adam"])
def test_device_scaler_follows_the_rules_step_for_step(rule):
    """planted overflow flags: floor at 1 (scale 4 halves to 1 and stays), growth exactly at the interval, reset after an
    overflow; a skipped step leaves p, state and Adam's counts bit-identical; gradients are cleared either way; the step
    uses 1/scale read on the device (equal to the (inv_scale, found_inf) entry point with the host's 1/scale)"""
    n, gi = 4 * 3001, 3
    r = "adam" if rule == "adam" else "sgd"
    nest = rule == "nesterov"
    p0, st0, g32, g16 = inputs(r, n, 7)
    a = Buffers(r, p0, st0, g32, g16, torch.float16)
    b = Buffers(r, p0, st0, g32, g16, torch.float16)
    sc = scaler_dev(4.0, gi)
    scale, unsk = 4.0, 0
    for k, ov in enumerate(PATTERN):
        for x in (a, b):
            x.g.copy_(torch.from_numpy(g32 * (k + 1)))
            x.g16.copy_((g16.float() * (k + 1)).half())
        sc[0].fill_(ov)
        before = [bits(a.p)] + [bits(s) for s in a.st] + [a.steps.cpu().clone()]
        assert a.step(scaler=sc, nesterov=nest) == 0
        found = torch.tensor([ov], dtype=torch.int32, device="cuda")
        assert b.step(inv_scale=float(1.0 / scale), found=found, nesterov=nest) == 0
        torch.cuda.synchronize()
        scale, unsk = model_step(scale, unsk, gi, ov)
        got = scaler_state(sc)
        assert got == (scale, unsk, ov, 0), (k, got, scale, unsk)
        assert torch.equal(bits(a.p), bits(b.p)) and all(torch.equal(bits(x), bits(y)) for x, y in zip(a.st, b.st))
        assert torch.equal(a.steps, b.steps)
        if ov:
            after = [bits(a.p)] + [bits(s) for s in a.st] + [a.steps.cpu()]
            assert all(torch.equal(x, y) for x, y in zip(before, after))
        assert not a.g16.float().any()
    # the pattern reaches the floor, stays there on a further overflow, and grows
    hist, s, u = [], 4.0, 0
    for ov in PATTERN:
        s, u = model_step(s, u, gi, ov)
        hist.append(s)
    assert min(hist) == 1.0 and hist.count(1.0) >= 2 and max(hist) > 1.0


# ---------------------------------------------------------------------------------------------------------------------
# 3. overflow detection: checked gather and the range check
# ---------------------------------------------------------------------------------------------------------------------
BAD = [("+inf", float("inf")), ("-inf", float("-inf")), ("nan", float("nan")), ("max", 65504.0)]


def _gather(srcs, offs, dst, dtype):
    l = lib()
    items = (l.sod_gather_item * len(srcs))(*[l.sod_gather_item(s.data_ptr(), o, s.numel()) for s, o in zip(srcs, offs)])
    finf = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc = L().sod_grad_gather16_checked(items, len(srcs), ptr(dst), dst.numel(), l.dtype_code(dtype), ptr(finf), sp())
    assert rc == 0
    torch.cuda.synchronize()
    return int(finf.item())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("what,val", BAD, ids=[b[0] for b in BAD])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("aligned", [True, False])
def test_checked_gather_flags_nonfinite_wgrads(dtype, what, val, where, aligned):
    # a wgrad of 9·1000+5 elements (vector body + scalar tail) among others; unaligned: a source 2 bytes off 16
    sizes = [4096, 9005, 640]
    offs = [0, 4096, 4096 + 9008]
    store = torch.randn(sum(sizes) + 64, device="cuda").to(dtype) * 0.01
    srcs, o = [], 0 if aligned else 1
    for s in sizes:
        srcs.append(store[o:o + s])
        o += s + 16
    dst = torch.zeros(offs[-1] + sizes[-1] + 64, dtype=dtype, device="cuda")
    assert _gather(srcs, offs, dst, dtype) == 0
    t = srcs[1]
    t[0 if where == "first" else -1] = val
    flagged = _gather(srcs, offs, dst, dtype)
    assert flagged == (1 if what != "max" else 0)
    for s, off in zip(srcs, offs):
        assert torch.equal(dst[off:off + s.numel()].view(torch.int16), s.view(torch.int16))


@pytest.mark.parametrize("what,val", BAD, ids=[b[0] for b in BAD])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("buf", ["bias16", "gamma32"])
def test_range_check_flags_folded_bias_and_bn_gradients(what, val, where, buf):
    l = lib()
    n = 4 * 4096
    g = torch.randn(n, device="cuda") * 0.01
    h = (torch.randn(n, device="cuda") * 0.01).half()
    # a folded bias gradient of 37 words at 8256, a BN γ range of 4100 elements at 10000 (not chunk-aligned)
    ranges = [(8256, 8256 + 37, l.SOD_SEG_GRAD16), (10000, 14100, 0)]
    arr = (l.sod_check_range * 2)(*[l.sod_check_range(*r) for r in ranges])

    def check():
        f = torch.zeros(1, dtype=torch.int32, device="cuda")
        assert L().sod_grad_check_ranges(ptr(g), ptr(h), n, arr, 2, l.SOD_GRAD16_F16, ptr(f), sp()) == 0
        torch.cuda.synchronize()
        return int(f.item())
    assert check() == 0
    b, e, _ = ranges[0] if buf == "bias16" else ranges[1]
    i = b if where == "first" else e - 1
    (h if buf == "bias16" else g)[i] = val
    # just outside the ranges: never read
    g[9999] = float("inf")
    h[8256 + 37] = float("inf")
    assert check() == (0 if what == "max" else 1)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the loss gradient at the workload shape, scaled before rounding
# ---------------------------------------------------------------------------------------------------------------------
def test_loss_gradient_scaled_before_fp16_rounding_at_workload_shape():
    """fp16 logits 16×1×320² through the autograd path amp uses (`loss * scale_dev`, backward): every element within one
    fp16 ulp plus the fp32 slack of the fp64 gradient × scale.  The gradient of the unscaled loss is ≈ 1/n ≈ 6e-7, in fp16's
    subnormal range: rounding it first and scaling afterwards (what the engine did before the device loss scale) misses
    that bound, which the second half checks."""
    import test_gpu_loss_regimes as lr
    from distributed_sod_project_b200.loss import _FusedLossFn, bce_cel_fwd_bwd
    gen = torch.Generator(device="cuda").manual_seed(320)
    shape = (16, 1, 320, 320)
    x = (torch.randn(shape, generator=gen, device="cuda") * 3).half()
    t = (torch.rand(shape, generator=gen, device="cuda") > 0.7).float()
    scale = 65536.0
    sdev = torch.tensor(scale, dtype=torch.float32, device="cuda")
    xl = x.detach().requires_grad_(True)
    holder = []
    total = _FusedLossFn.apply(xl, t, "mean", 1.0, 1.0, 1e-6, False, 0, holder, sdev)
    (total * sdev).backward()
    torch.cuda.synchronize()
    r = lr.reference(x, t, "mean", 1.0, 1.0, scale, 1e-6)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sb = lr.scalar_bounds(r, -(-x.numel() // sms // 4096) + 1)
    tol = lr.ulp(r["grad"], torch.float16) + lr.grad_slack(r, sb["rel_den"], sb["rel_num"])
    assert xl.grad.dtype == torch.float16
    lr.assert_within(xl.grad.reshape(-1), r["grad"], tol, "scaled loss gradient")
    # the old order — round d total/d x to fp16, then multiply by the scale — is outside the same bound
    _, g1 = bce_cel_fwd_bwd(x, t)
    old = (g1.float() * scale).half().reshape(-1)
    assert bool(((old.double() - r["grad"]).abs() > tol).any())


# ---------------------------------------------------------------------------------------------------------------------
# 5-7. Trainer: fp16 on CUDA graphs, the deterministic net, checkpoints and the command line
# ---------------------------------------------------------------------------------------------------------------------
def _trainer(**kw):
    from distributed_sod_project_b200.engine import Trainer
    return Trainer(model_name="res50", lr=0.05, momentum=0.9, weight_decay=5e-4, dtype=torch.float16, channels_last=True,
                   report_items=False, **kw)


@pytest.fixture
def amp_reset():
    from distributed_sod_project_b200 import amp
    yield amp
    amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None, dev=None)


def _run_history(tr, batches, sync_free_from):
    """(scale before the step, skipped) per iteration and the losses.  From iteration `sync_free_from` on (None: never)
    the iterations run under torch.cuda.set_sync_debug_mode("error"): the scaler's words are copied on the device and
    read afterwards."""
    hist = torch.zeros(len(batches), 2, dtype=torch.int32, device="cuda")
    losses = torch.zeros(len(batches), device="cuda")
    s = tr.optimizer.flat.scaler
    try:
        for i, (x, m) in enumerate(batches):
            if i == sync_free_from:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode("error")
            hist[i, 0].copy_(s[1])                       # scale bits before the step
            red, _, _ = tr.forward_backward_update(x, m)
            hist[i, 1].copy_(s[0])                       # the verdict
            losses[i].copy_(red.reshape(()))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    h = hist.cpu()
    return [(float(v), bool(k)) for v, k in zip(h[:, 0].view(torch.float32).tolist(), h[:, 1].tolist())], losses.tolist()


def _follows_the_rules(h, gi, unskipped=0):
    scale = h[0][0]
    for (s0, k0), (s1, _) in zip(h, h[1:]):
        assert s0 == scale
        scale, unskipped = model_step(scale, unskipped, gi, k0)
        assert s1 == scale, (h, s1, scale)


def test_trainer_fp16_graph_multiscale_matches_eager_and_recovers_from_overflow(amp_reset):
    """use_graph stays on with fp16 (one graph per input size, three sizes).  Eager and graph runs on the same batches:

    1. from a forced 2^40 scale every step overflows, skips and halves until the gradients fit.  No run has changed its
       parameters until then, so the (scale, skipped) histories up to the first clean step, and the losses, agree.  After
       it the two trajectories drift apart like any two runs (cuDNN picks non-deterministic algorithms), and an overflow
       verdict right at the fp16 limit may differ: from there each run is held to the rules on its own.
    2. the scale set from the host to 2^6, far below the limit, with the count of clean steps reset: every step is clean
       and the scale doubles every growth_interval = 3 steps, identically in both runs.

    The replays of both phases run under torch.cuda.set_sync_debug_mode("error")."""
    from distributed_sod_project_b200.synthetic import synth_batch
    amp = amp_reset
    sizes = [64, 96, 128] * 15
    batches = [tuple(t.cuda() for t in synth_batch(4000 + i, 2, s)) for i, s in enumerate(sizes)]
    batches2 = [tuple(t.cuda() for t in synth_batch(5000 + i, 2, s)) for i, s in enumerate([64, 96, 128] * 4)]
    runs = {}
    for graph in (False, True):
        tr = _trainer(use_graph=graph)
        assert amp._cfg["dynamic"] and tr.use_graph == graph
        assert tr.optimizer.flat.shadow16 is not None and tr.optimizer.flat.shadow16.dtype == torch.float16
        amp._cfg["scale"] = 2.0 ** 40
        amp._cfg["growth_interval"] = 3
        amp.push()                                       # on the device before the first recorded entry
        phase1 = _run_history(tr, batches, 3 if graph else None)     # (every input size is captured by then)
        if graph:
            assert len(tr._graphs) == 3
        amp.read_scaler()                                # the host mirror brought up to date (a sync, between the phases)
        amp._cfg["scale"], amp._cfg["good_steps"] = 2.0 ** 6, 0
        amp.push()
        phase2 = _run_history(tr, batches2, 0 if graph else None)
        assert len(tr._graphs) == (3 if graph else 0)
        st = amp.read_scaler()
        runs[graph] = (phase1, phase2, st)
    ((h0, l0), (g0, m0), st0), ((h1, l1), (g1, m1), st1) = runs[False], runs[True]
    skips = [k for _, k in h0]
    assert False in skips, f"the scale never fitted: {h0}"
    first_ok = skips.index(False)
    assert first_ok > 0 and all(skips[:first_ok]) and h0[first_ok][0] == 2.0 ** 40 / 2 ** first_ok
    assert h0[:first_ok + 2] == h1[:first_ok + 2]
    assert np.all(np.isfinite(l0[:first_ok + 1])) and np.all(np.isfinite(l1[:first_ok + 1]))
    assert l1[:first_ok + 1] == pytest.approx(l0[:first_ok + 1], rel=2e-3)
    for h in (h0, h1):
        _follows_the_rules(h, 3)
    want = [(2.0 ** (6 + i // 3), False) for i in range(len(batches2))]
    assert g0 == want and g1 == want
    assert st0 == st1 == {"scale": 2.0 ** (6 + len(batches2) // 3), "unskipped": len(batches2), "found_inf": 0}
    assert np.all(np.isfinite(m0)) and np.all(np.isfinite(m1))


def test_capture_warmup_leaves_the_scaler_untouched(amp_reset):
    from distributed_sod_project_b200.synthetic import synth_batch
    amp = amp_reset
    tr = _trainer(use_graph=True)
    amp._cfg["growth_interval"] = 5
    x, m = (t.cuda() for t in synth_batch(77, 2, 64))
    s0 = amp.read_scaler()
    tr.forward_backward_update(x, m)                    # warm-up iterations, capture, one replay
    s1 = amp.read_scaler()
    if s1["found_inf"]:
        assert (s1["scale"], s1["unskipped"]) == (s0["scale"] / 2, 0)
    else:
        assert (s1["scale"], s1["unskipped"]) == (s0["scale"], s0["unskipped"] + 1)
    assert tr.optimizer.steps == 1


def test_fp16_shadow_weights_exact_on_a_deterministic_net(amp_reset):
    """conv(+bias) → BN kernel → conv, no atomics: the fp16 shadow path (fp16 copy written by the fused step, fp16 gradients
    gathered and folded in, device loss scale) reproduces stock torch.autocast(float16) on the fp32 masters bit for bit"""
    import torch.nn as nn
    from distributed_sod_project_b200.optim import make_optimizer
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    amp = amp_reset

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.div_4 = nn.Conv2d(8, 16, 3, padding=1)
            self.bn = nn.BatchNorm2d(16)
            self.head = nn.Conv2d(16, 8, 1, bias=False)

        def forward(self, x):
            return self.head(torch.relu(self.bn(self.div_4(x))))

    outs = {}
    for shadow in (False, True):
        torch.manual_seed(0)
        net = Net().cuda().to(memory_format=torch.channels_last)
        opt = make_optimizer(net, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
        net = convert_syncbn_model(net)
        net, opt = amp.initialize(net, opt, opt_level="O1", dtype=torch.float16, shadow_weights=shadow)
        g = torch.Generator().manual_seed(1)
        for it in range(3):
            x = torch.randn(4, 8, 12, 12, generator=g).cuda().contiguous(memory_format=torch.channels_last)
            opt.zero_grad()
            with amp.scale_loss(net(x).float().square().mean(), opt) as scaled:
                scaled.backward()
            opt.step()
            assert not int(opt.found_inf.item())
        outs[shadow] = opt.flat.param.clone()
        assert (opt.flat.shadow16 is not None) == shadow
        if shadow:
            assert torch.equal(opt.flat.shadow16.view(torch.int16)[:1000], opt.flat.param.half().view(torch.int16)[:1000])
    assert torch.equal(outs[True], outs[False])


def test_checkpoint_round_trip_of_the_device_scaler(amp_reset, tmp_path):
    from distributed_sod_project_b200 import amp as amp_mod
    from distributed_sod_project_b200.checkpoint import resume_checkpoint, save_checkpoint
    from distributed_sod_project_b200.synthetic import synth_batch
    amp = amp_reset
    tr = _trainer(use_graph=True)
    amp._cfg["growth_interval"] = 2
    amp._cfg["scale"] = 2.0 ** 18
    for i in range(3):
        tr.forward_backward_update(*(t.cuda() for t in synth_batch(50 + i, 2, 64)))
    saved = amp.read_scaler()
    full, state = str(tmp_path / "full.pth"), str(tmp_path / "state.pth")
    save_checkpoint(model=tr.model, optimizer=tr.optimizer, amp=amp_mod, exp_name="x", current_epoch=1,
                    full_net_path=full, state_net_path=state)
    sd = torch.load(full, weights_only=False)["amp_state"]["loss_scaler0"]
    assert sd == {"loss_scale": saved["scale"], "unskipped": saved["unskipped"]}
    nxt = tuple(t.cuda() for t in synth_batch(60, 2, 64))
    tr.forward_backward_update(*nxt)
    after_a = amp.read_scaler()
    tr2 = _trainer(use_graph=True)
    amp._cfg["growth_interval"] = 2
    resume_checkpoint(model=tr2.model, optimizer=tr2.optimizer, amp=amp_mod, exp_name="x", load_path=full)
    assert amp.read_scaler()["scale"] == saved["scale"] and amp.read_scaler()["unskipped"] == saved["unskipped"]
    tr2.forward_backward_update(*nxt)
    after_b = amp.read_scaler()
    assert (after_a["scale"], after_a["unskipped"], after_a["found_inf"]) == \
        (after_b["scale"], after_b["unskipped"], after_b["found_inf"])


def test_train_cli_fp16_cuda_graph():
    import json
    import subprocess
    import sys
    cfg = {"epoch_num": 1, "synthetic_iters_per_epoch": 4, "batch_size": 2, "print_freq": 1, "save_freq": 0,
           "is_distributed": False, "input_size": 64, "size_list": [64], "model": "res50", "use_amp": True, "dtype": "fp16",
           "cuda_graph": True, "synthetic_eval_images": 2}
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "-ng", "1", "-p", "29731"], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=500)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "End Training" in out.stdout and out.stdout.count("[I:") == 4
