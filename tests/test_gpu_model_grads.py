"""Every parameter gradient of one whole training iteration against float64 autograd of the same model.

Each kernel has its own rounding-level test; this file checks the wiring that joins them: which flat-buffer slot each
of the model's gradients lands in and which buffer the step kernel reads it from (the group-major layout and its
[16-bit part | fp32 part] split per bucket, the stolen cuDNN weight gradients and their one gather launch, the folded
conv biases the SyncBN backward adds into a bound `.grad`, the BN γ/β gradients written straight into the fp32 buffer,
the `trans*` biases summed by `sod_colsum`, the resampling and max-pool backward kernels, the recompute of `cp_res50`).

* Oracle: `init_seed(0)` + the model factory, `.double()`, stock modules (no SyncBN, no amp, `resample.ENABLED` off),
  the reference loss BCEWithLogits(mean) + CEL (eps 1e-6) in float64 torch ops.
* Engine: one `Trainer.forward_backward_update` with momentum 0.9 and no weight decay.  The first step computes
  v = fmaf(0.9, 0, fmaf(0, p, g·inv_scale)), so the momentum buffer holds, bit for bit, the gradient the step kernel
  consumed (fp16: inv_scale is a power of two, still exact) — after the gather, the segment flags and the choice of
  buffer, none of which a hook on `p.grad` would see.
* Yardstick: stock PyTorch in the same precision on the same GPU and batch (fp32: TF32 off, deterministic cuDNN;
  bf16 / fp16: `torch.autocast`, fp16 with the engine's loss scale S and the gradients divided by S).  For every
  tensor P, e2 = ‖g − g64‖₂ / ‖g64‖₂ and emax = max|g − g64| / max|g64|; the engine must meet
      e(engine, P) ≤ A · (e(stock, P) + median_Q e(stock, Q))
  for both metrics, for every tensor and for the concatenation of all of them.  The same rule holds the BN running
  statistics after the iteration and the loss (there with a slack of one rounding of the precision).
  Gradients that are zero in exact arithmetic — the conv biases folded into a training-mode BN, whose output does not
  depend on them — carry only rounding noise, in the oracle too; for them (max|g64| ≤ 1e-9 of the model's largest
  gradient) both metrics are normalised by the model's largest gradient and the median is taken over them alone.

A wiring fault (a slot shifted, a range read from the wrong buffer, a gradient dropped or scaled) puts an error of order 1
on some tensor.  In fp32 that is 25 times the rounding error, and the rule above catches it.  In 16 bits it is not:
the model at its seeded initialisation amplifies the rounding of the logits' gradient by about 10³ on its way down
(fp32: 2e-5 at the classifier, 2e-3 at upconv2, 1e-2 at trans2 and the encoder), so stock bf16 gradients are as far
from fp64 as a zero gradient would be (median e2 1.26, cosine of the whole gradient 0.08; fp16: 0.85 and 0.57).  The
16-bit cases are therefore also held to a second reference in their own precision:
* the same Trainer iteration without shadow weights, where autograd accumulates every gradient into the fp32 `.grad`
  views: no gather, no 16-bit buffer or GRAD16 segments, no bound 16-bit bias views, no column sum.  The engine is
  deterministic, and the two differ only by where they round, so every tensor's e2 between them is bounded, per kind of
  tensor (conv weights, the conv biases that do not feed a BN, BN γ/β), by PLAIN_BOUND.  This reference shares the flat
  layout, the SyncBN, loss and resampling kernels with the engine; those are what the fp32 cases hold to float64.
  A zeroed, shifted, sign-flipped or partly copied 16-bit gradient puts e2 ≥ 0.25 on its tensor, which fails here.

Measured on an H100 80GB HBM3 at 700 W; worst ratio e(engine) / (e(stock) + median) over all cases of a precision:
    fp32  gradients  e2 0.75 (sim16.h2h_0.weight)  emax 7.5 (div_32.1.conv1.weight, see below)
          running stats  e2 1.31  emax 1.62 (upconv32.basicconv.1.running_mean)
    bf16  gradients  e2 0.60 (div_4.1.1.bn2.bias)  emax 0.76 (div_16.1.bn2.weight, 320²)
          running stats  e2 1.07 (sim32.bnh_2.running_mean, 320²)  emax 1.16 (div_32.1.bn1.running_var, 320²)
    fp16  gradients  e2 0.63  emax 1.06 (div_4.1.0.bn1.weight)
          running stats  e2 1.00 (upconv32.basicconv.1.running_mean)  emax 1.14 (div_32.2.bn2.running_mean)
and against the iteration without shadow weights, the worst e2 over bf16 and fp16 is 0.110 for conv weights
(trans2.weight), 0.074 for conv biases (trans4.bias) and 0.114 for BN parameters (div_2.1.bias, sgd_trick).  BOUND and
PLAIN_BOUND leave at least 2× over these.  The file runs in about a minute; the fp64 oracle takes 1-2 s per shape.

The fp32 emax outlier is one ReLU decision.  Its error sits in output channel 422 of div_32.1.conv1.weight alone (0.31
of max|g64| there, 0.018 in every other channel; stock: 0.017), and that error row is parallel to one input row of the
convolution (cosine 0.87 with row 13, at most 0.09 with the other 63).  So one element of dz differs, and in fp64 its
pre-ReLU BN output is 1.3e-4 standard deviations, the 4th smallest of the layer's 32768: the engine's fp32 forward
lands on the other side of zero there, stock's on the same side as fp64.  The channel is not degenerate (batch variance
2.7, invstd 0.61; layer median 5.4), and the error is the same with either SyncBN backward variant.
"""
import contextlib
import statistics
import time

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BS = 4
SEED = 1234
FP16_SCALE = 2.0 ** 12          # the first step must not overflow fp16 (asserted)
ZERO_REL = 1e-9                 # max|g64(P)| below this fraction of the model's largest gradient: zero in exact arithmetic
# A of the rule in the module docstring, per precision: (for e2, for emax)
BOUND = {torch.float32: (3.0, 15.0), torch.bfloat16: (2.5, 2.5), torch.float16: (2.5, 2.5)}
# relative slack of the loss check: fp32 ~ its summation error, bf16 as tests/test_gpu_step.py, fp16 one rounding at 2^-10
LOSS_SLACK = {torch.float32: 1e-5, torch.bfloat16: 5e-3, torch.float16: 2.0 ** -10}
# 16-bit: e2 of every tensor against the iteration without shadow weights, per kind of tensor (see `_kinds`)
PLAIN_BOUND = {"weight": 0.22, "bias": 0.15, "bn": 0.23}
NAME = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}


@contextlib.contextmanager
def _stock_modules():
    """the model's own torch ops: no resampling / max-pool / column-sum kernels (module globals the Trainer turns on)"""
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.network import blocks
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = False, False
    try:
        yield
    finally:
        resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old


@contextlib.contextmanager
def _strict(dtype):
    """fp32: TF32 off and deterministic cuDNN (as tests/test_gpu_step.py runs fp32), restored afterwards"""
    if dtype != torch.float32:
        yield
        return
    b = torch.backends
    old = b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic
    b.cudnn.allow_tf32 = b.cuda.matmul.allow_tf32 = False
    b.cudnn.deterministic = True
    try:
        yield
    finally:
        b.cudnn.allow_tf32, b.cuda.matmul.allow_tf32, b.cudnn.deterministic = old


def _reference_loss(logits, mask, eps=1e-6):
    """BCEWithLogits(mean) + CEL (oracle/loss.py), in the dtype of the inputs"""
    bce = F.binary_cross_entropy_with_logits(logits, mask)
    p = torch.sigmoid(logits)
    inter = p * mask
    cel = ((p - inter).sum() + (mask - inter).sum()) / (p.sum() + mask.sum() + eps)
    return bce + cel


def _batch(size):
    from distributed_sod_project_b200.synthetic import synth_batch
    return synth_batch(SEED, BS, size)


def _bn_buffers(model):
    return {n: b.detach().clone() for n, b in model.named_buffers()
            if n.rsplit(".", 1)[-1] in ("running_mean", "running_var", "num_batches_tracked")}


def _stock_iteration(model_name, size, dtype, scale=1.0):
    """one forward + backward of the stock model: (init params fp32, grads fp64, BN buffers, loss)"""
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    x, m = _batch(size)
    init_seed(0)
    model = getattr(network, model_name)()
    init = {n: p.detach().cuda() for n, p in model.named_parameters()}
    if dtype == torch.float64:
        model, x, m = model.double().cuda(), x.double().cuda(), m.double().cuda()
    else:
        model = model.cuda().to(memory_format=torch.channels_last)
        x, m = x.cuda().contiguous(memory_format=torch.channels_last), m.cuda()
    model.train()
    with _stock_modules(), _strict(dtype):
        with torch.autocast("cuda", dtype=dtype, enabled=dtype in (torch.bfloat16, torch.float16)):
            preds = model(x)
        loss = _reference_loss(preds.to(m.dtype), m)
        (loss * scale).backward()
    grads = {n: p.grad.double() / scale for n, p in model.named_parameters()}
    assert all(bool(torch.isfinite(g).all()) for g in grads.values()), "stock gradients overflowed"
    return init, grads, _bn_buffers(model), float(loss.detach())


def _kinds(model_name) -> dict:
    """parameter name → "weight" (conv weights), "bias" (conv biases) or "bn" (BN γ/β)"""
    import torch.nn as nn
    from distributed_sod_project_b200 import network
    out = {}
    for mn, mod in getattr(network, model_name)().named_modules():
        for pn, _ in mod.named_parameters(recurse=False):
            kind = "bn" if isinstance(mod, nn.BatchNorm2d) else ("weight" if pn == "weight" else "bias")
            out[f"{mn}.{pn}" if mn else pn] = kind
    return out


def _norms(ref: dict) -> dict:
    """per tensor: (zero in exact arithmetic, e2 normaliser, emax normaliser)"""
    top = max(float(t.double().abs().max()) for t in ref.values())
    out = {}
    for n, t in ref.items():
        t = t.double()
        mx = float(t.abs().max())
        zero = mx <= ZERO_REL * top
        out[n] = (zero, top, top) if zero else (zero, float(t.norm()), mx)
    return out


def _diffs(got: dict, ref: dict) -> dict:
    """per tensor: (‖got − ref‖₂, max|got − ref|), float64"""
    out = {}
    for n, r in ref.items():
        d = got[n].double() - r.double()
        out[n] = (float(d.norm()), float(d.abs().max()))
    return out


@pytest.fixture(scope="module")
def oracle():
    """float64 autograd, once per (model, size): {init, grads, buffers, loss, norms, bnorms, seconds}"""
    cache = {}

    def get(model_name, size):
        key = (model_name, size)
        if key not in cache:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            init, grads, bufs, loss = _stock_iteration(model_name, size, torch.float64)
            torch.cuda.synchronize()
            sec = time.perf_counter() - t0
            print(f"\nfp64 oracle {model_name} bs {BS} {size}²: {sec:.2f} s")
            stats = {n: b for n, b in bufs.items() if not n.endswith("num_batches_tracked")}
            cache[key] = dict(init=init, grads=grads, buffers=bufs, loss=loss, norms=_norms(grads), bnorms=_norms(stats),
                              kinds=_kinds(model_name), seconds=sec)
        return cache[key]
    yield get
    cache.clear()


@pytest.fixture(scope="module")
def stock(oracle):
    """stock torch in the engine's precision, once per (model, size, dtype): its differences from the oracle"""
    cache = {}

    def get(model_name, size, dtype):
        key = (model_name, size, dtype)
        if key not in cache:
            ref = oracle(model_name, size)
            _, grads, bufs, loss = _stock_iteration(model_name, size, dtype,
                                                    scale=FP16_SCALE if dtype == torch.float16 else 1.0)
            stats = {n: b for n, b in bufs.items() if not n.endswith("num_batches_tracked")}
            cache[key] = dict(grads=_diffs(grads, ref["grads"]), stats=_diffs(stats, {n: ref["buffers"][n] for n in stats}),
                              loss=loss)
        return cache[key]
    yield get
    cache.clear()


def _yardstick(what, eng: dict, stk: dict, norms: dict, names, bound: tuple) -> list:
    """e(engine) ≤ A · (e(stock) + median e(stock)) per tensor (median within its class: zero in exact arithmetic or not)
    and for the concatenation, A = bound[0] for e2 and bound[1] for emax; returns (worst ratio, where) per metric"""
    out = []
    for k, metric in ((1, "e2"), (2, "emax")):
        es = {n: stk[n][k - 1] / norms[n][k] for n in names}
        ee = {n: eng[n][k - 1] / norms[n][k] for n in names}
        med = {}
        for cls in (False, True):
            vals = [es[n] for n in names if norms[n][0] == cls]
            med[cls] = statistics.median(vals) if vals else 0.0
        checks = [(n, ee[n], es[n], med[norms[n][0]]) for n in names]
        # the concatenation of every tensor (the zero-class ones enter with their own oracle values)
        if k == 1:
            tot64 = sum(norms[n][1] ** 2 for n in names if not norms[n][0]) ** 0.5
            cat_e = sum(eng[n][0] ** 2 for n in names) ** 0.5 / tot64
            cat_s = sum(stk[n][0] ** 2 for n in names) ** 0.5 / tot64
        else:
            top = max(norms[n][2] for n in names if not norms[n][0])
            cat_e = max(eng[n][1] for n in names) / top
            cat_s = max(stk[n][1] for n in names) / top
        checks.append(("<all tensors>", cat_e, cat_s, med[False]))
        worst, where = 0.0, ""
        for n, e, s, md in checks:
            r = e / (s + md) if s + md > 0 else (0.0 if e == 0 else float("inf"))
            if r > worst:
                worst, where = r, f"{n} (engine {e:.3e}, stock {s:.3e}, median {md:.3e})"
        assert worst <= bound[k - 1], f"{what}: {metric} {worst:.2f}x (stock + median) > {bound[k - 1]} at {where}"
        out.append((worst, where))
    return out


def _engine_iteration(model_name, size, dtype, optim, use_graph=False, report=False, shadow=True):
    """one Trainer iteration: (initial params, consumed gradients from the momentum buffer, params after, BN buffers,
    loss)"""
    from distributed_sod_project_b200 import amp
    from distributed_sod_project_b200.engine import Trainer
    x, m = _batch(size)
    try:
        with _strict(dtype):
            tr = Trainer(model_name=model_name, lr=0.05, momentum=0.9, weight_decay=0.0, optim=optim, dtype=dtype,
                         channels_last=True, use_graph=use_graph, report_items=report, shadow_weights=shadow)
            assert tr.use_graph == use_graph
            named = dict(tr.module.named_parameters())
            p0 = {n: p.detach().clone() for n, p in named.items()}
            if dtype == torch.float16:
                assert amp._cfg["dynamic"]
                amp._cfg["scale"] = FP16_SCALE
            red, _, _ = tr.forward_backward_update(x.cuda(), m.cuda())
            torch.cuda.synchronize()
        if dtype == torch.float16:
            assert int(tr.optimizer.found_inf.item()) == 0, "the first fp16 step overflowed"
            assert amp.read_scaler()["scale"] == FP16_SCALE
    finally:
        if dtype == torch.float16:
            amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None,
                            dev=None)
    if dtype != torch.float32:
        assert (tr.optimizer.flat.shadow16 is not None) == shadow
    flat = tr.optimizer.flat
    grads = {n: flat.momentum_view(p).detach().clone() for n, p in named.items()}
    after = {n: p.detach().clone() for n, p in named.items()}
    return p0, grads, after, _bn_buffers(tr.module), float(red)


def _check_case(oracle, stock, model_name, size, dtype, optim, use_graph=False, report=False):
    ref = oracle(model_name, size)
    stk = stock(model_name, size, dtype)
    p0, grads, after, bufs, loss = _engine_iteration(model_name, size, dtype, optim, use_graph, report)
    names = set(ref["grads"])
    assert set(grads) == names, "the engine's parameters are not the model's"
    for n in names:                                   # same starting point, or the comparison means nothing
        assert torch.equal(p0[n], ref["init"][n]), n
    # f3_trick leaves the stem (div_2) out of every group: no gradient consumed, no update
    frozen = {n for n in names if n.startswith("div_2")} if optim == "f3_trick" else set()
    for n in frozen:
        assert float(grads[n].abs().max()) == 0.0 and torch.equal(after[n], p0[n]), n
    compared = sorted(names - frozen)
    assert set(compared) | frozen == names
    bound = BOUND[dtype]
    tag = f"{model_name} {size}² {NAME[dtype]} {optim}{' graph' if use_graph else ''}{' report' if report else ''}"
    report_lines = [f"{tag}: loss {loss:.6f} stock {stk['loss']:.6f} fp64 {ref['loss']:.6f}"]
    (g2, at_g2), (gm, at_gm) = _yardstick(f"{tag} gradients", _diffs(grads, {n: ref["grads"][n] for n in compared}),
                                          stk["grads"], ref["norms"], compared, bound)
    report_lines.append(f"  gradients vs fp64: worst e2 ratio {g2:.3f} at {at_g2}; worst emax ratio {gm:.3f} at {at_gm}")
    # running statistics after the iteration (cp_res50: the recompute updates them a second time, in both)
    stats = sorted(ref["bnorms"])
    (s2, at_s2), (sm, at_sm) = _yardstick(f"{tag} running stats", _diffs(bufs, {n: ref["buffers"][n] for n in stats}),
                                          stk["stats"], ref["bnorms"], stats, bound)
    report_lines.append(f"  running stats vs fp64: worst e2 ratio {s2:.3f} at {at_s2}; worst emax ratio {sm:.3f} at {at_sm}")
    for n, b in ref["buffers"].items():
        if n.endswith("num_batches_tracked"):
            assert int(bufs[n]) == int(b), n
    # the loss, computed before any gradient is used
    l64 = ref["loss"]
    assert abs(loss - l64) <= bound[0] * abs(stk["loss"] - l64) + LOSS_SLACK[dtype] * abs(l64), (loss, stk["loss"], l64)
    if dtype != torch.float32:
        # 16-bit: the same iteration without the shadow weights, where autograd accumulates every gradient into the fp32
        # `.grad` views (no gather, no 16-bit buffer or segments, no bound 16-bit bias views, no column sum)
        _, plain, _, _, _ = _engine_iteration(model_name, size, dtype, optim, shadow=False)
        # (the folded conv biases are left out: both runs hold rounding noise there, and their exact value is zero)
        e2 = {n: float((grads[n].double() - plain[n].double()).norm()) /
              max(float(plain[n].double().norm()), 1e-300) for n in compared if not ref["norms"][n][0]}
        for kind, bound in PLAIN_BOUND.items():
            of_kind = [n for n in e2 if ref["kinds"][n] == kind]
            worst = max(of_kind, key=e2.get)
            report_lines.append(f"  vs the engine without shadow weights, {kind}: worst e2 {e2[worst]:.3e} at {worst}")
            assert e2[worst] <= bound, f"{tag}: {worst} differs by {e2[worst]:.3e} from the plain-autograd iteration"
        assert {ref["kinds"][n] for n in e2} == set(PLAIN_BOUND)
    print("\n" + "\n".join(report_lines))


_F32, _BF16, _F16 = torch.float32, torch.bfloat16, torch.float16
CASES = [
    *[pytest.param("res50", 128, dt, opt, False, False, id=f"res50-128-{NAME[dt]}-{opt}")
      for dt in (_F32, _BF16, _F16) for opt in ("sgd_all", "f3_trick", "sgd_trick")],
    *[pytest.param("res50", 128, dt, "f3_trick", True, False, id=f"res50-128-{NAME[dt]}-f3_trick-graph") for dt in (_BF16, _F16)],
    *[pytest.param("res50", 128, dt, "f3_trick", False, True, id=f"res50-128-{NAME[dt]}-f3_trick-report") for dt in (_BF16, _F16)],
    pytest.param("cp_res50", 128, _BF16, "f3_trick", False, False, id="cp_res50-128-bf16-f3_trick"),
    pytest.param("cp_res50", 128, _BF16, "f3_trick", True, False, id="cp_res50-128-bf16-f3_trick-graph"),
    pytest.param("res50", 320, _BF16, "f3_trick", True, False, id="res50-320-bf16-f3_trick-graph"),
]


@pytest.mark.parametrize("model_name,size,dtype,optim,use_graph,report", CASES)
def test_iteration_gradients_match_fp64(oracle, stock, model_name, size, dtype, optim, use_graph, report):
    _check_case(oracle, stock, model_name, size, dtype, optim, use_graph, report)


@pytest.mark.parametrize("mask_from_x,l2_hints", [(False, True), (True, False), (False, False)])
@pytest.mark.parametrize("dtype", [_F32, _BF16], ids=["fp32", "bf16"])
def test_syncbn_backward_variants_gradients_match_fp64(oracle, stock, monkeypatch, dtype, mask_from_x, l2_hints):
    """the SyncBN backward without the ReLU mask re-derived from x and without L2 hints (both on by default); fp32 is the
    case where the float64 comparison is sharp enough to see a wrong variant"""
    from distributed_sod_project_b200 import syncbn
    monkeypatch.setattr(syncbn, "MASK_FROM_X", mask_from_x)
    monkeypatch.setattr(syncbn, "L2_HINTS", l2_hints)
    _check_case(oracle, stock, "res50", 128, dtype, "sgd_trick")
