"""Every block of `res50`, `vgg16`, `wsgn_res50`, `wsgn_resnext50` and `aim_res50`'s LightAIM neck through the engine's
autograd seam, against float64 autograd of the same block.

`tests/test_gpu_model_grads.py`, `tests/test_gpu_backbones.py` and `tests/test_gpu_aim.py` check the seam (`_SyncBNFn`,
`raw_backward`, `_Up2x`, `_AvgPool2x2`, `_MaxPool3x3s2`, `_MaxPool2x2s2`, `_UpNearest2x`, `_ConvBias`, `_FusedLossFn`,
`_GroupNormFn`, `_WSFn`, `_WSGroupConvFn`, the `network/blocks.py` helpers and the shadow-weight conv forward of `amp.py`)
only through the whole model, which amplifies rounding about 10³-fold: in 16 bits a wiring fault hides there.  A single
block has no such amplification, so here every site of oracle/block_sites.py is held close to float64 on its own.  Rows:
every representative site of each backbone (`bs.grid`); the WS-GN models' decoder is `res50`'s code at `res50`'s shapes
and runs in the `res50` rows, and so is everything of `aim_res50` but its five neck blocks `trans.conv0` … `trans.conv4`
(their float64 twin: the stock BatchNorm, `F.interpolate(mode="nearest")` and `nn.AvgPool2d`; operands non-negative, as
the backbone taps they stand for).

* Engine: the real `Trainer` construction (`sgd_all`, SyncBN and WS-GN conversion, bf16 / fp16 `amp.initialize` with
  shadow weights and a real `FusedSGD`), one backbone's Trainers at a time.  Each site runs on the engine's own modules; the gradients are read where the step reads them —
  the fp32 flat `.grad`, the bound 16-bit bias views, and the stolen 16-bit weight gradients after `_gather_stolen`.
  fp16 runs with a loss scale of 2¹² (the upstream gradient is scaled, the gradients read back divided by it).
* Reference: the site's modules copied from the stock model in float64 (`stock_twin`), run on exactly the engine's
  operands — the input rounded to the activation dtype, conv weights and biases equal to the 16-bit shadow values (VGG's
  folded backbone biases included), fp32 BN / GroupNorm parameters, the fp32 master of a WS convolution (no shadow: Ŵ is
  rounded once inside the block, by the engine and the stock yardstick alike) — so rounding inside the block is the only
  difference.
* Yardstick: the same stock modules in fp32 (TF32 off, deterministic cuDNN) or under `torch.autocast`, same operands.
  Per tensor, e2 = ‖g − g64‖₂/‖g64‖₂ and emax = max|g − g64|/max|g64|, and e(engine) ≤ A·(e(stock) + median) as in
  test_gpu_model_grads.py, for the output, the input gradient(s), every parameter gradient and the running statistics;
  gradients that are zero in exact arithmetic (conv biases folded into a training-mode BN) are measured against the
  site's largest gradient.  `num_batches_tracked` is exact.

Paths: eager training; the site captured in a CUDA graph and replayed on two fresh inputs (bit for bit against eager);
the site inside `torch.utils.checkpoint` as `cp_res50` runs it (bit for bit; running statistics updated twice,
`num_batches_tracked` + 2); eval mode with grad enabled (against float64 in eval mode).

The ×2 up-sample and GroupNorm keep their output in the activation dtype where stock autocast returns fp32 (so the WS-GN
bottlenecks' whole residual stream is 16-bit), so a 16-bit output that stock holds in fp32 is allowed one rounding of the
activation dtype more (OUT_SLACK).  A ReLU decision at a pre-activation within rounding of zero goes either way; one such
decision moves one element of a norm layer's gradient by its full size (e2 ≈ 1e-3 in a block, far above the fp32 bound),
for the stock yardstick as for the engine.  So when the A-rule fails, each is measured again against a float64 run that
takes its own ReLU decisions, provided every decision where the engine differs from float64 sits within TIE_REL (the
rounding of a 4608-term fp32 sum; four roundings of the 16-bit type) of zero.  Exact where an exact answer exists:
the two folded biases of a `pre` BN get the same Σ dz (and all three of a neck `conv3_bn_act`, whose second slot is the
non-leaf `b2 + b3`), the `trans*` bias gradient under shadow weights is `colsum(dy)`,
a residual's gradient is the ReLU-masked dy (for SyncBN and GroupNorm, in its own dtype), max-pool routes integer
gradients as torch does, GroupNorm gives the same bits for NCHW and channels-last operands, the γ/β and WS weight
gradients are the same bits added into a bound fp32 `.grad` or returned to autograd and a second backward doubles them,
`zero_grad` clears a backward whose only writes were the GroupNorm / WS kernels' adds, and the graph replay and the
checkpointed run equal eager.

Measured on an H100 80GB HBM3 at 700 W (S = 256, batch 2; batch 16 at 320² in bf16).  Worst ratio e(engine) /
(e(stock) + median) over all sites and paths, against BOUND (at least 2× above):
    fp32  e2 3.65 (head)  emax 5.02 (head)
    bf16  e2 0.98 (div_4.1.1, 320² bs 16)  emax 1.15 (sim16)
    fp16  e2 0.98 (div_4.1.1)  emax 1.21 (sim16)
Median stock e2 of the gradients per site (fp32 / bf16 / fp16; bf16 at 320² bs 16 within 20 % of 256² bs 2, upconv32
1.0e-2):
    stem 2.6e-7 / 3.3e-3 / 3.3e-4        bottlenecks ≤ 5.1e-4 / 4.9-6.4e-2 / 1.7-2.4e-2
    trans* 1.5e-7 / 2.3e-3 / 2.9e-4      sim* ≤ 3.0e-3 / 7.7-9.2e-2 / 1.8-4.8e-2
    upconv* ≤ 8.7e-5 / 2.6-4.1e-3 / ≤ 1.0e-3    upsample_add* 4e-8 / 1.7e-3 / 2.1e-4    head 2.3e-5 / 3.0e-3 / 3.8e-4
So the largest e2 a tensor may reach, A·(e(stock) + median), is below 0.1 for the stem, `trans*`, `upconv*`,
`upsample_add*` and the head in every precision and for every site in fp32, far under the e2 ≥ 0.25 of a zeroed,
shifted or sign-flipped gradient.  It does not clear that margin for the bf16 bottlenecks (0.30-0.41) and SIM blocks
(0.45-0.59), nor for fp16 sim32 (0.28; other fp16 bottlenecks and SIMs 0.10-0.21): stock bf16 autograd of a training-mode
BN block is itself 5-9 % from float64 there.  A wiring fault in those sites is caught by the fp32 and eval cases, by the
exact checks above and by reading the gradients from the step's buffers.  The file runs in about a minute.

The same measurements for the other rows (worst ratios without `upsample_add*`, whose output bound is OUT_SLACK alone):
    vgg16           fp32 e2 4.57 emax 10.26 (div_2, eval)   bf16 0.89 / 0.97 (head, eval; bs 16 0.74 / 0.96)
                    fp16 0.96 (head, eval) / 1.56 (sim32)
    wsgn_res50      fp32 0.88 / 1.15 (div_4.1.1)   bf16 0.66 / 0.87 (bs 16 0.62 / 0.89)   fp16 0.65 / 0.94
    wsgn_resnext50  fp32 1.40 / 2.23 (div_4.1.1, eval)   bf16 0.62 / 0.90 (bs 16 0.67 / 0.89)   fp16 0.68 / 0.94
Four cases took the ReLU-decision rule: wsgn_res50 div_16.0 fp32 eager (1 decision, |pre| / max 4.6e-8), vgg16 div_16
fp32 eval (2, 2.1e-7), vgg16 sim32 fp16 eval (7, 7.8e-5) and aim_res50 trans.conv0 fp32 eval (3, 5.5e-8); each then holds
at ratio ≤ 0.62 / 0.85 (aim_res50 0.92 / 1.50).  Median stock e2
of the gradients (fp32 / bf16 / fp16; bf16 at 320² bs 16 within 10 % of 256² bs 2):
    vgg16  slices 8.8e-6-7.2e-3 / 5.2-9.1e-2 / 1.8-3.3e-2   sim* ≤ 9.6e-4 / 8.2-9.6e-2 / 2.5-3.1e-2
           trans* 2e-7 / 2.4e-3 / 3.0e-4   upconv* ≤ 4.6e-7 / 2.9-9.2e-3 / ≤ 3.6e-4   head 5.2e-7 / 1.6e-3 / 1.9e-4
    wsgn_res50 / wsgn_resnext50  stem 2.7e-7 / 3.1-3.2e-2 / 1.1e-2   bottlenecks ≤ 1.3e-3 / 4.9-7.8e-2 / 1.4-2.8e-2
The bound stays above 0.25 for the 16-bit cases of the same kinds of site as in res50: bf16 (eager, eval and bs 16)
WS-GN bottlenecks 0.31-0.56, VGG slices 0.25-0.51 and VGG SIM blocks 0.27-0.59.
    aim_res50 (neck)  fp32 e2 1.01 (conv2) emax 1.67 (conv0)   bf16 0.66 / 0.80 (bs 16 0.58 / 0.71)   fp16 0.71 / 1.14
                      (conv4, eval)
Median stock e2 of the neck blocks' gradients: fp32 1.8e-6-4.4e-6 (conv1 … conv4; conv0 1.3e-3, its C = 64 stride-2
maps) / bf16 0.11-0.12 / fp16 0.040-0.049, eval 5.7e-7-6.3e-7 / 0.059-0.094 / 0.011-0.035.  As for the SIM blocks,
whose structure the neck blocks share, the bf16 bound stays above 0.25 (0.37-0.79), and so does fp16 eager conv3 (0.28;
the other fp16 cases 0.07-0.25): their wiring is held by the fp32 and eval cases, the exact checks and the dedicated
`conv3_bn_act` cases below (the same bits of Σ dz for all three biases through a bound fp32 or 16-bit `.grad` or a
temporary, in training and eval, with `b2` / `b3` frozen or one bias absent; a second backward doubles them; `zero_grad`
clears a backward whose only writes went through the non-leaf slot; biases of two dtypes in the two slots are refused).
In eval mode the folded biases' gradients are not zero in exact arithmetic and are measured against their own norm.
The whole file runs in about two and a half minutes on an H100 80GB HBM3 at 700 W.
"""
import collections
import contextlib
import statistics
import types

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.utils.checkpoint import checkpoint

from oracle import block_sites as bs

pytestmark = pytest.mark.gpu

S, BATCH = 256, 2
FP16_SCALE = 2.0 ** 12
DY_SCALE = 2.0 ** -10            # upstream gradient ~ N(0, 2⁻²⁰): fp16 wgrad sums stay finite under the loss scale
ZERO_REL = 1e-9
_F32, _BF16, _F16 = torch.float32, torch.bfloat16, torch.float16
NAME = {_F32: "fp32", _BF16: "bf16", _F16: "fp16"}
# A of e(engine) ≤ A·(e(stock) + median), (e2, emax), per precision
BOUND = {_F32: (8.0, 12.0), _BF16: (2.5, 2.5), _F16: (2.5, 2.5)}
# the ×2 up-sample stores its output in the activation dtype where stock autocast returns fp32: one rounding of it more
OUT_SLACK = {_F32: 0.0, _BF16: 2.0 ** -8, _F16: 2.0 ** -11}
LOSS_SLACK = {_F32: 1e-5, _BF16: 5e-3, _F16: 2.0 ** -10}
# a ReLU decision may differ from float64's only at a pre-activation this close to zero, relative to the layer's largest:
# fp32, the worst-case rounding of the longest sum in a block, K = 3·3·512 terms at u = 2⁻²⁴; 16 bits, four roundings of
# the activation dtype (the convolution output, pre_add and residual are each stored rounded, and so is the output)
TIE_REL = {_F32: 3 * 3 * 512 * 2.0 ** -24, _BF16: 4 * 2.0 ** -8, _F16: 4 * 2.0 ** -11}
PRECS = [pytest.param(d, id=NAME[d]) for d in (_F32, _BF16, _F16)]


def _row_id(model, name):
    return name if model == "res50" else f"{model}-{name}"       # res50's ids predate the other rows


# one row per (model, site) of the grid, grouped by model so that each backbone's Trainers are built once per test
SITES = [pytest.param(m, s.name, id=_row_id(m, s.name)) for m in bs.ALL_MODELS for s in bs.grid(m)]
RESULTS: list = []               # (model/site, precision, path, worst e2 ratio, worst emax ratio, stock e2 median, max bound e2)


@contextlib.contextmanager
def _strict(dtype):
    if dtype != _F32:
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


def _autocast(dtype):
    return torch.autocast("cuda", dtype=dtype, enabled=dtype != _F32)


def _one_backbone(cache, model):
    """the rows run backbone by backbone: entering another backbone's rows releases the previous one's objects"""
    for key in [k for k in cache if k[0] != model]:
        del cache[key]


@pytest.fixture(scope="module")
def engines():
    """one Trainer per (model, precision), built lazily, those of one backbone at a time; torn down with the module's
    global switches restored"""
    from distributed_sod_project_b200 import amp, resample
    from distributed_sod_project_b200.network import blocks
    old = resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    cache = {}

    def get(model, dtype):
        if (model, dtype) not in cache:
            _one_backbone(cache, model)
            torch.cuda.empty_cache()
            from distributed_sod_project_b200.engine import Trainer
            with _strict(dtype):
                tr = Trainer(model_name=model, lr=0.0, momentum=0.0, weight_decay=0.0, optim="sgd_all", dtype=dtype,
                             channels_last=True, report_items=False)
            if dtype != _F32:
                assert tr.optimizer.flat.shadow16 is not None and tr.optimizer.flat.shadow16.dtype == dtype
            cache[(model, dtype)] = tr
        # the Trainers share the module switches the engine turns on
        resample.ENABLED = blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = True
        return cache[(model, dtype)]
    yield get
    cache.clear()
    amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None, dev=None)
    resample.ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old


@pytest.fixture(scope="module")
def stock_model():
    """the stock model of a name (CPU, `init_seed(0)`, the engine's starting point), one backbone at a time"""
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    cache = {}

    def get(model):
        if (model,) not in cache:
            _one_backbone(cache, model)
            init_seed(0)
            cache[(model,)] = getattr(network, model)()
        return cache[(model,)]
    yield get
    cache.clear()


# ---- running one site ---------------------------------------------------------------------------------------------
def _site_buffers(model, site):
    return {f"{p}.{n}": b for p in site.paths for n, b in model.get_submodule(p).named_buffers()}


def _site_params(model, site):
    return {f"{p}.{n}": q for p in site.paths for n, q in model.get_submodule(p).named_parameters()}


def _operands(site, dtype, size, batch, seed):
    """(inputs in the activation dtype, channels-last; upstream gradient maker; mask)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    xs = [torch.randn(sh, device="cuda", generator=g) for sh in site.shapes(size, batch)]
    xs = [(x.relu() if site.relu_inputs else x).to(dtype).contiguous(memory_format=torch.channels_last) for x in xs]
    mask = (torch.rand(batch, 1, size, size, device="cuda", generator=g) > 0.6).float() if site.loss else None
    dy_seed = seed + 7919
    return xs, mask, dy_seed


def _upstream(out, dtype, seed):
    """the upstream gradient as the engine sees it (scaled, in the output's dtype) and its exact unscaled value"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = FP16_SCALE if dtype == _F16 else 1.0
    dy = (torch.randn(out.shape, device="cuda", generator=g) * (DY_SCALE * scale)).to(out.dtype)
    dy = dy.contiguous(memory_format=torch.channels_last)
    return dy, dy.double() / scale


def _clear_grads(opt):
    f = opt.flat
    f.grad.zero_()
    if f.grad16 is not None:
        f.grad16.zero_()
    opt.zero_grad()


def _read_grads(tr, site, scale):
    """every parameter gradient of the site, from where the fused step reads it (after the stolen-gradient gather)"""
    opt = tr.optimizer
    f = opt.flat
    opt._gather_stolen()
    shadowed = {id(m.weight) for m in tr.module.modules() if hasattr(m, "_sod_w16")} | \
               {id(m.bias) for m in tr.module.modules() if getattr(m, "_sod_b16", None) is not None}
    out = {}
    for n, p in _site_params(tr.module, site).items():
        if id(p) in shadowed:
            # a shadowed parameter's gradient lives in the 16-bit buffer alone; nothing may reach the fp32 master
            assert float(p.grad.abs().max()) == 0.0, f"{n}: fp32 gradient written under shadow weights"
            out[n] = f.view16(f.grad16, p).double() / scale
        else:
            out[n] = p.grad.double() / scale
    return out


def _engine_run(tr, site, dtype, xs, mask, dy_seed, path="eager", train=True):
    """one forward + backward of the site on the engine: dict(out, dx, grads, bufs, loss)"""
    model, opt = tr.module, tr.optimizer
    mods = bs.modules(model, site)
    for m in mods.values():
        m.train(train)
    _clear_grads(opt)
    scale = FP16_SCALE if dtype == _F16 else 1.0
    xs = [x.detach().clone().requires_grad_(ok) for x, ok in zip(xs, site.input_grad)]
    with _strict(dtype):
        with _autocast(dtype):
            if path == "checkpoint":
                out = checkpoint(lambda *a: site.run(mods, *a), *xs, use_reentrant=False, preserve_rng_state=False)
            else:
                out = site.run(mods, *xs)
        loss = None
        if site.loss:
            loss, scaled = _engine_loss(out, mask, dtype)
            scaled.backward()
        else:
            dy, _ = _upstream(out, dtype, dy_seed)
            out.backward(dy)
    for m in mods.values():
        m.train(True)
    grads = _read_grads(tr, site, scale)
    return dict(out=out.detach(), dx=[x.grad.double() / scale for x in xs], grads=grads,
                bufs={n: b.clone() for n, b in _site_buffers(model, site).items()},
                loss=None if loss is None else float(loss))


def _engine_loss(out, mask, dtype):
    from distributed_sod_project_b200.loss import _FusedLossFn
    holder = []
    if dtype == _F16:
        sdev = torch.full((), FP16_SCALE, dtype=torch.float32, device="cuda")
        total = _FusedLossFn.apply(out, mask, "mean", 1.0, 1.0, 1e-6, False, 0, holder, sdev)
        return total.detach(), total * sdev
    total = _FusedLossFn.apply(out, mask, "mean", 1.0, 1.0, 1e-6, True, 0, holder)
    return total.detach(), total


def _twin(tr, site, stock_model, dtype, ref_dtype, bufs0):
    """stock copies of the site's modules with the engine's operands: shadow values for 16-bit conv parameters (float64
    twin), fp32 masters otherwise (autocast rounds them to the same values; a WS convolution, which has no shadow,
    standardises its fp32 master and rounds Ŵ once, in the engine and in the stock yardstick alike), BN buffers as the
    engine had them"""
    mods = bs.stock_twin(site, stock_model, dtype=ref_dtype)
    f = tr.optimizer.flat
    eng = _site_params(tr.module, site)
    shadowed = {id(m.weight): m for m in tr.module.modules() if hasattr(m, "_sod_w16")}
    shadow_b = {id(m.bias) for m in tr.module.modules() if getattr(m, "_sod_b16", None) is not None}
    with torch.no_grad():
        for p, m in mods.items():
            m.cuda()
            for n, q in m.named_parameters():
                src = eng[f"{p}.{n}"]
                if ref_dtype == torch.float64 and (id(src) in shadowed or id(src) in shadow_b):
                    q.copy_(f.view16(f.shadow16, src).double())
                else:
                    q.copy_(src.detach().to(ref_dtype))
            for n, b in m.named_buffers():
                b.copy_(bufs0[f"{p}.{n}"])
            if ref_dtype != torch.float64:
                m.to(memory_format=torch.channels_last)
    return mods


def _stock_run(tr, site, stock_model, dtype, xs, mask, dy_seed, bufs0, ref_dtype, train=True):
    mods = _twin(tr, site, stock_model, dtype, ref_dtype, bufs0)
    for m in mods.values():
        m.train(train)
    scale = FP16_SCALE if (dtype == _F16 and ref_dtype != torch.float64) else 1.0
    xs = [x.detach().to(ref_dtype if ref_dtype == torch.float64 else x.dtype).requires_grad_(ok)
          for x, ok in zip(xs, site.input_grad)]
    with bs.stock_modules(), _strict(_F32 if ref_dtype == torch.float64 else dtype):
        with _autocast(dtype if ref_dtype != torch.float64 else _F32):
            out = site.run(mods, *xs)
        loss = None
        if site.loss:
            loss = bs.reference_loss(out.to(mask.dtype if ref_dtype != torch.float64 else torch.float64),
                                     mask.to(torch.float64) if ref_dtype == torch.float64 else mask)
            (loss * scale).backward()
        else:
            dy_eng, dy64 = _upstream(out, dtype, dy_seed)
            out.backward(dy64 if ref_dtype == torch.float64 else dy_eng.to(out.dtype))
    grads = {f"{p}.{n}": q.grad.double() / scale for p, m in mods.items() for n, q in m.named_parameters()}
    bufs = {f"{p}.{n}": b.detach().clone() for p, m in mods.items() for n, b in m.named_buffers()}
    return dict(out=out.detach(), dx=[x.grad.double() / scale for x in xs], grads=grads, bufs=bufs,
                loss=None if loss is None else float(loss))


# ---- the yardstick ---------------------------------------------------------------------------------------------------
def _tensors(run, with_bufs=True):
    t = {"<output>": run["out"]}
    for i, d in enumerate(run["dx"]):
        t[f"<input grad {i}>"] = d
    t.update(run["grads"])
    if with_bufs:
        t.update({n: b for n, b in run["bufs"].items() if not n.endswith("num_batches_tracked")})
    return t


def _yardstick(tag, eng, stk, ref, bound, out_slack=0.0, ref_eng=None):
    """e(engine) ≤ A·(e(stock) + median e(stock)) per tensor, medians per class (output, gradients, gradients zero in
    exact arithmetic, running statistics); returns (worst e2 ratio, worst emax ratio, median stock e2, max e2 bound).
    `ref_eng`: the float64 reference the engine is measured against, if not `ref` (see `_check_against_fp64`)"""
    ref_eng = ref if ref_eng is None else ref_eng
    def cls(n):
        return "out" if n == "<output>" else ("stat" if n.endswith(("running_mean", "running_var")) else "grad")
    top = max(float(ref[n].double().abs().max()) for n in ref if cls(n) == "grad")
    norms = {}
    for n, r in ref.items():
        r = r.double()
        mx = float(r.abs().max())
        zero = cls(n) == "grad" and mx <= ZERO_REL * top
        norms[n] = ("zero" if zero else cls(n), top if zero else float(r.norm()), top if zero else mx)
    worst, med_e2, max_bound = [0.0, 0.0], 0.0, 0.0
    for k, metric in ((0, "e2"), (1, "emax")):
        def err(run, n, r):
            d = run[n].double() - r[n].double()
            return (float(d.norm()) if k == 0 else float(d.abs().max())) / norms[n][1 + k]
        es = {n: err(stk, n, ref) for n in ref}
        ee = {n: err(eng, n, ref_eng) for n in ref}
        med = {c: statistics.median([es[n] for n in ref if norms[n][0] == c]) for c in {v[0] for v in norms.values()}}
        for n in ref:
            m = med[norms[n][0]]
            lim = bound[k] * (es[n] + m) + (out_slack if n == "<output>" else 0.0)
            r = ee[n] / (es[n] + m) if es[n] + m > 0 else (0.0 if ee[n] == 0 else float("inf"))
            assert ee[n] <= lim, f"{tag}: {n} {metric} {ee[n]:.3e} > {bound[k]} x (stock {es[n]:.3e} + median {m:.3e})"
            worst[k] = max(worst[k], r)
            if k == 0 and norms[n][0] in ("grad", "out"):
                max_bound = max(max_bound, lim)
        if k == 0:
            med_e2 = med.get("grad", 0.0)
    return worst[0], worst[1], med_e2, max_bound


@contextlib.contextmanager
def _relu_decisions(record=None, impose=None, margins=None, engine=False):
    """record: receives the ReLU decisions of every norm layer with ReLU, in call order: the engine's fused norm calls'
    y > 0 (`engine`), or the stock modules' `bn_act` pre-activation > 0.
    impose: such a list; the stock modules' `bn_act` then applies the k-th decisions instead of its own ReLU, counts the
    layers in `margins["layers"]` and lists in `margins["differ"]` |pre-activation| / max |pre-activation| of the layer
    at every position where the two differ."""
    from distributed_sod_project_b200.network import blocks
    from distributed_sod_project_b200.syncbn import SyncBatchNorm
    from distributed_sod_project_b200.wsgn import GroupNorm32
    saved = {c: c.fused_forward for c in (SyncBatchNorm, GroupNorm32)}
    bn_act = blocks.bn_act

    def recording(orig):
        def fused_forward(self, x, **kw):
            y = orig(self, x, **kw)
            if kw.get("relu", False):
                record.append(y.detach() > 0)
            return y
        return fused_forward

    def imposed(bn, x, *, relu=True, pre_add=None, residual=None):
        pre = bn_act(bn, x, relu=False, pre_add=pre_add, residual=residual)
        if not relu:
            return pre
        if impose is None:
            record.append(pre.detach() > 0)
            return F.relu(pre)
        keep = impose[len(margins["layers"])]
        margins["layers"].append(None)
        p = pre.detach()
        differ = keep != (p > 0)
        margins["differ"].extend((p[differ].abs() / p.abs().max()).tolist())
        return pre * keep

    try:
        if engine:
            for c, f in saved.items():
                c.fused_forward = recording(f)
        else:
            blocks.bn_act = imposed
        yield
    finally:
        for c, f in saved.items():
            c.fused_forward = f
        blocks.bn_act = bn_act


def _check_against_fp64(tr, stock_model, site, dtype, xs, mask, dy_seed, bufs0, path, train=True):
    """the A-rule against float64.  If it fails, the engine and the stock yardstick are each measured again against a
    float64 reference that takes their own ReLU decisions, provided every decision of the engine that differs from
    float64's sits at a pre-activation within TIE_REL of zero.  Such a tie goes either way with the rounding: one
    moves one element of a norm layer's gradient by its full size, an e2 of about 1/√(elements) ≈ 1e-3 in a block, far
    above the fp32 bound, and it is as likely for the stock yardstick as for the engine."""
    decisions, stock_decisions = [], []
    with _relu_decisions(record=decisions, engine=True):
        eng = _engine_run(tr, site, dtype, xs, mask, dy_seed, train=train)
    _restore(tr, site, bufs0)
    ref = _stock_run(tr, site, stock_model, dtype, xs, mask, dy_seed, bufs0, torch.float64, train=train)
    with _relu_decisions(record=stock_decisions):
        stk = _stock_run(tr, site, stock_model, dtype, xs, mask, dy_seed, bufs0, torch.float32, train=train)
    row = _row_id(type(tr.module).__name__, site.name)
    tag = f"{row} {NAME[dtype]} {path}"
    assert set(eng["grads"]) == set(ref["grads"]), tag
    for r in (eng, stk):
        assert all(bool(torch.isfinite(t).all()) for t in _tensors(r).values()), f"{tag}: non-finite"
    for n, b in ref["bufs"].items():
        if n.endswith("num_batches_tracked"):
            assert int(eng["bufs"][n]) == int(b) == int(bufs0[n]) + (1 if train else 0), (tag, n)
    slack = OUT_SLACK[dtype] if (eng["out"].dtype != _F32 and stk["out"].dtype == _F32) else 0.0
    try:
        w2, wm, med, mb = _yardstick(tag, _tensors(eng), _tensors(stk), _tensors(ref), BOUND[dtype], slack)
    except AssertionError:
        refs = []
        for taken in (decisions, stock_decisions):
            margins = {"layers": [], "differ": []}
            with _relu_decisions(impose=taken, margins=margins):
                refs.append(_stock_run(tr, site, stock_model, dtype, xs, mask, dy_seed, bufs0, torch.float64, train=train))
            assert len(margins["layers"]) == len(taken), tag
            if taken is decisions:
                differ = margins["differ"]
                assert differ and max(differ) <= TIE_REL[dtype], f"{tag}: ReLU decisions differ at |pre| / max {differ[:8]}"
        print(f"\n{tag}: {len(differ)} ReLU decision(s) of the engine differ from float64's, at |pre-activation| / max "
              f"<= {max(differ):.1e}")
        tag += " (own ReLU decisions)"
        w2, wm, med, mb = _yardstick(tag, _tensors(eng), _tensors(stk), _tensors(refs[1]), BOUND[dtype], slack,
                                     ref_eng=_tensors(refs[0]))
    # the SyncBN backward adds the same Σ dz into both folded biases of a conv_bn_act with `pre`, and conv3_bn_act's
    # second slot (the sum of two biases) hands it on to both of them
    for group in _folded(site):
        gs = [eng["grads"][f"{site.name}.{a}.bias"] for a in group]
        assert all(torch.equal(gs[0], g) for g in gs[1:]) and float(gs[0].abs().max()) > 0, f"{tag}: folded biases {group}"
    if site.loss:
        l64 = ref["loss"]
        assert abs(eng["loss"] - l64) <= BOUND[dtype][0] * abs(stk["loss"] - l64) + LOSS_SLACK[dtype] * abs(l64), \
            (tag, eng["loss"], stk["loss"], l64)
    RESULTS.append((row, NAME[dtype], path, w2, wm, med, mb))
    print(f"\n{tag}: worst ratio e2 {w2:.3f} emax {wm:.3f}; stock median gradient e2 {med:.2e}; largest e2 bound {mb:.2e}")
    return eng


_SIM_FOLDED = (("h2h_1", "l2h_1"), ("l2l_1", "h2l_1"), ("h2h_2", "l2h_2"))
# LightAIM: Conv2nV1 (blocks 0 and 4, merging into the high / low stream) and Conv3nV1 (blocks 1 … 3)
_NECK_FOLDED = {0: (("h2h_1", "l2h_1"), ("l2l_1", "h2l_1"), ("h2h_2", "l2h_2")),
                4: (("h2h_1", "l2h_1"), ("l2l_1", "h2l_1"), ("h2l_2", "l2l_2")),
                **dict.fromkeys((1, 2, 3), (("h2h_1", "m2h_1"), ("h2m_1", "m2m_1", "l2m_1"), ("m2l_1", "l2l_1"),
                                            ("h2m_2", "m2m_2", "l2m_2")))}


def _folded(site):
    """the groups of conv biases of the site that one BatchNorm's backward gives the same Σ dz"""
    if site.kind == "sim":
        return _SIM_FOLDED
    if site.kind == "neck":
        return _NECK_FOLDED[int(site.name[len("trans.conv"):])]
    return ()


def _restore(tr, site, bufs0):
    with torch.no_grad():
        for n, b in _site_buffers(tr.module, site).items():
            b.copy_(bufs0[n])


def _setup(engines, model, name, dtype, size=S, batch=BATCH, seed=11):
    tr = engines(model, dtype)
    site = bs.by_name(model)[name]
    xs, mask, dy_seed = _operands(site, dtype, size, batch, seed)
    bufs0 = {n: b.clone() for n, b in _site_buffers(tr.module, site).items()}
    return tr, site, xs, mask, dy_seed, bufs0


def _equal_runs(a, b, tag):
    assert torch.equal(a["out"], b["out"]), f"{tag}: output"
    for i, (u, v) in enumerate(zip(a["dx"], b["dx"])):
        assert torch.equal(u, v), f"{tag}: input gradient {i}"
    for n in a["grads"]:
        assert torch.equal(a["grads"][n], b["grads"][n]), f"{tag}: {n}"
    if a["loss"] is not None:
        assert a["loss"] == b["loss"], tag


# ---- the grid ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", PRECS)
@pytest.mark.parametrize("model,name", SITES)
def test_eager_matches_fp64(engines, stock_model, model, name, dtype):
    tr, site, xs, mask, dy_seed, bufs0 = _setup(engines, model, name, dtype)
    eng = _check_against_fp64(tr, stock_model(model), site, dtype, xs, mask, dy_seed, bufs0, "eager")
    _restore(tr, site, bufs0)
    if site.kind == "trans" and dtype != _F32:
        # the shadow-weight forward routes trans* through `conv_bias`: its bias gradient is colsum(dy) of the same dy
        from distributed_sod_project_b200 import resample
        f = tr.optimizer.flat
        shape = (BATCH, 64) + tuple(xs[0].shape[2:])          # the upstream gradient depends on the output's shape only
        dy, _ = _upstream(torch.empty(shape, dtype=dtype, device="cuda"), dtype, dy_seed)
        bias = tr.module.get_submodule(name).bias
        scale = FP16_SCALE if dtype == _F16 else 1.0
        assert torch.equal(eng["grads"][f"{name}.bias"], resample.colsum(dy).double() / scale)
        assert f.view16(f.grad16, bias).dtype == dtype


@pytest.mark.parametrize("model,name", SITES)
def test_eager_bs16_320_bf16(engines, stock_model, model, name):
    tr, site, xs, mask, dy_seed, bufs0 = _setup(engines, model, name, _BF16, size=320, batch=16, seed=29)
    _check_against_fp64(tr, stock_model(model), site, _BF16, xs, mask, dy_seed, bufs0, "bs16-320")
    _restore(tr, site, bufs0)


@pytest.mark.parametrize("dtype", PRECS)
@pytest.mark.parametrize("model,name", SITES)
def test_eval_mode_backward_matches_fp64(engines, stock_model, model, name, dtype):
    tr, site, xs, mask, dy_seed, bufs0 = _setup(engines, model, name, dtype, seed=13)
    if bufs0:       # non-trivial running statistics, so the eval forward differs from the batch-statistics one
        g = torch.Generator(device="cuda").manual_seed(3)
        with torch.no_grad():
            for n, b in _site_buffers(tr.module, site).items():
                if n.endswith("running_mean"):
                    b.copy_(torch.randn(b.shape, device="cuda", generator=g) * 0.3)
                elif n.endswith("running_var"):
                    b.copy_(torch.rand(b.shape, device="cuda", generator=g) + 0.5)
        shifted = {n: b.clone() for n, b in _site_buffers(tr.module, site).items()}
    else:
        shifted = bufs0
    eng = _check_against_fp64(tr, stock_model(model), site, dtype, xs, mask, dy_seed, shifted, "eval", train=False)
    for n, b in eng["bufs"].items():
        assert torch.equal(b, shifted[n]), f"{name}: eval changed {n}"
    _restore(tr, site, bufs0)


@pytest.mark.parametrize("dtype", PRECS)
@pytest.mark.parametrize("model,name", SITES)
def test_checkpoint_equals_eager(engines, model, name, dtype):
    tr, site, xs, mask, dy_seed, bufs0 = _setup(engines, model, name, dtype, seed=17)
    eager = _engine_run(tr, site, dtype, xs, mask, dy_seed)
    with torch.no_grad(), _strict(dtype), _autocast(dtype):
        site.run(bs.modules(tr.module, site), *xs)            # the recompute's second statistics update
    twice = {n: b.clone() for n, b in _site_buffers(tr.module, site).items()}
    _restore(tr, site, bufs0)
    cp = _engine_run(tr, site, dtype, xs, mask, dy_seed, path="checkpoint")
    _equal_runs(cp, eager, f"{name} {NAME[dtype]} checkpoint")
    for n, b in cp["bufs"].items():
        if n.endswith("num_batches_tracked"):
            assert int(b) == int(bufs0[n]) + 2, n
        assert torch.equal(b, twice[n]), n
    _restore(tr, site, bufs0)


@pytest.mark.parametrize("dtype", PRECS)
@pytest.mark.parametrize("model,name", SITES)
def test_graph_replay_equals_eager(engines, model, name, dtype):
    from distributed_sod_project_b200 import syncbn
    tr, site, xs, mask, dy_seed, bufs0 = _setup(engines, model, name, dtype, seed=19)
    model, opt = tr.module, tr.optimizer
    mods = bs.modules(model, site)
    scale = FP16_SCALE if dtype == _F16 else 1.0
    static = [x.detach().clone().requires_grad_(ok) for x, ok in zip(xs, site.input_grad)]
    with torch.no_grad(), _autocast(dtype):
        out_shape_probe = site.run(mods, *[x.detach() for x in xs])
    _restore(tr, site, bufs0)
    dy_static = _upstream(out_shape_probe, dtype, dy_seed)[0].clone()
    m_static = mask.clone() if mask is not None else None

    def body():
        opt.flat.grad.zero_()
        if opt.flat.grad16 is not None:
            opt.flat.grad16.zero_()
        with _autocast(dtype):
            out = site.run(mods, *static)
        if site.loss:
            loss, scaled = _engine_loss(out, m_static, dtype)
            scaled.backward()
            return out, loss
        out.backward(dy_static)
        return out, None

    with _strict(dtype):
        _clear_grads(opt)
        for x in static:
            x.grad = None
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                body()
                for x in static:
                    x.grad = None
                opt.zero_grad()
        torch.cuda.current_stream().wait_stream(side)
        _restore(tr, site, bufs0)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        syncbn.begin_iteration(torch.device("cuda", torch.cuda.current_device()), graph=True)
        try:
            with torch.cuda.graph(graph):
                out_g, loss_g = body()
                syncbn.end_iteration(torch.device("cuda", torch.cuda.current_device()))
        finally:
            syncbn.begin_iteration(torch.device("cuda", torch.cuda.current_device()), graph=False)
        # the stolen 16-bit weight gradients live in the graph's memory; the eager runs in between rebind `.grad`
        stolen = [(leaf, leaf.grad) for leaf, _, steal in opt.flat.shadow_leaves if steal]
        _restore(tr, site, bufs0)
        for k, seed in enumerate((101, 202)):
            xs_k, mask_k, dy_seed_k = _operands(site, dtype, S, BATCH, seed)
            dy_k = _upstream(out_shape_probe, dtype, dy_seed_k)[0]
            _restore(tr, site, bufs0)
            eager = _engine_run(tr, site, dtype, xs_k, mask_k, dy_seed_k)
            _restore(tr, site, bufs0)
            with torch.no_grad():
                for s_, x in zip(static, xs_k):
                    s_.copy_(x)
                dy_static.copy_(dy_k)
                if m_static is not None:
                    m_static.copy_(mask_k)
            graph.replay()
            torch.cuda.synchronize()
            for leaf, g in stolen:
                leaf.grad = g
            rep = dict(out=out_g.detach(), dx=[x.grad.double() / scale for x in static], grads=_read_grads(tr, site, scale),
                       loss=None if loss_g is None else float(loss_g))
            _equal_runs(rep, eager, f"{_row_id(model, name)} {NAME[dtype]} graph replay {k}")
            for n, b in _site_buffers(model, site).items():
                assert torch.equal(b, eager["bufs"][n]), f"{name} replay {k}: {n}"
    del graph
    _restore(tr, site, bufs0)
    _clear_grads(opt)


def _walk(fn):
    """backward node name → how many are reachable from fn"""
    seen, stack, names = set(), [fn], collections.Counter()
    while stack:
        f = stack.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        names[type(f).__name__] += 1
        stack.extend(g for g, _ in f.next_functions)
    return names


@pytest.mark.parametrize("size", bs.SIZES)
@pytest.mark.parametrize("model,dtype", [pytest.param(m, d, id=_row_id(m, NAME[d])) for m in bs.ALL_MODELS for d in (_F32, _BF16)])
def test_dispatch_matches_site_table(engines, model, size, dtype):
    tr = engines(model, dtype)
    for site in bs.grid(model):
        bufs0 = {n: b.clone() for n, b in _site_buffers(tr.module, site).items()}
        xs, mask, _ = _operands(site, dtype, size, 1, 5)
        xs = [x.requires_grad_(ok) for x, ok in zip(xs, site.input_grad)]
        with _strict(dtype), _autocast(dtype):
            out = site.run(bs.modules(tr.module, site), *xs)
        if site.loss:
            out, _ = _engine_loss(out, mask, dtype)[1], None
        names = _walk(out.grad_fn)
        want = bs.dispatch(site, size, dtype != _F32, model)
        for node, present in want.items():
            assert (node in names) == present, (model, site.name, size, NAME[dtype], node, sorted(names))
        assert (bs.LOSS in names) == site.loss
        if site.kind == "neck":
            # one SyncBN node per BatchNorm, every nearest up-sample and average pool on the kernels (none of torch's)
            for node, k in bs.counts(site, dtype != _F32).items():
                assert names[node] == k, (model, site.name, size, NAME[dtype], node, names[node], k)
            assert names[bs.BN] == sum(isinstance(m, nn.BatchNorm2d) for m in tr.module.get_submodule(site.name).modules())
            assert not [n for n in names if "Upsample" in n or "AvgPool2D" in n], sorted(names)
        _restore(tr, site, bufs0)


# ---- seam cases on one SyncBatchNorm ---------------------------------------------------------------------------------
def _bn(c, seed=0):
    from distributed_sod_project_b200.syncbn import SyncBatchNorm
    g = torch.Generator().manual_seed(seed)
    bn = SyncBatchNorm(c).cuda()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        bn.bias.copy_(torch.randn(c, generator=g) * 0.2)
        bn.running_mean.copy_(torch.randn(c, generator=g) * 0.3)
        bn.running_var.copy_(torch.rand(c, generator=g) + 0.5)
    return bn


def _t(shape, dtype, seed, cl=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(shape, device="cuda", generator=g).to(dtype)
    return t.contiguous(memory_format=torch.channels_last) if cl else t.contiguous()


def _ref_bn(x, pre, res, cbs, bn, relu, training):
    """float64 autograd of act(BN(x + pre + Σ cb) + res), stock F.batch_norm"""
    d = lambda t: None if t is None else t.detach().double().requires_grad_()   # noqa: E731
    xx, pp, rr = d(x), d(pre), d(res)
    cc = [d(c) for c in cbs]
    w, b = d(bn.weight), d(bn.bias)
    z = xx if pp is None else xx + pp
    for c in cc:
        z = z + c.view(1, -1, 1, 1)
    rm, rv = bn.running_mean.detach().double().clone(), bn.running_var.detach().double().clone()
    y = F.batch_norm(z, rm, rv, w, b, training=training, momentum=bn.momentum, eps=bn.eps)
    if rr is not None:
        y = y + rr
    if relu:
        y = F.relu(y)
    return y, dict(x=xx, pre=pp, res=rr, w=w, b=b, cb=cc)


def _close(got, want, rtol, what):
    got, want = got.double(), want.double()
    err = float((got - want).abs().max())
    lim = rtol * max(float(want.abs().max()), 1e-30)
    assert err <= lim, f"{what}: max error {err:.3e} > {lim:.3e}"


@pytest.mark.parametrize("relu,use_pre,use_res,use_cb", [
    (False, False, False, False), (True, False, False, False), (True, True, False, True), (False, False, True, False),
    (True, False, True, False), (True, True, True, True)])
@pytest.mark.parametrize("dtype", [pytest.param(_F32, id="fp32"), pytest.param(_BF16, id="bf16")])
def test_eval_mode_backward_against_fp64_batch_norm(dtype, relu, use_pre, use_res, use_cb):
    """eval-mode SyncBatchNorm with grad: dz = dy·γ·rsqrt(running_var + eps) (ReLU-masked), dγ = Σ dy·x̂, dβ = Σ dy"""
    c = 64
    bn = _bn(c, 1).eval()
    x = _t((4, c, 12, 10), dtype, 1).requires_grad_()
    pre = _t((4, c, 12, 10), dtype, 2).requires_grad_() if use_pre else None
    res = _t((4, c, 12, 10), dtype, 3).requires_grad_() if use_res else None
    cbs = [(torch.randn(c, device="cuda") * 0.1).to(dtype).requires_grad_() for _ in range(2)] if use_cb else []
    rm0, rv0, nbt0 = bn.running_mean.clone(), bn.running_var.clone(), int(bn.num_batches_tracked)
    y = bn.fused_forward(x, pre_add=pre, residual=res, relu=relu, conv_bias=tuple(cbs) if cbs else (None, None))
    dy = _t(y.shape, dtype, 4)
    y.backward(dy)
    y64, leaves = _ref_bn(x, pre, res, cbs, bn, relu, training=False)
    y64.backward(dy.double())
    tol = 1e-5 if dtype == _F32 else 2e-2
    _close(y, y64, tol, "output")
    _close(x.grad, leaves["x"].grad, tol, "dx")
    if use_pre:
        _close(pre.grad, leaves["pre"].grad, tol, "dpre")
    if use_res:
        _close(res.grad, leaves["res"].grad, tol, "dres")
    _close(bn.weight.grad, leaves["w"].grad, 1e-4 if dtype == _F32 else 2e-2, "dgamma")
    _close(bn.bias.grad, leaves["b"].grad, 1e-4 if dtype == _F32 else 2e-2, "dbeta")
    for i, cb in enumerate(cbs):
        _close(cb.grad, leaves["cb"][i].grad, 1e-4 if dtype == _F32 else 2e-2, f"dcb{i}")
    assert torch.equal(bn.running_mean, rm0) and torch.equal(bn.running_var, rv0)
    assert int(bn.num_batches_tracked) == nbt0


@pytest.mark.parametrize("mode", ["returned", "direct", "gamma_frozen", "beta_frozen", "both_frozen"])
@pytest.mark.parametrize("cb_mode", ["temporary", "bound"])
def test_param_grad_paths_and_second_backward(mode, cb_mode):
    """BN γ/β through a bound fp32 .grad (the kernel adds into it) or returned to autograd, with either frozen; folded
    conv biases through a bound 16-bit .grad or a zeroed temporary.  A second backward without zeroing doubles them."""
    c, dtype = 64, _BF16
    bn = _bn(c, 2).train()
    bn.weight.requires_grad_(mode not in ("gamma_frozen", "both_frozen"))
    bn.bias.requires_grad_(mode not in ("beta_frozen", "both_frozen"))
    if mode == "direct":
        bn.weight.grad = torch.zeros(c, device="cuda")
        bn.bias.grad = torch.zeros(c, device="cuda")
    cbs = [(torch.randn(c, device="cuda") * 0.1).to(dtype).requires_grad_() for _ in range(2)]
    if cb_mode == "bound":
        for cb in cbs:
            cb.grad = torch.zeros_like(cb)
    x = _t((4, c, 16, 8), dtype, 5).requires_grad_()
    pre = _t((4, c, 16, 8), dtype, 6).requires_grad_()
    dy = _t((4, c, 16, 8), dtype, 7)
    runs = []
    for k in range(2):
        y = bn.fused_forward(x, pre_add=pre, relu=True, conv_bias=tuple(cbs))
        y.backward(dy)
        runs.append({"dx": x.grad.clone(), "dpre": pre.grad.clone(),
                     "dw": None if bn.weight.grad is None else bn.weight.grad.clone(),
                     "db": None if bn.bias.grad is None else bn.bias.grad.clone(),
                     "cb": [cb.grad.clone() for cb in cbs]})
    with torch.no_grad():
        bn.running_mean.zero_(); bn.running_var.fill_(1.0)
    y64, leaves = _ref_bn(x, pre, None, cbs, bn, True, training=True)
    y64.backward(dy.double())
    first, second = runs
    _close(first["dx"], leaves["x"].grad, 2e-2, "dx")
    assert torch.equal(first["dx"], first["dpre"])                                  # pre_add's gradient is dz
    for key, leaf, trains in (("dw", bn.weight, bn.weight.requires_grad), ("db", bn.bias, bn.bias.requires_grad)):
        if not trains:
            assert first[key] is None or mode == "direct", key
            continue
        _close(first[key], leaves["w" if key == "dw" else "b"].grad, 2e-2, key)
        assert torch.equal(second[key], 2 * first[key]), key                       # fp32: g + g is exact
        assert first[key].dtype == torch.float32
    assert torch.equal(first["cb"][0], first["cb"][1]) and float(first["cb"][0].abs().max()) > 0   # both get Σ dz
    for i, cb in enumerate(cbs):
        g1, g2 = first["cb"][i], second["cb"][i]
        # zero in exact arithmetic (training-mode BN): compare with the largest dz, not with itself
        assert float(g1.double().abs().max()) <= 1e-2 * float(first["dx"].double().abs().max()) * 4 * 16 * 8
        if cb_mode == "temporary":
            assert torch.equal(g2, 2 * g1), i                                      # autograd: round(g) + round(g)
        else:
            # the kernel adds its fp32 sum into the bf16 buffer: one rounding of 2g
            ulp = torch.finfo(dtype).eps * (2 * g1.float()).abs() + torch.finfo(dtype).tiny
            assert bool(((g2.float() - 2 * g1.float()).abs() <= ulp).all()), i
    assert torch.equal(second["dx"], 2 * first["dx"])


def test_residual_gradient_is_the_masked_upstream():
    bn = _bn(64, 3).train()
    for dtype in (_F32, _BF16, _F16):
        x = _t((4, 64, 8, 8), dtype, 8).requires_grad_()
        res = _t((4, 64, 8, 8), dtype, 9).requires_grad_()
        y = bn.fused_forward(x, residual=res, relu=True)
        dy = _t(y.shape, dtype, 10)
        y.backward(dy)
        assert torch.equal(res.grad, dy * (y > 0)), NAME[dtype]


def test_maxpool_backward_routes_to_the_window_maximum():
    """exact: with distinct fp32 inputs and integer upstream gradients, dx equals torch's max-pool backward bit for bit"""
    from distributed_sod_project_b200 import resample
    old = resample.ENABLED
    resample.ENABLED = True
    try:
        g = torch.Generator(device="cuda").manual_seed(12)
        x = torch.randperm(2 * 64 * 17 * 15, device="cuda", generator=g).float().view(2, 64, 17, 15)
        x = x.contiguous(memory_format=torch.channels_last).requires_grad_()
        y = resample.maxpool3x3s2(x)
        assert y is not None and type(y.grad_fn).__name__ == bs.MAX
        dy = torch.randint(-8, 9, y.shape, device="cuda", generator=g).float().contiguous(memory_format=torch.channels_last)
        y.backward(dy)
        x2 = x.detach().clone().requires_grad_()
        y2 = F.max_pool2d(x2, 3, 2, 1)
        y2.backward(dy)
        assert torch.equal(y, y2) and torch.equal(x.grad, x2.grad)
    finally:
        resample.ENABLED = old


def test_layouts_give_identical_results():
    """NCHW-contiguous and sliced (non-contiguous) inputs and an NCHW-contiguous dy are converted on entry: the results
    equal the channels-last run bit for bit"""
    bn = _bn(64, 4).train()
    dtype = _BF16
    big = _t((4, 64, 12, 12), dtype, 11, cl=False)
    views = {"channels_last": big[:, :, 1:-1, :].contiguous(memory_format=torch.channels_last),
             "nchw": big[:, :, 1:-1, :].contiguous(), "sliced": big[:, :, 1:-1, :]}
    assert not views["sliced"].is_contiguous() and not views["sliced"].is_contiguous(memory_format=torch.channels_last)
    dy_cl = _t((4, 64, 10, 12), dtype, 12)
    out = {}
    for name, v in views.items():
        for dyn, dy in (("dy_cl", dy_cl), ("dy_nchw", dy_cl.contiguous())):
            x = v.detach().clone() if name != "sliced" else big.detach().clone()[:, :, 1:-1, :]
            x.requires_grad_()
            bn.weight.grad = bn.bias.grad = None
            y = bn.fused_forward(x, relu=True)
            y.backward(dy)
            out[(name, dyn)] = (y.detach(), x.grad, bn.weight.grad.clone(), bn.bias.grad.clone())
    ref = out[("channels_last", "dy_cl")]
    for k, v in out.items():
        for a, b in zip(v, ref):
            assert torch.equal(a.contiguous(), b.contiguous()), k


def test_mixed_dtype_pre_add_and_residual_are_rounded_to_x_dtype():
    """a pre_add / residual of another dtype than x (as autocast can hand over) is rounded to x's dtype once on entry,
    where stock torch would promote the add to fp32; its gradient comes back in its own dtype, equal to dz / dres"""
    bn = _bn(64, 5).train()
    x = _t((4, 64, 8, 8), _BF16, 13)
    pre32 = _t((4, 64, 8, 8), _F32, 14).requires_grad_()
    res32 = _t((4, 64, 8, 8), _F32, 15).requires_grad_()
    dy = _t((4, 64, 8, 8), _BF16, 16)
    y = bn.fused_forward(x.requires_grad_(), pre_add=pre32, residual=res32, relu=True)
    y.backward(dy)
    x2 = x.detach().clone().requires_grad_()
    pre16, res16 = pre32.detach().to(_BF16).requires_grad_(), res32.detach().to(_BF16).requires_grad_()
    y2 = bn.fused_forward(x2, pre_add=pre16, residual=res16, relu=True)
    y2.backward(dy)
    assert y.dtype == _BF16 and torch.equal(y, y2)
    assert pre32.grad.dtype == _F32 and res32.grad.dtype == _F32
    assert torch.equal(pre32.grad, pre16.grad.float()) and torch.equal(res32.grad, res16.grad.float())
    assert torch.equal(x.grad, x2.grad)


class _ConvBN(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(16, 64, 3, 1, 1, bias=True)
        self.bn = nn.BatchNorm2d(64)

    def forward(self, x):
        from distributed_sod_project_b200.network.blocks import conv_bn_act
        return conv_bn_act(self.conv, self.bn, x)


@pytest.mark.parametrize("dtype", [pytest.param(_F32, id="fp32"), pytest.param(_BF16, id="bf16")])
def test_zero_grad_clears_a_folded_bias_only_backward(dtype):
    """BN affine frozen, conv bias trainable: the only write outside autograd's sight is the folded-bias gradient the
    SyncBN backward adds into the bound .grad.  After a step, such a backward and zero_grad, the next backward must see
    a clean buffer."""
    from distributed_sod_project_b200 import amp
    from distributed_sod_project_b200.optim import make_optimizer
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    torch.manual_seed(0)
    model = _ConvBN().cuda().to(memory_format=torch.channels_last)
    model.bn.weight.requires_grad_(False)
    model.bn.bias.requires_grad_(False)
    if dtype == _F32:
        model.conv.weight.requires_grad_(False)        # fp32: its gradient would go through autograd (a version bump)
    opt = make_optimizer(model, "sgd_all", dict(lr=0.0, momentum=0.0, weight_decay=0.0))
    model = convert_syncbn_model(model)
    try:
        if dtype != _F32:
            model, opt = amp.initialize(model, opt, opt_level="O1", dtype=dtype)
        f = opt.flat

        def bias_grad():
            return (f.view16(f.grad16, model.conv.bias) if dtype != _F32 else model.conv.bias.grad).float().clone()

        x = _t((4, 16, 8, 8), dtype, 17)
        dy = _t((4, 64, 8, 8), dtype, 18)
        opt.zero_grad()
        model(x).backward(dy)
        # zero in exact arithmetic (a bias folded into a training-mode BN), but the rounding noise is not, and the
        # backward is deterministic: a stale gradient shows as twice it
        once = bias_grad()
        assert float(once.abs().max()) > 0
        opt.step()
        model(x).backward(dy)                           # after the step: a write only the folded-bias path makes
        opt.zero_grad()
        model(x).backward(dy)
        assert torch.equal(bias_grad(), once), "stale folded-bias gradient survived zero_grad"
    finally:
        amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None, dev=None)


# ---- seam cases on conv3_bn_act: three convolutions into one SyncBatchNorm --------------------------------------------
_TRIPLE = ("h2m", "m2m", "l2m")
_GRAD_PATHS = ("bound32", "temporary", "bound16")


class _Triple(nn.Module):
    """Conv3nV1's `bnm_1` / `bnm_2`: three 3×3 64→64 convolutions summed into one BatchNorm by `conv3_bn_act`, which
    folds the first bias into the SyncBN kernel's first slot and `b2 + b3` (a non-leaf) into its second"""

    def __init__(self, nobias=None):
        super().__init__()
        for name in _TRIPLE:
            setattr(self, name, nn.Conv2d(64, 64, 3, 1, 1, bias=name != nobias))
        self.bnm = nn.BatchNorm2d(64)

    def forward(self, h, m, l):  # noqa: E741
        from distributed_sod_project_b200.network.blocks import conv3_bn_act
        return conv3_bn_act(self.h2m, self.bnm, h, (self.m2m, m), (self.l2m, l))


def _triple(path, variant="all", frozen_affine=False):
    """(model, optimizer | None, activation dtype): a `_Triple` converted as the Trainer converts it.  `path`: where the
    bias gradients go — "bound32" (FusedSGD binds every .grad to its fp32 flat buffer), "bound16" (bf16 amp: the
    biases are 16-bit shadows whose .grad is bound to the 16-bit flat buffer) or "temporary" (no optimizer: the kernel
    adds into zeroed temporaries that autograd accumulates).  `variant`: "all", "<conv>_frozen" or "<conv>_nobias"."""
    from distributed_sod_project_b200 import amp
    from distributed_sod_project_b200.optim import make_optimizer
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    torch.manual_seed(40)
    model = _Triple(nobias=variant[:3] if variant.endswith("_nobias") else None).cuda()
    model = model.to(memory_format=torch.channels_last)
    with torch.no_grad():
        model.bnm.weight.uniform_(0.5, 1.5)
        model.bnm.bias.normal_(0.0, 0.2)
        model.bnm.running_mean.normal_(0.0, 0.3)
        model.bnm.running_var.uniform_(0.5, 1.5)
    if variant.endswith("_frozen"):
        getattr(model, variant[:3]).bias.requires_grad_(False)
    if frozen_affine:
        model.bnm.requires_grad_(False)
    opt = None if path == "temporary" else make_optimizer(model, "sgd_all", dict(lr=0.0, momentum=0.0, weight_decay=0.0))
    model = convert_syncbn_model(model)
    if path == "bound16":
        model, opt = amp.initialize(model, opt, opt_level="O1", dtype=_BF16)
        return model, opt, _BF16
    return model, opt, _F32


def _triple_inputs(dtype, seed):
    """non-negative h, m, l (the neck's operands are post-ReLU maps) and dy, channels-last"""
    return [_t((4, 64, 16, 16), _F32, seed + k).relu().to(dtype) for k in range(3)], _t((4, 64, 16, 16), dtype, seed + 3)


def _triple_bias_grads(model, opt):
    """conv name → its bias gradient where the fused step reads it (None: no gradient was made)"""
    out = {}
    for name in _TRIPLE:
        b = getattr(model, name).bias
        if b is None:
            continue
        if getattr(getattr(model, name), "_sod_b16", None) is not None:
            out[name] = opt.flat.view16(opt.flat.grad16, b).clone()
        else:
            out[name] = None if b.grad is None else b.grad.clone()
    return out


def _amp_off():
    from distributed_sod_project_b200 import amp
    amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None, dev=None)


@pytest.mark.parametrize("variant", ["all", "m2m_frozen", "l2m_frozen", "h2m_nobias", "m2m_nobias", "l2m_nobias"])
@pytest.mark.parametrize("train", [pytest.param(True, id="train"), pytest.param(False, id="eval")])
def test_conv3_folded_biases_get_the_same_bits(train, variant):
    """every trainable bias of the three gets the same bits of Σ dz — the first through the kernel's first slot, the
    other two through `b2 + b3` in the second (autograd routes that slot's gradient on) — whether the .grad is bound
    fp32, bound 16-bit or a temporary, with `b2` or `b3` frozen or one convolution without a bias (so the second slot is
    a leaf); a frozen bias gets nothing.  The fp32 bound and temporary paths give the same bits.  In eval mode Σ dz is
    not zero in exact arithmetic: it must be within rounding of Σ dy·[y > 0]·γ/√(running_var + eps) in float64."""
    got = {}
    for path in _GRAD_PATHS:
        model, opt, dtype = _triple(path, variant)
        try:
            model.train(train)
            if opt is not None:
                _clear_grads(opt)
            (h, m, l), dy = _triple_inputs(dtype, 41)  # noqa: E741
            y = model(h, m, l)
            y.backward(dy)
            grads = _triple_bias_grads(model, opt)
        finally:
            _amp_off()
        trainable = [n for n in _TRIPLE if getattr(model, n).bias is not None and getattr(model, n).bias.requires_grad]
        assert len(trainable) == (3 if variant == "all" else 2)
        for n in set(grads) - set(trainable):                       # frozen: its buffer untouched, or no .grad at all
            assert grads[n] is None or float(grads[n].abs().max()) == 0.0, (path, n)
        first = grads[trainable[0]]
        assert first.dtype == dtype and float(first.abs().max()) > 0, path
        for n in trainable[1:]:
            assert torch.equal(grads[n], first), f"{path} {variant}: {n} differs from {trainable[0]}"
        if not train:
            bn = model.bnm
            scale = bn.weight.detach().double() / torch.sqrt(bn.running_var.double() + bn.eps)
            want = (dy.double() * (y.detach() > 0) * scale.view(1, -1, 1, 1)).sum(dim=(0, 2, 3))
            _close(first, want, 1e-4 if dtype == _F32 else 2e-2, f"{path} eval Σ dz")
        got[path] = first
    assert torch.equal(got["bound32"], got["temporary"])


@pytest.mark.parametrize("path", _GRAD_PATHS)
def test_conv3_second_backward_doubles_the_bias_gradients(path):
    """a second backward without zeroing doubles every bias gradient: exactly where autograd adds g + g (fp32, and the
    16-bit .grad of `b2` / `b3`, which autograd accumulates from the second slot's temporary), within one rounding of
    the 16-bit type where the kernel adds its fp32 Σ dz into the bound 16-bit .grad of `b1`"""
    model, opt, dtype = _triple(path)
    try:
        if opt is not None:
            _clear_grads(opt)
        (h, m, l), dy = _triple_inputs(dtype, 45)  # noqa: E741
        runs = []
        for _ in range(2):
            model(h, m, l).backward(dy)
            runs.append(_triple_bias_grads(model, opt))
    finally:
        _amp_off()
    first, second = runs
    assert all(torch.equal(first[n], first["h2m"]) for n in _TRIPLE)
    for n in _TRIPLE:
        if dtype == _F32 or n != "h2m":
            assert torch.equal(second[n], 2 * first[n]), (path, n)
        else:
            g1, g2 = first[n].float(), second[n].float()
            assert bool(((g2 - 2 * g1).abs() <= torch.finfo(dtype).eps * (2 * g1).abs() + torch.finfo(dtype).tiny).all())


@pytest.mark.parametrize("dtype", [pytest.param(_F32, id="fp32"), pytest.param(_BF16, id="bf16")])
def test_zero_grad_clears_a_backward_through_the_non_leaf_bias_slot(dtype):
    """γ/β and `b1` frozen (and, in fp32, the weights): the only gradient writes of the backward are `b2`'s and `b3`'s,
    which autograd accumulates from conv3_bn_act's second slot.  After a step, such a backward and zero_grad, the next
    backward must see a clean buffer."""
    model, opt, _ = _triple("bound16" if dtype == _BF16 else "bound32", "h2m_frozen", frozen_affine=True)
    try:
        if dtype == _F32:
            for n in _TRIPLE:
                getattr(model, n).weight.requires_grad_(False)
        (h, m, l), dy = _triple_inputs(dtype, 47)  # noqa: E741
        opt.zero_grad()
        model(h, m, l).backward(dy)
        once = _triple_bias_grads(model, opt)
        assert float(once["m2m"].abs().max()) > 0 and torch.equal(once["m2m"], once["l2m"])
        opt.step()
        model(h, m, l).backward(dy)                     # after the step: writes only the non-leaf slot makes
        opt.zero_grad()
        model(h, m, l).backward(dy)
        again = _triple_bias_grads(model, opt)
        for n in ("m2m", "l2m"):
            assert torch.equal(again[n], once[n]), f"stale {n} bias gradient survived zero_grad"
    finally:
        _amp_off()


@pytest.mark.parametrize("shadowed", [pytest.param(("h2m",), id="b1_16bit"), pytest.param(("m2m", "l2m"), id="b23_16bit"),
                                      pytest.param(("h2m", "m2m"), id="b1_b2_16bit")])
def test_conv3_biases_of_mixed_dtypes_are_refused(shadowed):
    """the SyncBN kernel reads both folded-bias slots under one dtype code, so a conv3_bn_act call whose slots would hold
    biases of different dtypes raises SodError before any launch.  (`b2 + b3` of two dtypes is promoted by the add, so
    what counts is the two slots.)  amp does not produce the case: `test_amp_gives_every_neck_bias_one_dtype`."""
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    torch.manual_seed(42)
    model = convert_syncbn_model(_Triple().cuda().to(memory_format=torch.channels_last))
    for n in shadowed:                              # a 16-bit shadow on some of the three only, as amp never leaves it
        conv = getattr(model, n)
        conv._sod_w16 = conv.weight.detach().to(_BF16).requires_grad_()
        conv._sod_b16 = conv.bias.detach().to(_BF16).requires_grad_()
    (h, m, l), _ = _triple_inputs(_BF16, 49)  # noqa: E741
    launches = _lib.launches
    with torch.autocast("cuda", dtype=_BF16), pytest.raises(_lib.SodError, match="share a dtype"):
        model(h, m, l)
    assert _lib.launches == launches


def test_amp_gives_every_neck_bias_one_dtype(engines):
    """under amp every biased convolution of the LightAIM neck has a 16-bit shadow bias of the activation dtype, so no
    conv_bn_act / conv3_bn_act call of the neck hands the SyncBN kernel biases of two dtypes"""
    for dtype in (_BF16, _F16):
        tr = engines("aim_res50", dtype)
        convs = [m for m in tr.module.trans.modules() if isinstance(m, nn.Conv2d)]
        assert convs and all(c.bias is not None for c in convs)
        assert all(getattr(c, "_sod_b16", None) is not None and c._sod_b16.dtype == dtype for c in convs)


# ---- seam cases on one GroupNorm32 and the weight-standardised convolutions -------------------------------------------
def _gn(c, seed=0):
    from distributed_sod_project_b200.wsgn import GroupNorm32
    g = torch.Generator().manual_seed(seed)
    gn = GroupNorm32(32, c).cuda()
    with torch.no_grad():
        gn.weight.copy_(torch.rand(c, generator=g) + 0.5)
        gn.bias.copy_(torch.randn(c, generator=g) * 0.2)
    return gn


def _ref_gn(x, res, gn, relu):
    """float64 autograd of act(GroupNorm(32)(x) + res), res rounded to x's dtype first as the kernel takes it"""
    xx = x.detach().double().requires_grad_()
    w, b = gn.weight.detach().double().requires_grad_(), gn.bias.detach().double().requires_grad_()
    y = F.group_norm(xx, 32, w, b, gn.eps)
    if res is not None:
        y = y + res.detach().to(x.dtype).double()
    return (F.relu(y) if relu else y), xx, w, b


_GN_TOL = {_F32: 1e-5, _BF16: 2e-2, _F16: 4e-3}


@pytest.mark.parametrize("x_dtype,res_dtype", [
    pytest.param(d, r, id=f"x_{NAME[d]}-res_{NAME[r]}")
    for d, r in ((_F32, _F32), (_BF16, _BF16), (_F16, _F16), (_BF16, _F32), (_F16, _F32), (_F32, _BF16))])
def test_groupnorm_residual_gradient_is_the_masked_upstream(x_dtype, res_dtype):
    """GroupNorm32 with the bottleneck's residual and ReLU: the output is in x's dtype (the residual rounded to it once on
    entry); the residual's gradient is exactly the ReLU-masked upstream, handed back in the residual's own dtype.  Output,
    dx, dγ and dβ against float64."""
    gn = _gn(64, 1)
    x = _t((4, 64, 8, 8), x_dtype, 20).requires_grad_()
    res = _t((4, 64, 8, 8), res_dtype, 21).requires_grad_()
    y = gn.fused_forward(x, residual=res, relu=True)
    assert y.dtype == x_dtype and type(y.grad_fn).__name__ == bs.GN
    dy = _t(y.shape, x_dtype, 22)
    y.backward(dy)
    assert res.grad.dtype == res_dtype
    assert torch.equal(res.grad, (dy * (y > 0)).to(res_dtype))
    y64, x64, w64, b64 = _ref_gn(x, res, gn, relu=True)
    y64.backward(dy.double())
    tol = _GN_TOL[x_dtype]
    _close(y, y64, tol, "output")
    _close(x.grad, x64.grad, tol, "dx")
    _close(gn.weight.grad, w64.grad, max(tol, 1e-4), "dgamma")
    _close(gn.bias.grad, b64.grad, max(tol, 1e-4), "dbeta")


@pytest.mark.parametrize("scale", [pytest.param(2.0 ** -6, id="var_2e-4"), pytest.param(2.0 ** -10, id="var_1e-6")])
@pytest.mark.parametrize("dtype", [pytest.param(_F32, id="fp32"), pytest.param(_BF16, id="bf16")])
def test_groupnorm_takes_the_module_eps(dtype, scale):
    """at a group variance near eps (x of std 2⁻⁶ and 2⁻¹⁰ against eps = 1e-5) the output and every gradient depend on
    eps at first order: GroupNorm32 against float64 GroupNorm with the module's eps"""
    gn = _gn(64, 7)
    x = (_t((4, 64, 8, 8), _F32, 35) * scale).to(dtype).detach().requires_grad_()
    y = gn.fused_forward(x)
    dy = _t(y.shape, dtype, 36)
    y.backward(dy)
    y64, x64, w64, b64 = _ref_gn(x, None, gn, relu=False)
    y64.backward(dy.double())
    tol = _GN_TOL[dtype]
    _close(y, y64, tol, "output")
    _close(x.grad, x64.grad, tol, "dx")
    _close(gn.weight.grad, w64.grad, max(tol, 1e-4), "dgamma")
    _close(gn.bias.grad, b64.grad, max(tol, 1e-4), "dbeta")


def test_groupnorm_layouts_give_identical_results():
    """NCHW-contiguous and sliced (non-contiguous) x, residual and dy are converted on entry: the GroupNorm results equal
    the channels-last run bit for bit"""
    gn = _gn(64, 2)
    dtype = _BF16
    big = _t((4, 64, 12, 12), dtype, 26, cl=False)
    big_res = _t((4, 64, 12, 12), dtype, 27, cl=False)
    dy_cl = _t((4, 64, 10, 12), dtype, 28)

    def views(t):
        return {"channels_last": t[:, :, 1:-1, :].contiguous(memory_format=torch.channels_last),
                "nchw": t[:, :, 1:-1, :].contiguous(), "sliced": t.detach().clone()[:, :, 1:-1, :]}
    assert not views(big)["sliced"].is_contiguous(memory_format=torch.channels_last)
    out = {}
    for name in ("channels_last", "nchw", "sliced"):
        for dyn, dy in (("dy_cl", dy_cl), ("dy_nchw", dy_cl.contiguous())):
            x, res = views(big)[name].requires_grad_(), views(big_res)[name].requires_grad_()
            gn.weight.grad = gn.bias.grad = None
            y = gn.fused_forward(x, residual=res, relu=True)
            y.backward(dy)
            out[(name, dyn)] = (y.detach(), x.grad, res.grad, gn.weight.grad.clone(), gn.bias.grad.clone())
    ref = out[("channels_last", "dy_cl")]
    for k, v in out.items():
        for a, b in zip(v, ref):
            assert torch.equal(a.contiguous(), b.contiguous()), k


@pytest.mark.parametrize("mode", ["direct", "gamma_frozen", "beta_frozen", "both_frozen"])
def test_groupnorm_param_grad_paths_and_second_backward(mode):
    """γ/β gradients the kernel adds into bound fp32 .grad buffers (as the fused optimizers bind them) equal, bit for bit,
    those it hands back to autograd; with γ, β or both frozen the trainable one comes back through autograd into its
    bound .grad and a frozen one's stays untouched.  A second backward without zeroing doubles every gradient exactly."""
    c, dtype = 64, _BF16
    x0, res0, dy = _t((4, c, 16, 8), dtype, 23), _t((4, c, 16, 8), dtype, 24), _t((4, c, 16, 8), dtype, 25)

    def run(gn, k):
        x, res = x0.detach().clone().requires_grad_(), res0.detach().clone().requires_grad_()
        runs = []
        for _ in range(k):
            y = gn.fused_forward(x, residual=res, relu=True)
            y.backward(dy)
            runs.append({"y": y.detach(), "dx": x.grad.clone(), "dres": res.grad.clone(),
                         "dw": None if gn.weight.grad is None else gn.weight.grad.clone(),
                         "db": None if gn.bias.grad is None else gn.bias.grad.clone()})
        return runs

    from distributed_sod_project_b200 import _lib
    ref = run(_gn(c, 6), 1)[0]                                  # both trainable, nothing bound: returned to autograd
    y64, x64, w64, b64 = _ref_gn(x0, res0, _gn(c, 6), relu=True)
    y64.backward(dy.double())
    _close(ref["dw"], w64.grad, 2e-2, "dgamma")
    _close(ref["db"], b64.grad, 2e-2, "dbeta")
    gn = _gn(c, 6)
    gn.weight.requires_grad_(mode not in ("gamma_frozen", "both_frozen"))
    gn.bias.requires_grad_(mode not in ("beta_frozen", "both_frozen"))
    for p in (gn.weight, gn.bias):
        p.grad = torch.zeros_like(p)
    writes = _lib.grad_writes
    first, second = run(gn, 2)
    assert (_lib.grad_writes > writes) == (mode == "direct")
    for key, p in (("dw", gn.weight), ("db", gn.bias)):
        if p.requires_grad:
            assert torch.equal(first[key], ref[key]), key
            assert torch.equal(second[key], 2 * ref[key]), key                   # fp32: g + g is exact
        else:
            assert float(first[key].abs().max()) == 0.0 and float(second[key].abs().max()) == 0.0, key
    for key in ("y", "dx", "dres"):
        assert torch.equal(first[key], ref[key]), key
    assert torch.equal(second["dx"], 2 * ref["dx"]) and torch.equal(second["dres"], 2 * ref["dres"])


def _fused_ws(cin, cout, stride, groups, seed):
    from distributed_sod_project_b200 import wsgn
    from distributed_sod_project_b200.network.blocks import WSConv2d
    torch.manual_seed(seed)
    conv = WSConv2d(cin, cout, 3, stride, 1, groups=groups, bias=False).cuda().to(memory_format=torch.channels_last)
    return wsgn.convert_wsgn_model(conv)


@pytest.mark.parametrize("bound", [pytest.param(False, id="returned"), pytest.param(True, id="bound")])
@pytest.mark.parametrize("groups", [pytest.param(1, id="ws"), pytest.param(32, id="ws_gconv")])
def test_ws_weight_grad_paths_and_second_backward(groups, bound):
    """the weight gradient of a WS convolution (`_WSFn` after cuDNN; `_WSGroupConvFn` for the 32-group 3×3 on the
    kernels) is the same bit for bit whether the kernel adds it into a bound fp32 .grad or returns it to autograd, close to
    float64, and a second backward without zeroing doubles it exactly"""
    from distributed_sod_project_b200 import _lib
    c = 256 if groups > 1 else 64                           # 8 channels per group at stride 2: csrc/gconv.cu
    conv = _fused_ws(c, c, 2, groups, 30)
    x0, dtype = _t((2, c, 16, 12), _BF16, 31), _BF16

    def run(k, bind):
        conv.weight.grad = torch.zeros_like(conv.weight) if bind else None
        x = x0.detach().clone().requires_grad_()
        runs = []
        for _ in range(k):
            with torch.autocast("cuda", dtype=dtype):
                y = conv(x)
            names = _walk(y.grad_fn)
            assert (bs.WSG in names) == (groups > 1) and (bs.WS in names) == (groups == 1), names
            y.backward(_t(y.shape, dtype, 32))
            runs.append((x.grad.clone(), conv.weight.grad.clone()))
        return runs

    writes = _lib.grad_writes
    (dx_ref, dw_ref), = run(1, False)
    assert _lib.grad_writes == writes                       # nothing bound: returned to autograd
    (dx1, dw1), (dx2, dw2) = run(2, bound)                  # unbound: autograd's .grad is bound from the second on
    assert _lib.grad_writes > writes
    assert torch.equal(dx1, dx_ref) and torch.equal(dw1, dw_ref)
    assert torch.equal(dx2, 2 * dx_ref) and torch.equal(dw2, 2 * dw_ref)
    assert dw1.dtype == torch.float32
    # float64: the same x and dy through the stock WSConv2d
    w64 = conv.weight.detach().double().requires_grad_()
    wt = types.SimpleNamespace(weight=w64, eps=conv.eps)
    y64 = F.conv2d(x0.double(), type(conv).standardized_weight(wt), None, 2, 1, 1, groups)
    y64.backward(_t(y64.shape, dtype, 32).double())
    _close(dw1, w64.grad, 2e-2, "dW")


class _WSGN(nn.Module):
    def __init__(self):
        super().__init__()
        from distributed_sod_project_b200.network.blocks import WSConv2d
        self.conv = WSConv2d(16, 64, 3, 1, 1, bias=False)
        self.gn = nn.GroupNorm(32, 64)

    def forward(self, x):
        from distributed_sod_project_b200.network.blocks import bn_act
        return bn_act(self.gn, self.conv(x))


@pytest.mark.parametrize("trains", ["gn", "ws", "both"])
@pytest.mark.parametrize("dtype", [pytest.param(_F32, id="fp32"), pytest.param(_BF16, id="bf16")])
def test_zero_grad_clears_a_groupnorm_or_ws_only_backward(dtype, trains):
    """a backward whose only gradient writes are the GroupNorm and / or WS kernels' adds into the bound fp32 .grad
    (input without gradient; the other module frozen): after a step, such a backward and zero_grad, the next backward
    must see a clean buffer"""
    from distributed_sod_project_b200 import amp, wsgn
    from distributed_sod_project_b200.optim import make_optimizer
    from distributed_sod_project_b200.syncbn import convert_syncbn_model
    torch.manual_seed(1)
    model = _WSGN().cuda().to(memory_format=torch.channels_last)
    with torch.no_grad():
        model.gn.weight.uniform_(0.5, 1.5)
        model.gn.bias.normal_(0, 0.2)
    if trains == "ws":
        model.gn.requires_grad_(False)
    if trains == "gn":
        model.conv.requires_grad_(False)
    opt = make_optimizer(model, "sgd_all", dict(lr=0.0, momentum=0.0, weight_decay=0.0))
    model = wsgn.convert_wsgn_model(convert_syncbn_model(model))
    try:
        if dtype != _F32:
            model, opt = amp.initialize(model, opt, opt_level="O1", dtype=dtype)
        params = [p for p in model.parameters() if p.requires_grad]
        assert params

        def grads():
            return [p.grad.clone() for p in params]

        x = _t((4, 16, 8, 8), dtype, 33)
        dy = _t((4, 64, 8, 8), dtype, 34)
        opt.zero_grad()
        model(x).backward(dy)
        once = grads()
        assert all(float(g.abs().max()) > 0 for g in once)
        opt.step()
        model(x).backward(dy)                           # after the step: writes only the kernels' adds make
        opt.zero_grad()
        model(x).backward(dy)
        for g, g1 in zip(grads(), once):
            assert torch.equal(g, g1), "stale GroupNorm / WS gradient survived zero_grad"
    finally:
        amp._cfg.update(enabled=False, dynamic=False, scale=1.0, good_steps=0, growth_interval=2000, owner=None, dev=None)


def test_report(engines):
    """prints the measured table (the module docstring quotes it); runs last"""
    if not RESULTS:
        pytest.skip("no grid case ran")
    import json
    import os
    lines = ["site precision path worst_e2_ratio worst_emax_ratio stock_median_e2 max_e2_bound"]
    for r in RESULTS:
        lines.append(" ".join(str(v) if isinstance(v, str) else f"{v:.3e}" for v in r))
    print("\n" + "\n".join(lines))
    out = os.environ.get("SOD_BLOCK_SEAMS_REPORT")
    if out:
        with open(out, "w") as fh:
            json.dump(RESULTS, fh)
