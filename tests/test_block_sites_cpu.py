"""The block-site tables of oracle/block_sites.py against the models they cut up (CPU only), for each of the five
models (`res50`, `vgg16`, `wsgn_res50`, `wsgn_resnext50`, `aim_res50`):

* every parameter and buffer of the model belongs to exactly one site;
* the sites, run one after the other, are the model's forward bit for bit (fp32, stock modules) and leave the same
  norm buffers behind;
* the site shapes are what the model feeds its modules;
* `dispatch` — which of the engine's resampling / max-pool / nearest / column-sum / GroupNorm / weight-standardisation
  kernels each site reaches (and, for the LightAIM neck sites, `counts`: how often) — agrees with the predicates of `resample.py`, `wsgn.py` and `network/blocks.py` at 256², 288², 320², 352²
  and 384².  The forward runs on CPU tensors that report `is_cuda`, through the engine's own GroupNorm and WS modules
  (`convert_wsgn_model`), with the kernels' autograd Functions (and `wsgn.standardize_weight`, whose `is_cuda` check
  reads the CPU weight) replaced by recorders that hand back the torch result, so the predicates are evaluated exactly
  as the engine evaluates them.
"""
import contextlib
import copy
import types

import pytest
import torch
import torch.nn.functional as F

from oracle import block_sites as bs


MODELS = list(bs.ALL_MODELS)
PLUGINS = [m for m in MODELS if m != "res50"]      # res50's checks keep their own (older) test names
RESNET_BACKBONE = ["stem", "pool+div_4.1.0", "div_4.1.1", "div_8.0", "div_8.1", "div_16.0", "div_16.1", "div_32.0",
                   "div_32.1"]
DECODER = [f"{k}{s}" for k in ("trans", "sim", "upconv") for s in bs.TAPS] + [f"upsample_add{s}" for s in bs.TAPS[1:]] + \
    ["head"]
NECK = [f"trans.conv{i}" for i in range(5)]


def _model(name="res50"):
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return getattr(network, name)()


def _ownership(name):
    model = _model(name)
    names = [n for n, _ in model.named_parameters()] + [n for n, _ in model.named_buffers()]
    assert len(names) > (150 if name == "vgg16" else 350)
    for n in names:
        assert len(bs.owner(n, name)) == 1, (n, bs.owner(n, name))
    table = bs.sites(name)
    assert len({s.name for s in table}) == len(table)
    # every site's paths exist, and the representative ones are those the GPU grid runs (the WS-GN rows without their
    # decoder, which is res50's)
    for s in table:
        bs.modules(model, s)
    rep = [s.name for s in table if s.representative]
    backbone = [f"div_{s}" for s in reversed(bs.TAPS)] if name == "vgg16" else RESNET_BACKBONE
    if name == "aim_res50":                          # the neck in place of trans*; the grid runs the neck alone
        assert rep == backbone + NECK + [d for d in DECODER if not d.startswith("trans")]
        assert [s.name for s in bs.grid(name)] == NECK
        return
    assert rep == backbone + DECODER
    assert [s.name for s in bs.grid(name)] == (backbone if name in bs.WSGN else rep)


def test_every_parameter_and_buffer_belongs_to_exactly_one_site():
    _ownership("res50")


@pytest.mark.parametrize("name", PLUGINS)
def test_every_parameter_and_buffer_of_a_plugin_belongs_to_exactly_one_site(name):
    _ownership(name)


def _compose(name):
    model = _model(name).train()
    twin = copy.deepcopy(model)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = model(x)
        got = bs.compose(twin, x, name)
    assert want.shape == (2, 1, 64, 64)
    assert torch.equal(got, want)
    bufs = list(model.named_buffers())
    assert bufs and len(bufs) == len(list(twin.named_buffers()))
    for (n, a), (_, b) in zip(bufs, twin.named_buffers()):
        assert torch.equal(a, b), n


def test_sites_compose_to_the_model_forward_bit_for_bit():
    _compose("res50")


@pytest.mark.parametrize("name", PLUGINS)
def test_plugin_sites_compose_to_the_model_forward_bit_for_bit(name):
    _compose(name)


def _shapes(name):
    model = _model(name).eval()
    seen = {}
    table = bs.by_name(name)

    def hook(name):
        def fn(mod, args):
            seen.setdefault(name, [tuple(a.shape) for a in args])
        return fn

    for s in bs.sites(name):
        if s.paths and s.kind not in ("head",):
            model.get_submodule(s.paths[0]).register_forward_pre_hook(hook(s.name))
    model.get_submodule("upconv1").register_forward_pre_hook(hook("upconv1"))
    def head_input(mod, args, out):                   # the head's input d2 is upconv2's output
        seen.setdefault("head", [tuple(out.shape)])

    model.get_submodule("upconv2").register_forward_hook(head_input)
    with torch.no_grad():
        model(torch.zeros(1, 3, 128, 128))
    assert len(seen) == len([s for s in bs.sites(name) if s.paths]) + 1, sorted(seen)
    for site, shape in seen.items():
        if site == "upconv1":
            assert shape == [(1, 32, 128, 128)]              # res50 up-samples d2 ×2 first, vgg16 does not
        else:
            assert shape == [tuple(sh) for sh in table[site].shapes(128, 1)], site


def test_site_shapes_are_what_the_model_feeds_them():
    _shapes("res50")


@pytest.mark.parametrize("name", PLUGINS)
def test_plugin_site_shapes_are_what_the_model_feeds_them(name):
    _shapes(name)


class _Cudaish(torch.Tensor):
    """a CPU tensor that says it is on CUDA, so that the engine's dispatch predicates run as they do on the GPU"""

    @property
    def is_cuda(self):
        return True


@contextlib.contextmanager
def _recording():
    """resample.ENABLED on; every kernel autograd Function (and `wsgn.standardize_weight`) replaced by a recorder
    returning the torch result"""
    from distributed_sod_project_b200 import resample, wsgn
    from distributed_sod_project_b200.network import blocks
    taken = []

    def gn(x, res, w, b, eps, relu):
        y = F.group_norm(x, 32, w, b, eps) + (0 if res is None else res)
        return F.relu(y) if relu else y

    def std(w):
        return blocks.WSConv2d.standardized_weight(types.SimpleNamespace(weight=w, eps=blocks.WSConv2d.eps))

    torch_op = {
        (resample, "_Up2x"): lambda x, add: F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False) + (0 if add is None else add),
        (resample, "_AvgPool2x2"): lambda x: F.avg_pool2d(x, 2, 2),
        (resample, "_MaxPool3x3s2"): lambda x: F.max_pool2d(x, 3, 2, 1),
        (resample, "_MaxPool2x2s2"): lambda x: F.max_pool2d(x, 2, 2),
        (resample, "_ConvBias"): lambda x, w, b, *conf: F.conv2d(x, w, b, *conf),
        (resample, "_UpNearest2x"): lambda x: F.interpolate(x, scale_factor=2, mode="nearest"),
        (wsgn, "_GroupNormFn"): gn,
        (wsgn, "_WSGroupConvFn"): lambda x, w, dtype, eps, stride: F.conv2d(x, std(w), None, stride, 1, 1, 32),
    }
    saved = {k: getattr(*k).apply for k in torch_op}
    saved_std = wsgn.standardize_weight
    old = resample.ENABLED, resample.MAXPOOL_ENABLED, resample.COLSUM_ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    try:
        for (mod, n), op in torch_op.items():
            def rec(*a, n=n, op=op):
                taken.append(n + "Backward")
                return op(*a)
            setattr(getattr(mod, n), "apply", rec)

        def standardize(w, dtype, eps=1e-5):
            assert dtype == w.dtype and eps == blocks.WSConv2d.eps
            taken.append("_WSFnBackward")
            return std(w)
        wsgn.standardize_weight = standardize
        resample.ENABLED = resample.MAXPOOL_ENABLED = resample.COLSUM_ENABLED = True
        yield taken
    finally:
        for (mod, n), fn in saved.items():
            setattr(getattr(mod, n), "apply", fn)
        wsgn.standardize_weight = saved_std
        resample.ENABLED, resample.MAXPOOL_ENABLED, resample.COLSUM_ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old


@pytest.mark.parametrize("name,size", [pytest.param(m, z, id=str(z) if m == "res50" else f"{m}-{z}")   # res50's ids predate
                                       for m in MODELS for z in bs.SIZES])                               # the other rows
def test_dispatch_matches_the_engine_predicates(name, size):
    from distributed_sod_project_b200 import resample, wsgn
    model = wsgn.convert_wsgn_model(_model(name).eval())
    assert any(isinstance(m, (wsgn.GroupNorm32, wsgn.FusedWSConv2d)) for m in model.modules()) == (name in bs.WSGN)
    odd = size in (288, 352)
    assert odd == bool((size // 32) % 2)
    for site in bs.sites(name):
        if not site.representative:
            continue
        mods = bs.modules(model, site)
        xs = [torch.zeros(sh).as_subclass(_Cudaish) for sh in site.shapes(size, 1)]
        with _recording() as taken, torch.no_grad():
            site.run(mods, *xs)
        want = bs.dispatch(site, size, False, name)
        got = set(taken)
        for node in (bs.UP, bs.AVG, bs.MAX, bs.MAX2, bs.GN, bs.WS, bs.WSG, bs.NEAR):
            assert (node in got) == want[node], (name, site.name, size, node, taken)
        assert bs.CONVB not in got                       # plain convolutions never take conv_bias
        if site.kind == "neck":                          # stock BatchNorms here: the SyncBN count is the GPU walk's
            for node in (bs.NEAR, bs.AVG):
                assert taken.count(node) == bs.counts(site, False)[node], (site.name, size, node, taken)
        if site.kind == "sim":
            assert want[bs.UP] == want[bs.AVG] == (name == "vgg16" or not odd or site.stride != 32)
        # under amp the shadow-weight forward offers every biased convolution called as a module to `conv_bias`: all of
        # those of trans* and the head, the neck's 1×1 `identity` alone (its 3×3 ones fold their biases into the SyncBN
        # kernel)
        with _recording() as taken, torch.no_grad(), torch.enable_grad():
            for p, m in mods.items():
                for cname, conv in m.named_modules():
                    as_module = site.kind in ("trans", "head") or (site.kind == "neck" and cname == "identity")
                    if isinstance(conv, torch.nn.Conv2d) and conv.bias is not None and as_module:
                        w = conv.weight.detach().to(torch.bfloat16).as_subclass(_Cudaish)
                        x = torch.zeros(1, conv.in_channels, 4, 4, dtype=torch.bfloat16).as_subclass(_Cudaish)
                        resample.conv_bias(conv, x, w, conv.bias.detach().to(torch.bfloat16).as_subclass(_Cudaish))
        assert (bs.CONVB in taken) == bs.dispatch(site, size, True, name)[bs.CONVB], (site.name, taken)
