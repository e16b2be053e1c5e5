"""The block-site table of oracle/block_sites.py against the model it cuts up (CPU only).

* every parameter and buffer of `res50` belongs to exactly one site;
* the sites, run one after the other, are the model's forward bit for bit (fp32, stock modules) and leave the same BN
  buffers behind;
* `dispatch` — which of the engine's resampling / max-pool / column-sum kernels each site reaches — agrees with the
  predicates of `resample.py` and `network/blocks.py` at 256², 288², 320², 352² and 384².  The forward runs on CPU
  tensors that report `is_cuda`, with the kernels' autograd Functions replaced by recorders that hand back the torch
  result, so the predicates are evaluated exactly as the engine evaluates them.
"""
import contextlib
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import block_sites as bs


def _model():
    from distributed_sod_project_b200 import network
    from distributed_sod_project_b200.utils import init_seed
    init_seed(0)
    return network.res50()


def test_every_parameter_and_buffer_belongs_to_exactly_one_site():
    model = _model()
    names = [n for n, _ in model.named_parameters()] + [n for n, _ in model.named_buffers()]
    assert len(names) > 500
    for n in names:
        assert len(bs.owner(n)) == 1, (n, bs.owner(n))
    table = bs.sites()
    assert len({s.name for s in table}) == len(table)
    # every site's paths exist, and the representative ones are those the GPU grid runs
    for s in table:
        bs.modules(model, s)
    rep = [s.name for s in table if s.representative]
    assert rep[:9] == ["stem", "pool+div_4.1.0", "div_4.1.1", "div_8.0", "div_8.1", "div_16.0", "div_16.1", "div_32.0",
                       "div_32.1"]
    assert len(rep) == 9 + 5 + 5 + 5 + 4 + 1


def test_sites_compose_to_the_model_forward_bit_for_bit():
    model = _model().train()
    twin = copy.deepcopy(model)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        want = model(x)
        got = bs.compose(twin, x)
    assert want.shape == (2, 1, 64, 64)
    assert torch.equal(got, want)
    for (n, a), (_, b) in zip(model.named_buffers(), twin.named_buffers()):
        assert torch.equal(a, b), n


def test_site_shapes_are_what_the_model_feeds_them():
    model = _model().eval()
    seen = {}
    table = bs.by_name()

    def hook(name):
        def fn(mod, args):
            seen.setdefault(name, tuple(args[0].shape))
        return fn

    for s in bs.sites():
        if s.paths and s.kind not in ("head",):
            model.get_submodule(s.paths[0]).register_forward_pre_hook(hook(s.name))
    model.get_submodule("upconv1").register_forward_pre_hook(hook("upconv1"))
    with torch.no_grad():
        model(torch.zeros(1, 3, 128, 128))
    for name, shape in seen.items():
        if name == "upconv1":
            assert shape == tuple(table["head"].shapes(128, 1)[0][:2]) + (128, 128)
        else:
            assert shape == tuple(table[name].shapes(128, 1)[0]), name


class _Cudaish(torch.Tensor):
    """a CPU tensor that says it is on CUDA, so that the engine's dispatch predicates run as they do on the GPU"""

    @property
    def is_cuda(self):
        return True


@contextlib.contextmanager
def _recording():
    """resample.ENABLED on; every kernel autograd Function replaced by a recorder returning the torch result"""
    from distributed_sod_project_b200 import resample
    from distributed_sod_project_b200.network import blocks
    taken = []
    torch_op = {
        "_Up2x": lambda x, add: F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=False) + (0 if add is None else add),
        "_AvgPool2x2": lambda x: F.avg_pool2d(x, 2, 2),
        "_MaxPool3x3s2": lambda x: F.max_pool2d(x, 3, 2, 1),
        "_ConvBias": lambda x, w, b, *conf: F.conv2d(x, w, b, *conf),
    }
    saved = {n: getattr(resample, n).apply for n in torch_op}
    old = resample.ENABLED, resample.MAXPOOL_ENABLED, resample.COLSUM_ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE
    try:
        for n, op in torch_op.items():
            def rec(*a, n=n, op=op):
                taken.append(n + "Backward")
                return op(*a)
            setattr(getattr(resample, n), "apply", rec)
        resample.ENABLED = resample.MAXPOOL_ENABLED = resample.COLSUM_ENABLED = True
        yield taken
    finally:
        for n, fn in saved.items():
            setattr(getattr(resample, n), "apply", fn)
        resample.ENABLED, resample.MAXPOOL_ENABLED, resample.COLSUM_ENABLED, blocks.INTERPOLATE_IN_ACTIVATION_DTYPE = old


@pytest.mark.parametrize("size", bs.SIZES)
def test_dispatch_matches_the_engine_predicates(size):
    from distributed_sod_project_b200 import resample
    model = _model().eval()
    odd = size in (288, 352)
    assert odd == bool((size // 32) % 2)
    for site in bs.sites():
        if not site.representative:
            continue
        mods = bs.modules(model, site)
        xs = [torch.zeros(sh).as_subclass(_Cudaish) for sh in site.shapes(size, 1)]
        with _recording() as taken, torch.no_grad():
            site.run(mods, *xs)
        want = bs.dispatch(site, size, amp=False)
        got = set(taken)
        for node in (bs.UP, bs.AVG, bs.MAX):
            assert (node in got) == want[node], (site.name, size, node, taken)
        assert bs.CONVB not in got                       # plain convolutions never take conv_bias
        if site.kind == "sim":
            assert want[bs.UP] == want[bs.AVG] == (not odd or site.stride != 32)
        # under amp the shadow-weight forward offers every biased convolution called as a module to `conv_bias`
        with _recording() as taken, torch.no_grad(), torch.enable_grad():
            for p, m in mods.items():
                for name, conv in m.named_modules():
                    if isinstance(conv, torch.nn.Conv2d) and conv.bias is not None and site.kind in ("trans", "head"):
                        w = conv.weight.detach().to(torch.bfloat16).as_subclass(_Cudaish)
                        x = torch.zeros(1, conv.in_channels, 4, 4, dtype=torch.bfloat16).as_subclass(_Cudaish)
                        resample.conv_bias(conv, x, w, conv.bias.detach().to(torch.bfloat16).as_subclass(_Cudaish))
        assert (bs.CONVB in taken) == bs.dispatch(site, size, amp=True)[bs.CONVB], (site.name, taken)
