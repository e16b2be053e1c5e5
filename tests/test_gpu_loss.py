"""Parity of the fused BCE+CEL kernel (through the C ABI) with the oracle and the reference's golden vectors."""
import numpy as np
import pytest
import torch

from oracle import loss as oloss

pytestmark = pytest.mark.gpu

CASES = ["n1", "n7", "n1000", "n4097", "img", "mask_zero", "mask_one", "binary", "extreme"]


def _run(x, t, **kw):
    from distributed_sod_project_b200.loss import bce_cel_fwd_bwd
    scalars, grad = bce_cel_fwd_bwd(x, t, **kw)
    torch.cuda.synchronize()
    return scalars.cpu().numpy().astype(np.float64), grad


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("red", ["mean", "sum"])
@pytest.mark.parametrize("mode", [0, 2])
def test_golden_fp32(golden, case, red, mode):
    g = golden("loss_kat.npz")
    x = torch.tensor(g[f"{case}/{red}/x"], dtype=torch.float32, device="cuda")
    t = torch.tensor(g[f"{case}/{red}/t"], dtype=torch.float32, device="cuda")
    ref = oloss.bce_cel_fwd_bwd(x.cpu().numpy(), t.cpu().numpy(), reduction=red)   # oracle on the fp32-rounded inputs
    s, grad = _run(x, t, reduction=red, mode=mode)
    assert s[0] == pytest.approx(ref["bce"], rel=2e-6, abs=1e-7)
    assert s[1] == pytest.approx(ref["cel"], rel=2e-6, abs=1e-7)
    assert s[2] == pytest.approx(ref["total"], rel=2e-6, abs=1e-7)
    # and against the reference's own numbers (fp64 inputs → allow the fp32 input rounding)
    assert s[0] == pytest.approx(float(g[f"{case}/{red}/bce"]), rel=1e-5, abs=1e-6)
    assert s[1] == pytest.approx(float(g[f"{case}/{red}/cel"]), rel=1e-5, abs=1e-6)
    gr = grad.cpu().numpy().astype(np.float64)
    scale = np.abs(ref["grad"]).max() + 1e-30
    assert np.abs(gr - ref["grad"]).max() / scale < 5e-6


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(16, 1, 320, 320), (3, 1, 37, 41), (16, 1, 256, 256), (16, 1, 384, 384)])
@pytest.mark.parametrize("mode", [0, 2])
def test_lowp_logits(dtype, shape, mode):
    gcpu = torch.Generator().manual_seed(5)
    x = (torch.randn(shape, generator=gcpu) * 2).to(dtype)
    t = (torch.rand(shape, generator=gcpu) * 255).round() / 255
    # fp16 gradients of a mean loss are subnormal without the amp loss scale (apex O1 uses 2^16): apply it
    gs = 65536.0 if dtype == torch.float16 else 1.0
    ref = oloss.bce_cel_fwd_bwd(x.float().numpy(), t.numpy(), grad_scale=gs)
    s, grad = _run(x.cuda(), t.cuda(), mode=mode, grad_scale=gs)
    assert s[0] == pytest.approx(ref["bce"], rel=1e-5)
    assert s[1] == pytest.approx(ref["cel"], rel=1e-5)
    assert grad.dtype == dtype
    gr = grad.float().cpu().numpy().astype(np.float64)
    scale = np.abs(ref["grad"]).max()
    ulp = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    assert np.abs(gr - ref["grad"]).max() / scale < 1.5 * ulp      # one output rounding
    assert int(s[7]) == x.numel()


def test_spill_path_large_tensor():
    """more elements than the shared-memory window: the overflow streams from global memory"""
    n = 9_000_017
    gcpu = torch.Generator().manual_seed(9)
    x = torch.randn(n, generator=gcpu)
    t = (torch.rand(n, generator=gcpu) > 0.7).float()
    ref = oloss.bce_cel_fwd_bwd(x.numpy(), t.numpy())
    s, grad = _run(x.cuda(), t.cuda())
    assert s[0] == pytest.approx(ref["bce"], rel=1e-5)
    assert s[1] == pytest.approx(ref["cel"], rel=1e-5)
    gr = grad.cpu().numpy().astype(np.float64)
    assert np.abs(gr - ref["grad"]).max() / np.abs(ref["grad"]).max() < 1e-5


def test_mode1_refuses_when_not_resident():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.loss import bce_cel_fwd_bwd
    x = torch.zeros(9_000_000, device="cuda"); t = torch.zeros_like(x)
    with pytest.raises(_lib.SodError):
        bce_cel_fwd_bwd(x, t, mode=1)


def test_linearity_and_decomposition():
    """size-independent properties at the BASELINE shape: grad(w_bce,w_cel) is linear in the weights and
    in grad_scale."""
    gcpu = torch.Generator().manual_seed(3)
    x = torch.randn(16, 1, 320, 320, generator=gcpu).cuda()
    t = (torch.rand(16, 1, 320, 320, generator=gcpu) > 0.8).float().cuda()
    _, g_all = _run(x, t)
    _, g_b = _run(x, t, w_cel=0.0)
    _, g_c = _run(x, t, w_bce=0.0)
    _, g_2 = _run(x, t, grad_scale=2.0)
    assert torch.allclose(g_all, g_b + g_c, rtol=1e-5, atol=1e-9)
    assert torch.allclose(g_2, 2 * g_all, rtol=1e-6, atol=0)
    assert abs(float(g_b.sum())) < 1.0    # Σ(p-t)/N is O(1)


def test_autograd_module_and_get_total_loss(golden):
    from distributed_sod_project_b200.loss import BCEWithLogitsLoss, CEL, FusedBCECEL, get_total_loss
    g = golden("loss_kat.npz")
    x = torch.tensor(g["img/mean/x"], dtype=torch.float32, device="cuda").requires_grad_(True)
    t = torch.tensor(g["img/mean/t"], dtype=torch.float32, device="cuda")
    total, strs = get_total_loss(x, t, [BCEWithLogitsLoss(reduction="mean"), CEL()])
    assert strs == list(g["total_loss/strings"])
    assert float(total) == pytest.approx(float(g["total_loss/value"]), rel=1e-6)
    (total * 3.0).backward()                     # non-unit upstream → the scale kernel runs
    ref = torch.tensor(g["img/mean/grad"], device="cuda") * 3.0
    assert torch.allclose(x.grad.double(), ref, rtol=1e-5, atol=1e-9)
    # torch's own BCEWithLogitsLoss object in the list is recognised too
    x2 = x.detach().clone().requires_grad_(True)
    total2, strs2 = get_total_loss(x2, t, [torch.nn.BCEWithLogitsLoss(), CEL()], unit_upstream=True)
    total2.backward()
    assert strs2 == strs and torch.allclose(x2.grad.double(), ref / 3.0, rtol=1e-5, atol=1e-9)
    # single-loss objects
    x3 = x.detach().clone().requires_grad_(True)
    (BCEWithLogitsLoss()(x3, t) + CEL()(x3, t)).backward()
    assert torch.allclose(x3.grad.double(), ref / 3.0, rtol=1e-5, atol=1e-9)
    assert str(CEL()) == "You are using `CEL`!"
    assert FusedBCECEL()(x.detach(), t).shape == ()


def test_rejects_cpu_and_misuse():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.loss import bce_cel_fwd_bwd
    with pytest.raises(_lib.SodError):
        bce_cel_fwd_bwd(torch.zeros(4), torch.zeros(4))
    with pytest.raises(ValueError):
        bce_cel_fwd_bwd(torch.zeros(4, device="cuda"), torch.zeros(5, device="cuda"))


def _sm_count() -> int:
    import ctypes
    from distributed_sod_project_b200 import _lib
    sms = ctypes.c_int(0)
    _lib.check(_lib.lib().sod_device_info(ctypes.byref(sms), None, None), "sod_device_info")
    return sms.value


def _check_ring_streamed(n, dtype):
    from distributed_sod_project_b200.loss import bce_cel_fwd_bwd
    gcpu = torch.Generator().manual_seed(n % 1000)
    x = (torch.randn(n, generator=gcpu) * 3).to(dtype)
    t = (torch.rand(n, generator=gcpu) > 0.6).float()
    ref = oloss.bce_cel_fwd_bwd(x.float().numpy(), t.numpy())
    scalars, grad = bce_cel_fwd_bwd(x.cuda(), t.cuda(), mode=2)
    s = scalars.cpu().numpy()
    assert s[0] == pytest.approx(ref["bce"], rel=2e-5) and s[1] == pytest.approx(ref["cel"], rel=2e-5)
    gr = grad.float().cpu().numpy().astype(np.float64)
    scale = np.abs(ref["grad"]).max()
    tol = 1e-5 if dtype == torch.float32 else 1.5 * 2.0 ** -8
    assert np.abs(gr - ref["grad"]).max() / scale < tol
    resident, _ = bce_cel_fwd_bwd(x.cuda(), t.cuda(), mode=0)
    assert resident.cpu().numpy()[2] == pytest.approx(s[2], rel=1e-6)


@pytest.mark.parametrize("n", [4096 * 3 + 5, 148 * 4096 * 9, 148 * 4096 * 10 + 777, 148 * 4096 * 23 + 8, 33_000_001])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ring_streamed_kernel_matches_oracle(n, dtype):
    """mode 2 forces the ring-streamed kernel (producer warp + shared-memory ring, re-stream newest first) at fixed sizes,
    including a ragged scalar tail"""
    _check_ring_streamed(n, dtype)


# n = chunks_per_sm * #SMs * 4096 + extra: one CTA per SM, 4096-element chunks, so the chunk count per CTA does not depend
# on how many SMs the device has
@pytest.mark.parametrize("chunks_per_sm, extra", [(9, 0), (10, 777), (23, 8)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ring_streamed_kernel_chunks_per_cta(chunks_per_sm, extra, dtype):
    """the ring-streamed kernel with the same number of chunks per CTA on any device: fewer chunks than stages (nothing
    re-streamed), exactly as many, one more, many more"""
    _check_ring_streamed(chunks_per_sm * _sm_count() * 4096 + extra, dtype)
