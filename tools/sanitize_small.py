#!/usr/bin/env python
"""GPU-box tool for compute-sanitizer: one small launch of every hand-written kernel family (world 1, or world N under
torchrun: then the SyncBN packet exchange and the fused all-reduce+SGD run across ranks).
    compute-sanitizer --tool racecheck|synccheck|memcheck [--target-processes all] python tools/sanitize_small.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

world = int(os.environ.get("WORLD_SIZE", "1"))
local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
from distributed_sod_project_b200 import _lib, comm  # noqa: E402
from distributed_sod_project_b200.loss import bce_cel_fwd_bwd  # noqa: E402
from distributed_sod_project_b200.metrics import SaliencyMetrics  # noqa: E402
from distributed_sod_project_b200.pipeline import Ragged, preprocess_batch  # noqa: E402
from distributed_sod_project_b200.syncbn import SyncBatchNorm  # noqa: E402

cl = lambda t: t.cuda().contiguous(memory_format=torch.channels_last)  # noqa: E731
for shape, dt in (((4, 64, 12, 12), torch.bfloat16), ((2, 256, 6, 6), torch.float32), ((4, 32, 20, 20), torch.bfloat16), ((2, 2048, 2, 2), torch.bfloat16)):
    for variant in ("plain", "relu", "pre_relu", "res_relu", "bias"):
        c = shape[1]
        bn = SyncBatchNorm(c).cuda()
        x = cl(torch.randn(shape).to(dt)).requires_grad_(True)
        pre = cl(torch.randn(shape).to(dt)).requires_grad_(True) if variant == "pre_relu" else None
        res = cl(torch.randn(shape).to(dt)).requires_grad_(True) if variant == "res_relu" else None
        cb = torch.randn(c, device="cuda").requires_grad_(True) if variant == "bias" else None
        y = bn.fused_forward(x, pre_add=pre, residual=res, relu=variant != "plain", conv_bias=(cb, None))
        y.backward(cl(torch.randn(shape).to(dt)))
torch.cuda.synchronize()
bce_cel_fwd_bwd(torch.randn(2, 1, 64, 64, device="cuda").bfloat16(), (torch.rand(2, 1, 64, 64, device="cuda") > 0.5).float())
n = 8192
p, v, g = (torch.randn(n, device="cuda") for _ in range(3))
segs = (_lib.sod_sgd_segment * 1)(_lib.sod_sgd_segment(0, n, 0.1, 5e-4, 0.9, 0))
assert _lib.lib().sod_sgd_momentum(p.data_ptr(), v.data_ptr(), g.data_ptr(), None, None, n, segs, 1, None, 1.0, None, 1, _lib.stream_ptr()) == 0
srcs = [torch.randn(s, device="cuda").bfloat16() for s in (7, 64, 9000)]
flat = torch.zeros(16384, dtype=torch.bfloat16, device="cuda")
items = (_lib.sod_gather_item * 3)(*[_lib.sod_gather_item(t.data_ptr(), off, t.numel()) for t, off in zip(srcs, (0, 64, 128))])
assert _lib.lib().sod_grad_gather16(items, 3, flat.data_ptr(), flat.numel(), _lib.stream_ptr()) == 0
img = torch.randint(0, 256, (2, 20, 24, 3), dtype=torch.uint8, device="cuda")
msk = torch.randint(0, 256, (2, 20, 24), dtype=torch.uint8, device="cuda")
preprocess_batch(img, msk, size=16)
cal = SaliencyMetrics(wfm="gpu")
cal.update_batch(torch.randint(0, 256, (2, 20, 24), dtype=torch.uint8, device="cuda"), (torch.rand(2, 20, 24, device="cuda") > 0.6).to(torch.uint8) * 255)
pr = Ragged(torch.randint(0, 256, (20 * 24 + 7 * 40 + 1,), dtype=torch.uint8, device="cuda"),
            torch.tensor([[20, 24], [7, 40], [1, 1]], dtype=torch.int32), 1)
gr = Ragged((torch.rand(pr.data.numel(), device="cuda") > 0.7).to(torch.uint8) * 255, pr.hw, 1)
cal.update_ragged(pr, gr)
if world > 1:
    arena = comm.Arena(payload_bytes=2 * 4 * n + 4096)
    p_off, g_off = arena.alloc(4 * n), arena.alloc(4 * n)
    arena.view(p_off, n, torch.float32).copy_(p); arena.view(g_off, n, torch.float32).copy_(g)
    torch.cuda.synchronize(); dist.barrier()
    for flags in (1, 1 | _lib.SOD_ALGO_NO_MULTIMEM):
        assert _lib.lib().sod_allreduce_sgd(arena.ref, g_off, 0, p_off, v.data_ptr(), None, n, segs, 1, None, 1.0, None, flags, _lib.stream_ptr()) == 0
    arena.allreduce_(g_off, n, algo=1); arena.allreduce_(g_off, n, algo=2)
    torch.cuda.synchronize(); dist.barrier()
    arena.check_error(); comm.small_arena().check_error()
res = cal.show()
torch.cuda.synchronize()
print("sanitize ok", {k: round(v, 4) for k, v in res.items() if v is not None}, flush=True)
if world > 1:
    dist.barrier(); dist.destroy_process_group()
