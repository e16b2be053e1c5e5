#!/usr/bin/env python
"""GPU-box diagnostic: per-parameter gradient error of iteration 0 (fp32) of the engine vs the CPU oracle
trainer, with this repo's SyncBN kernels and, for attribution, with stock torch BatchNorm on the GPU."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from oracle.step import OracleCEL, total_loss
from distributed_sod_project_b200 import network
from distributed_sod_project_b200.utils import init_seed
from distributed_sod_project_b200.synthetic import synth_batch
from distributed_sod_project_b200.syncbn import convert_syncbn_model

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
bs, size = int(os.environ.get("BS", 2)), int(os.environ.get("SIZE", 64))
x, m = synth_batch(1234, bs, size)
loss_funcs = [torch.nn.BCEWithLogitsLoss(), OracleCEL()]


def grads(model, x, m):
    model.train()
    out = model(x)
    loss, _ = total_loss(out, m, loss_funcs)
    loss.backward()
    return float(loss), out.detach().float().cpu(), {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}


init_seed(0); cpu_model = network.res50()
t0 = time.time(); l_cpu, o_cpu, g_cpu = grads(cpu_model, x, m); print(f"cpu  loss {l_cpu:.6f}  ({time.time()-t0:.1f}s, {os.cpu_count()} cores)")
init_seed(0); gm = network.res50().cuda().to(memory_format=torch.channels_last)
l_t, o_t, g_t = grads(gm, x.cuda().contiguous(memory_format=torch.channels_last), m.cuda())
init_seed(0); sm = convert_syncbn_model(network.res50().cuda().to(memory_format=torch.channels_last))
l_s, o_s, g_s = grads(sm, x.cuda().contiguous(memory_format=torch.channels_last), m.cuda())
print(f"gpu torch-BN loss {l_t:.6f} logits relerr {((o_t-o_cpu).abs().max()/o_cpu.abs().max()):.2e}")
print(f"gpu sod-BN   loss {l_s:.6f} logits relerr {((o_s-o_cpu).abs().max()/o_cpu.abs().max()):.2e}")
rows = []
for n in g_cpu:
    sc = g_cpu[n].abs().max().item() + 1e-30
    rows.append((n, (g_t[n] - g_cpu[n]).abs().max().item() / sc, (g_s[n] - g_cpu[n]).abs().max().item() / sc, sc))
rows.sort(key=lambda r: -r[2])
print("worst 12 params by sod-BN grad relerr:   name  torchBN_err  sodBN_err  |g|max")
for r in rows[:12]:
    print(f"  {r[0]:40s} {r[1]:.2e} {r[2]:.2e} {r[3]:.3e}")
print("median relerr  torchBN %.2e   sodBN %.2e" % (np.median([r[1] for r in rows]), np.median([r[2] for r in rows])))
