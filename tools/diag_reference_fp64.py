#!/usr/bin/env python
"""How well-conditioned is "per-pixel logits of iteration 1"?  Runs the UNMODIFIED reference model / loss / optimizer
(SOD_REFERENCE, CPU) twice on the same seeded inputs — once in float32 (what the golden vectors hold) and once in
float64 — and prints the distance between the two trajectories.  The float64 run is the exact-arithmetic proxy: whatever
separates it from the float32 run is rounding noise of the REFERENCE ITSELF, i.e. the floor below which no other
implementation can be compared with the float32 golden vectors.  (Build container only; output committed under
profiles/.)"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from make_golden import install_reference  # noqa: E402
from distributed_sod_project_b200.synthetic import synth_batch  # noqa: E402


def run(dtype, bs, size, iters):
    import network
    from loss.CEL import CEL
    from utils.misc import init_seed
    from utils.pipeline_ops import get_total_loss, make_optimizer
    init_seed(0)
    model = network.res50().to(dtype)
    opt = make_optimizer(model, "f3_trick", dict(lr=0.05, momentum=0.9, weight_decay=5e-4, nesterov=False))
    loss_funcs = [torch.nn.BCEWithLogitsLoss(reduction="mean"), CEL()]
    model.train()
    out = []
    for it in range(iters):
        x, m = synth_batch(1234 + 1000 * it, bs, size)
        preds = model(x.to(dtype))
        loss, _ = get_total_loss(preds, m.to(dtype), loss_funcs)
        opt.zero_grad(); loss.backward(); opt.step()
        out.append((float(loss), preds.detach().double().numpy()))
    return out


def main():
    install_reference()
    torch.set_num_threads(8)
    bs, size = (int(v) for v in (sys.argv[1:3] if len(sys.argv) > 2 else (4, 320)))
    a, b = run(torch.float32, bs, size, 3), run(torch.float64, bs, size, 3)
    for it, ((l32, p32), (l64, p64)) in enumerate(zip(a, b)):
        d = np.abs(p32 - p64)
        span = np.abs(p64).max()
        print(f"bs {bs} size {size} iter {it}: loss fp32 {l32:.7f} fp64 {l64:.7f} rel {abs(l32 - l64) / abs(l64):.2e} | "
              f"logits max|d|/max|ref| {d.max() / span:.2e}  rms {np.sqrt((d ** 2).mean()) / span:.2e}  "
              f"99.9th pct {np.quantile(d, 0.999) / span:.2e}", flush=True)


if __name__ == "__main__":
    main()
