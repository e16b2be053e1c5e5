"""fp16 amp at world > 1 on one GPU: W = 2, 3, 4, 8 virtual ranks (the harness of test_gpu_virtual_world.py) run
`sod_allreduce_sgd_scaler` / `sod_allreduce_adam_scaler` with fp16 gradients on the wire and a loss scaler in every
rank's arena.

* The fp16 wire sum equals the world-1 kernel on the rank-order fp32 sum bit for bit (fp16 values summed in fp32 from 0,
  inv_scale = fp32(1/scale)/fp32(W), which is what the kernel forms from the scaler).
* An inf planted in one rank's flag only (the last rank's, or the first's) makes every rank skip; the scalers stay
  bit-identical on all ranks and follow the host model of the rules; clean steps grow every rank's scale identically.
"""
import numpy as np
import pytest
import torch

import test_gpu_virtual_world as vwh
from oracle import comm_geometry as cgeo

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(vwh._SERIAL, reason="serialised kernel launches cannot run virtual ranks side by side")]

L, lib, sm_count, stream_ptr = vwh.L, vwh._lib, vwh.sm_count, vwh.stream_ptr


def model_step(scale, unskipped, gi, overflow):
    if overflow:
        return max(scale / 2.0, 1.0), 0
    unskipped += 1
    return (min(scale * 2.0, 2.0 ** 24) if unskipped % gi == 0 else scale), unskipped


CASES = [(w, rule, bad) for w in vwh.WORLDS for rule in ("sgd", "adam") for bad in ("last", "first")]


@pytest.mark.parametrize("world,rule,bad", CASES, ids=[f"W{w}-{r}-inf-on-{b}" for w, r, b in CASES])
def test_fp16_wire_and_shared_verdict_at_world_w(world, rule, bad):
    l = lib()
    W = world
    nvec = W * 2 * cgeo.VEC_PER_CTA + 3 * W + 1
    n = 4 * nvec
    half = (nvec // 2) * 4
    table = [(0, half, l.SOD_SEG_GRAD16), (half, n, 0)]
    if rule == "adam":
        segs = (l.sod_adam_segment * 2)(*[l.sod_adam_segment(b, e, 1e-3, 5e-4, 0.9, 0.999, 1e-8, f) for b, e, f in table])
    else:
        segs = (l.sod_sgd_segment * 2)(*[l.sod_sgd_segment(b, e, 0.05, 5e-4, 0.9, f) for b, e, f in table])
    rng = vwh.rng_for("amp16", W, rule, bad)
    # steps: clean, overflow on one rank, clean ×3 (growth at interval 2), overflow on one rank, clean
    planted = [None, bad, None, None, None, bad, None]
    K, gi, scale0 = len(planted), 2, 1024.0
    bad_rank = W - 1 if bad == "last" else 0
    p0 = vwh.spread(rng, n, -3, 3)
    st0 = [vwh.spread(rng, n, -4, 0)] + ([np.abs(vwh.spread(rng, n, -12, -4))] if rule == "adam" else [])
    g32 = [[vwh.spread(rng, n, -6, 2) for _ in range(W)] for _ in range(K)]
    g16 = [[torch.from_numpy(vwh.spread(rng, n, -6, 2)).half() for _ in range(W)] for _ in range(K)]
    g32_dev = [[torch.from_numpy(g).cuda() for g in gk] for gk in g32]
    g16_dev = [[g.cuda() for g in gk] for gk in g16]
    flags = l.SOD_SGD_ZERO_GRAD | l.SOD_ALGO_NO_MULTIMEM | l.SOD_GRAD16_F16

    vw = vwh.VirtualWorld(W, 4 * n * 2 + 2 * n + 2048)
    p_off, g_off, h_off, s_off = vw.alloc(4 * n), vw.alloc(4 * n), vw.alloc(2 * n), vw.alloc(32)
    grid = cgeo.step_grid(n, W, sm_count())
    state = {}

    def make():
        st = [[torch.from_numpy(s).cuda() for s in st0] for _ in range(W)]
        steps = [torch.zeros(l.SOD_ADAM_STEP_WORDS, dtype=torch.int32, device="cuda") for _ in range(W)]
        shadows = [torch.zeros(n, dtype=torch.float16, device="cuda") for _ in range(W)]
        hist = [torch.zeros(K, l.SOD_LOSS_SCALER_WORDS, dtype=torch.int32, device="cuda") for _ in range(W)]
        state.update(st=st, steps=steps, shadows=shadows, hist=hist)
        calls = []
        for r in range(W):
            vw.view(r, p_off, n, torch.float32).copy_(torch.from_numpy(p0))
            sc = vw.view(r, s_off, l.SOD_LOSS_SCALER_WORDS, torch.int32)
            sc.zero_()
            sc.view(torch.float32)[1].fill_(scale0)
            sc[3].fill_(gi)
            seq = []
            for k in range(K):
                def fill(r=r, k=k, sc=sc):
                    vw.view(r, g_off, n, torch.float32).copy_(g32_dev[k][r])
                    vw.view(r, h_off, n, torch.float16).copy_(g16_dev[k][r])
                    sc[0].fill_(1 if (planted[k] is not None and r == bad_rank) else 0)   # this rank's own check
                seq.append(vwh.Launch(fill))
                if rule == "adam":
                    fn = (lambda r=r, sc=sc: L().sod_allreduce_adam_scaler(
                        vw.ref(r), g_off, h_off, p_off, st[r][0].data_ptr(), st[r][1].data_ptr(), shadows[r].data_ptr(), n,
                        segs, 2, None, steps[r].data_ptr(), sc.data_ptr(), flags, stream_ptr()))
                else:
                    fn = (lambda r=r, sc=sc: L().sod_allreduce_sgd_scaler(
                        vw.ref(r), g_off, h_off, p_off, st[r][0].data_ptr(), shadows[r].data_ptr(), n, segs, 2, None,
                        sc.data_ptr(), flags, stream_ptr()))
                seq.append(vwh.Launch(fn, grid=grid, channel=cgeo.CH_STEP))
                seq.append(vwh.Launch(lambda r=r, k=k, sc=sc: hist[r][k].copy_(sc)))
            calls.append(seq)
        return calls
    vw.run(make, "interleaved" if W % 2 == 0 else "reversed")

    # world-1 reference on the rank-order sums with the host model's scale
    p1 = torch.from_numpy(p0).cuda()
    st1 = [torch.from_numpy(s).cuda() for s in st0]
    steps1 = torch.zeros(l.SOD_ADAM_STEP_WORDS, dtype=torch.int32, device="cuda")
    sh1 = torch.zeros(n, dtype=torch.float16, device="cuda")
    scale, unsk = scale0, 0
    want_hist = []
    for k in range(K):
        gsum = vwh.rank_order_sum(g32[k])
        h = np.zeros(n, np.float32)
        for r in range(W):
            h += g16[k][r].float().numpy()
        gsum[:half] = h[:half]
        g1 = torch.from_numpy(gsum).cuda()
        ov = planted[k] is not None
        finf = torch.tensor([1 if ov else 0], dtype=torch.int32, device="cuda")
        inv = float(np.float32(np.float32(1.0) / np.float32(scale)) / np.float32(W))
        if rule == "adam":
            rc = L().sod_adam(p1.data_ptr(), st1[0].data_ptr(), st1[1].data_ptr(), g1.data_ptr(), None, sh1.data_ptr(), n,
                              segs, 2, None, steps1.data_ptr(), inv, finf.data_ptr(), l.SOD_GRAD16_F16, stream_ptr())
        else:
            rc = L().sod_sgd_momentum(p1.data_ptr(), st1[0].data_ptr(), g1.data_ptr(), None, sh1.data_ptr(), n, segs, 2,
                                      None, inv, finf.data_ptr(), l.SOD_GRAD16_F16, stream_ptr())
        assert rc == 0
        scale, unsk = model_step(scale, unsk, gi, ov)
        want_hist.append((scale, unsk, int(ov)))
    torch.cuda.synchronize()
    seq = [scale0] + [s for s, _, _ in want_hist]
    assert any(b == a / 2 for a, b in zip(seq, seq[1:])) and any(b == 2 * a for a, b in zip(seq, seq[1:]))

    for r in range(W):
        p = vw.view(r, p_off, n, torch.float32)
        assert np.array_equal(vwh.bits(p), vwh.bits(p1)), f"rank {r}: parameters differ from the world-1 step"
        lo, hi = (4 * x for x in cgeo.shard_bounds(r, nvec, W))
        for i, (got, want) in enumerate(zip(state["st"][r], st1)):
            assert np.array_equal(vwh.bits(got)[lo:hi], vwh.bits(want)[lo:hi]), f"rank {r}: state {i} of the shard"
        if rule == "adam":
            assert state["steps"][r].tolist() == steps1.tolist()
        assert torch.equal(state["shadows"][r].view(torch.int16), p.half().view(torch.int16)), f"rank {r}: fp16 shadow"
        hist = state["hist"][r].cpu()
        got = [(float(hist[k].view(torch.float32)[1]), int(hist[k][2]), int(hist[k][0])) for k in range(K)]
        assert got == want_hist, f"rank {r}: scaler history {got} != {want_hist}"
        assert not hist[:, 4].any(), f"rank {r}: ticket not re-armed"
        assert torch.equal(hist, state["hist"][0].cpu()), f"rank {r}: scaler differs from rank 0's"
        assert not vw.view(r, h_off, n, torch.float16).float().any()
