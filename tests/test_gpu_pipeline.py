"""Data-side kernels of csrc/pipeline.cu against their oracles: batch pre-processing (oracle/pipeline.py = the reference's
ToTensor / Normalize / flip / multi-scale collate in torch CPU ops) and the saliency-metric statistics (golden vectors from
the UNMODIFIED reference classes, tests/golden/metrics_kat.npz)."""
import numpy as np
import pytest
import torch

from oracle import pipeline as opipe

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("hs,ws,size", [(320, 320, None), (320, 320, 384), (320, 320, 256), (37, 53, 64), (64, 64, (48, 80)), (5, 7, 3)])
@pytest.mark.parametrize("with_mask,with_flip", [(True, False), (True, True), (False, False)])
def test_preprocess_batch_matches_the_reference_transforms(hs, ws, size, with_mask, with_flip):
    from distributed_sod_project_b200.pipeline import preprocess_batch
    g = torch.Generator().manual_seed(hs * 1000 + ws)
    n = 5
    img = torch.randint(0, 256, (n, hs, ws, 3), generator=g, dtype=torch.uint8)
    mask = torch.randint(0, 256, (n, hs, ws), generator=g, dtype=torch.uint8) if with_mask else None
    flip = torch.tensor([1, 0, 1, 1, 0], dtype=torch.uint8) if with_flip else None
    want_x, want_m = opipe.preprocess(img, mask, size=size, flip=flip)
    x, m = preprocess_batch(img.cuda(), mask.cuda() if with_mask else None, size=size, flip=flip.cuda() if with_flip else None)
    assert x.shape == want_x.shape and x.is_contiguous(memory_format=torch.channels_last)
    if size is None or (hs, ws) == ((size, size) if isinstance(size, int) else tuple(size)):
        assert torch.equal(x.cpu(), want_x)                      # no resize: torch's fp32 operations exactly
    else:
        # the taps and λ are torch's; the 4-term blend may round differently (tests/test_gpu_data_regimes.py bounds
        # the kernel against float64 at 1.2e-6, torch's own fp32 blend adds as much again)
        assert float((x.cpu() - want_x).abs().max()) <= 4e-6
    if with_mask:
        assert torch.equal(m.cpu(), want_m)                      # nearest neighbour of k/255: exact
    else:
        assert m is None
    # bf16 and fp16 (the apex O1 input dtype): the fp32 output rounded once
    for dt in (torch.bfloat16, torch.float16):
        x16, _ = preprocess_batch(img.cuda(), mask.cuda() if with_mask else None, size=size,
                                  flip=flip.cuda() if with_flip else None, dtype=dt)
        assert x16.dtype == dt and torch.equal(x16, x.to(dt))


def test_device_prefetcher_yields_every_batch_in_order():
    from distributed_sod_project_b200.pipeline import DevicePrefetcher
    g = torch.Generator().manual_seed(0)
    host = [(torch.randint(0, 256, (3, 40, 40, 3), generator=g, dtype=torch.uint8).pin_memory(),
             torch.randint(0, 256, (3, 40, 40), generator=g, dtype=torch.uint8).pin_memory(), [f"b{i}_{k}" for k in range(3)]) for i in range(6)]
    pre = DevicePrefetcher(host, size_list=[32, 40, 48], seed=5)
    import random
    rng = random.Random(5)
    seen = 0
    for (x, m, names), (img, mask, want_names) in zip(pre, host):
        size = rng.choice([32, 40, 48])
        wx, wm = opipe.preprocess(img, mask, size=size)
        assert names == want_names and tuple(x.shape) == (3, 3, size, size)
        assert float((x.cpu() - wx).abs().max()) <= 4e-6 and torch.equal(m.cpu(), wm)
        seen += 1
    assert seen == 6


def _cases(golden):
    g = golden("metrics_kat.npz")
    return g, [(g[f"pred{i}"], g[f"gt{i}"]) for i in range(int(g["n"]))]


def test_metric_kernels_count_exactly(golden):
    """head / hist kernels against a numpy count of the same definition (oracle/metrics.py::emulate_kernels)"""
    from distributed_sod_project_b200 import _lib
    from oracle.metrics import emulate_kernels
    _, cases = _cases(golden)
    rng = np.random.default_rng(1)
    cases = cases + [(rng.integers(0, 256, (320, 320)).astype(np.uint8), (rng.random((320, 320)) < 0.3).astype(np.uint8) * 255)]
    for p8, g8 in cases:
        h, w = p8.shape
        p, g = torch.tensor(p8).cuda()[None], torch.tensor(g8).cuda()[None]
        head = torch.zeros((1, 8), dtype=torch.int64, device="cuda")
        hist = torch.zeros((1, 4, 2, 256), dtype=torch.int32, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        assert _lib.lib().sod_saliency_head(p.data_ptr(), g.data_ptr(), 1, h, w, head.data_ptr(), s) == 0
        want_head, want_hist = emulate_kernels(p8, g8)
        assert np.array_equal(head.cpu().numpy()[0], want_head)
        n_fg = max(int(want_head[4]), 1)
        split = torch.tensor([[int(round(int(want_head[5]) / n_fg)) + 1, int(round(int(want_head[6]) / n_fg)) + 1]], dtype=torch.int32, device="cuda")
        assert _lib.lib().sod_saliency_hist(p.data_ptr(), g.data_ptr(), 1, h, w, head.data_ptr(), split.data_ptr(), hist.data_ptr(), s) == 0
        assert np.array_equal(hist.cpu().numpy()[0].astype(np.int64), want_hist)
        assert int(hist.sum()) == h * w


def test_saliency_metrics_match_the_reference_dataset_numbers(golden):
    from distributed_sod_project_b200.metrics import SaliencyMetrics
    g, cases = _cases(golden)
    cal = SaliencyMetrics(num=len(cases), wfm="host")
    for p8, g8 in cases:
        cal.update(torch.tensor(p8).cuda(), torch.tensor(g8).cuda())
    res = cal.show()
    want = dict(zip((str(k) for k in g["show_keys"]), (float(v) for v in g["show_vals"])))
    for k in ("MaxF", "MeanF", "MAE", "EM", "WFM"):
        assert res[k] == pytest.approx(want[k], rel=1e-10), k
    assert res["SM"] == pytest.approx(want["SM"], rel=2e-7)       # float32 ground-truth statistics in the reference (test_metrics_cpu.py)
    # batched entry: same-size images in one call give the same numbers as one call per image
    same = [c for c in cases if c[0].shape == (32, 32)]
    a, b = SaliencyMetrics(), SaliencyMetrics()
    a.update_batch(torch.tensor(np.stack([c[0] for c in same])).cuda(), torch.tensor(np.stack([c[1] for c in same])).cuda())
    for p8, g8 in same:
        b.update(torch.tensor(p8).cuda(), torch.tensor(g8).cuda())
    ra, rb = a.show(), b.show()
    assert all(ra[k] == rb[k] for k in ("MaxF", "MeanF", "MAE", "SM", "EM")) and ra["WFM"] is None


def test_quantize_is_topilimage():
    from distributed_sod_project_b200.metrics import SaliencyMetrics
    g = torch.Generator().manual_seed(2)
    p = torch.rand(3, 1, 50, 70, generator=g).cuda()
    assert torch.equal(SaliencyMetrics.quantize(p), p.mul(255).byte())         # torchvision ToPILImage: mul(255).byte()
    logits = (torch.randn(3, 1, 50, 70, generator=g) * 4).cuda()
    got, want = SaliencyMetrics.quantize(logits, apply_sigmoid=True), logits.sigmoid().mul(255).byte()
    assert torch.equal(got, want)                          # torch's CUDA sigmoid is the same 1 / (1 + expf(−x))
    lb = logits.to(torch.bfloat16)
    assert torch.equal(SaliencyMetrics.quantize(lb, apply_sigmoid=True), lb.float().sigmoid().mul(255).byte())


def test_distributed_style_evaluation_single_rank():
    """evaluate.test_process over a sharded synthetic set == feeding the same images to the oracle on the CPU"""
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.evaluate import shard, test_process
    from distributed_sod_project_b200.synthetic import synth_eval_set
    from oracle import metrics as om
    tr = Trainer(model_name="res50", dtype=torch.bfloat16, channels_last=True, report_items=False)
    n_img = 6
    batches = list(synth_eval_set("ecssd", shard(n_img), 4, 64))
    res = test_process(tr.model, batches, length=n_img)
    assert tr.model.training                                           # restored
    tot = om.TotalMetric(n_img, with_wfm=False)
    tr.model.eval()
    with torch.no_grad():
        for x, gt in batches:
            p8 = tr.model(x).float().sigmoid().mul(255).byte()[:, 0].cpu().numpy()
            for i in range(p8.shape[0]):
                tot.update(*om.normalise(p8[i], gt[i].cpu().numpy()))
    want = tot.show()
    for k in ("MaxF", "MeanF", "MAE", "EM", "SM"):
        assert res[k] == pytest.approx(float(want[k]), rel=5e-3, abs=1e-4), k   # sigmoid last-ulp ties can move a pixel by 1/255
