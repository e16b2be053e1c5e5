"""Evaluation on on-disk SOD test sets: the Pillow-exact resize kernel (csrc/resize.cu), the ragged metric kernels
(csrc/pipeline.cu), the end-to-end `evaluate.test_process` path over `data.EvalBatch` batches, and the command line
(`train.py` / `test.py` with `"synthetic_eval": false`)."""
import ast
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import metrics as om

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ragged(arrays, channels):
    from distributed_sod_project_b200.pipeline import Ragged
    flat = torch.from_numpy(np.concatenate([a.reshape(-1) for a in arrays])).cuda()
    return Ragged(flat, torch.tensor([a.shape[:2] for a in arrays], dtype=torch.int32), channels)


def _content(rng, h, w, ch):
    """noise over a hard-edged half: every tap and the clipping at 0 and 255 matter"""
    a = rng.integers(0, 256, (h, w) if ch == 1 else (h, w, ch)).astype(np.uint8)
    a[: h // 2] = np.where(a[: h // 2] > 127, 255, 0)
    return a


# (in_h, in_w) → (out_h, out_w): 17 distinct source sizes
L_CASES = [((320, 320), (1000, 1400)), ((320, 320), (300, 400)), ((320, 320), (400, 300)), ((320, 320), (1, 77)),
           ((320, 320), (77, 1)), ((57, 83), (57, 83)), ((1000, 1400), (150, 200)), ((64, 64), (64, 500)),
           ((65, 65), (9, 65)), ((1, 1), (5, 3)), ((1, 90), (40, 1)), ((200, 150), (1200, 900)), ((37, 53), (320, 320)),
           ((333, 222), (222, 333)), ((20, 640), (20, 20)), ((700, 90), (6, 640)), ((2, 2), (1, 1))]
RGB_SOURCES = [(1000, 1400), (1400, 1000), (320, 320), (1, 500), (500, 1), (300, 400), (400, 300), (150, 500),
               (2, 3), (319, 321), (640, 640), (64, 48), (321, 319), (50, 2000), (257, 255), (480, 360)]


def test_resize_kernel_bicubic_l_ragged_equals_pillow():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import resize_u8
    rng = np.random.default_rng(0)
    srcs = [_content(rng, *s, 1) for s, _ in L_CASES]
    before = _lib.launches
    out = resize_u8(_ragged(srcs, 1), torch.tensor([d for _, d in L_CASES], dtype=torch.int32), _lib.SOD_RESIZE_BICUBIC)
    assert _lib.launches - before == 3                   # one launch per pass for the whole batch
    for i, (a, (_, (oh, ow))) in enumerate(zip(srcs, L_CASES)):
        want = np.asarray(Image.fromarray(a, "L").resize((ow, oh), Image.BICUBIC))
        assert np.array_equal(out.image(i).cpu().numpy(), want), L_CASES[i]


def test_resize_kernel_bilinear_rgb_ragged_equals_pillow():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import resize_u8
    rng = np.random.default_rng(1)
    srcs = [_content(rng, h, w, 3) for h, w in RGB_SOURCES]
    out = resize_u8(_ragged(srcs, 3), (320, 320), _lib.SOD_RESIZE_BILINEAR)
    got = out.as_batch().cpu().numpy()
    for i, a in enumerate(srcs):
        want = np.asarray(Image.fromarray(a, "RGB").resize((320, 320), Image.BILINEAR))
        assert np.array_equal(got[i], want), RGB_SOURCES[i]
    # the other two modes over the same ragged batch: L BILINEAR, RGB BICUBIC
    grey = [a[..., 0].copy() for a in srcs]
    outs = resize_u8(_ragged(grey, 1), (200, 300), _lib.SOD_RESIZE_BILINEAR).as_batch().cpu().numpy()
    outc = resize_u8(_ragged(srcs, 3), (300, 200), _lib.SOD_RESIZE_BICUBIC).as_batch().cpu().numpy()
    for i in range(len(srcs)):
        assert np.array_equal(outs[i], np.asarray(Image.fromarray(grey[i], "L").resize((300, 200), Image.BILINEAR)))
        assert np.array_equal(outc[i], np.asarray(Image.fromarray(srcs[i], "RGB").resize((200, 300), Image.BICUBIC)))


def test_resize_kernel_rejects_bad_arguments():
    from distributed_sod_project_b200 import _lib
    lib = _lib.lib()
    src = torch.zeros(64, dtype=torch.uint8, device="cuda")
    dst = torch.zeros(64, dtype=torch.uint8, device="cuda")
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    hw = torch.tensor([[8, 8]], dtype=torch.int32, device="cuda")
    hw_h = torch.tensor([[8, 8]], dtype=torch.int32)
    hw2_h = torch.tensor([[4, 4]], dtype=torch.int32)
    ws_n = lib.sod_resize_u8_workspace_bytes(1, hw_h.data_ptr(), hw2_h.data_ptr(), 1, _lib.SOD_RESIZE_BICUBIC)
    assert ws_n > 0
    ws = torch.zeros(ws_n, dtype=torch.uint8, device="cuda")
    s = _lib.stream_ptr()
    args = [src.data_ptr(), off.data_ptr(), hw.data_ptr(), dst.data_ptr(), off.data_ptr(), hw.data_ptr(), 1, 1,
            _lib.SOD_RESIZE_BICUBIC, ws.data_ptr(), ws_n, s]
    assert lib.sod_resize_u8(*args) == 0
    for i, bad in [(0, None), (1, None), (2, None), (3, None), (4, None), (5, None), (6, 0), (6, -1), (7, 2), (7, 4),
                   (8, 0), (8, 1), (8, 4), (9, None), (10, 0)]:
        a = list(args)
        a[i] = bad
        assert lib.sod_resize_u8(*a) == -1, (i, bad)            # SOD_EINVAL
    for n, ch, f in [(0, 1, 3), (1, 2, 3), (1, 1, 0)]:
        assert lib.sod_resize_u8_workspace_bytes(n, hw_h.data_ptr(), hw2_h.data_ptr(), ch, f) == 0
    zero = torch.tensor([[0, 8]], dtype=torch.int32)
    assert lib.sod_resize_u8_workspace_bytes(1, zero.data_ptr(), hw2_h.data_ptr(), 1, 3) == 0
    assert lib.sod_resize_u8_workspace_bytes(1, None, hw2_h.data_ptr(), 1, 3) == 0


def test_ragged_metric_kernels_count_exactly_and_fixed_entries_agree():
    from distributed_sod_project_b200 import _lib
    rng = np.random.default_rng(2)
    sizes = [(300, 400), (400, 300), (1, 1), (1, 37), (53, 1), (17, 19), (320, 320), (500, 150), (2, 2)]
    preds = [rng.integers(0, 256, s).astype(np.uint8) for s in sizes]
    preds[5][:] = 77                                                   # constant prediction
    gts = [((rng.random(s) < 0.3) * 255).astype(np.uint8) for s in sizes]
    gts[6][:] = 0                                                      # empty ground truth
    gts[7] = rng.integers(0, 256, sizes[7]).astype(np.uint8)           # soft ground truth
    p, g = _ragged(preds, 1), _ragged(gts, 1)
    n = len(sizes)
    lib, s = _lib.lib(), _lib.stream_ptr()
    head = torch.zeros((n, 8), dtype=torch.int64, device="cuda")
    hist = torch.zeros((n, 4, 2, 256), dtype=torch.int32, device="cuda")
    assert lib.sod_saliency_head_ragged(p.data.data_ptr(), g.data.data_ptr(), n, p.off_d.data_ptr(), p.hw_d.data_ptr(),
                                        head.data_ptr(), s) == 0
    want = [om.emulate_kernels(a, b) for a, b in zip(preds, gts)]
    assert np.array_equal(head.cpu().numpy(), np.stack([w[0] for w in want]))
    split = []
    for wh, _ in want:
        nf = max(int(wh[4]), 1)
        split.append([int(round(int(wh[5]) / nf)) + 1, int(round(int(wh[6]) / nf)) + 1])
    split = torch.tensor(split, dtype=torch.int32, device="cuda")
    assert lib.sod_saliency_hist_ragged(p.data.data_ptr(), g.data.data_ptr(), n, p.off_d.data_ptr(), p.hw_d.data_ptr(),
                                        head.data_ptr(), split.data_ptr(), hist.data_ptr(), s) == 0
    hh = hist.cpu().numpy().astype(np.int64)
    for i, (_, wh) in enumerate(want):
        assert np.array_equal(hh[i], wh), sizes[i]
        assert int(hh[i].sum()) == sizes[i][0] * sizes[i][1]
    for bad in [dict(n=0), dict(off=None), dict(hw=None), dict(head=None)]:
        a = dict(n=n, off=p.off_d.data_ptr(), hw=p.hw_d.data_ptr(), head=head.data_ptr())
        a.update(bad)
        assert lib.sod_saliency_head_ragged(p.data.data_ptr(), g.data.data_ptr(), a["n"], a["off"], a["hw"], a["head"], s) == -1
    # the fixed-size entries on an equal-size batch write what the ragged ones write
    eq_p = np.stack([rng.integers(0, 256, (33, 45)).astype(np.uint8) for _ in range(4)])
    eq_g = np.stack([((rng.random((33, 45)) < 0.4) * 255).astype(np.uint8) for _ in range(4)])
    pf, gf = torch.tensor(eq_p).cuda(), torch.tensor(eq_g).cuda()
    pr, gr = _ragged(list(eq_p), 1), _ragged(list(eq_g), 1)
    outs = []
    for ragged in (False, True):
        hd = torch.zeros((4, 8), dtype=torch.int64, device="cuda")
        hs = torch.zeros((4, 4, 2, 256), dtype=torch.int32, device="cuda")
        sp = torch.tensor([[10, 20], [0, 0], [33, 45], [5, 44]], dtype=torch.int32, device="cuda")
        if ragged:
            assert lib.sod_saliency_head_ragged(pr.data.data_ptr(), gr.data.data_ptr(), 4, pr.off_d.data_ptr(), pr.hw_d.data_ptr(), hd.data_ptr(), s) == 0
            assert lib.sod_saliency_hist_ragged(pr.data.data_ptr(), gr.data.data_ptr(), 4, pr.off_d.data_ptr(), pr.hw_d.data_ptr(),
                                                hd.data_ptr(), sp.data_ptr(), hs.data_ptr(), s) == 0
        else:
            assert lib.sod_saliency_head(pf.data_ptr(), gf.data_ptr(), 4, 33, 45, hd.data_ptr(), s) == 0
            assert lib.sod_saliency_hist(pf.data_ptr(), gf.data_ptr(), 4, 33, 45, hd.data_ptr(), sp.data_ptr(), hs.data_ptr(), s) == 0
        outs.append((hd.cpu(), hs.cpu()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def _write_set(root, n=24, seed=0):
    """JPEG images of 150–500 px in both orientations, PNG masks with soft edges; one all-black mask, one stored as RGB
    and one as a palette image"""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "Image"))
    os.makedirs(os.path.join(root, "Mask"))
    for i in range(n):
        a, b = int(rng.integers(150, 501)), int(rng.integers(150, 501))
        h, w = (max(a, b), min(a, b)) if i % 2 else (min(a, b), max(a, b))
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        img = np.stack([(xx * 255 / w), (yy * 255 / h), rng.integers(0, 256, (h, w))], -1)
        img = np.clip(img + rng.normal(0, 20, img.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(root, "Image", f"img_{i:03d}.jpg"), quality=90)
        cy, cx, r = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w, rng.uniform(0.15, 0.35) * min(h, w)
        d = np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)
        m = (np.clip((r - d) / 4.0 + 0.5, 0, 1) * 255).round().astype(np.uint8)
        if i == 3:
            m[:] = 0
        im = Image.fromarray(m, "L")
        if i == 5:
            im = im.convert("RGB")
        elif i == 7:
            im = im.convert("P")
        im.save(os.path.join(root, "Mask", f"img_{i:03d}.png"))
    return root


def test_on_disk_evaluation_end_to_end(tmp_path):
    import torchvision.transforms as T
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.data import make_eval_loader
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.evaluate import prepare_inputs, test_process
    from distributed_sod_project_b200.metrics import SaliencyMetrics
    from distributed_sod_project_b200.pipeline import Ragged, resize_u8
    root = _write_set(str(tmp_path / "SET"))
    S = 96
    tr = Trainer(model_name="res50", dtype=torch.float32, channels_last=True, report_items=False)
    model = tr.model
    model.eval()
    loader, n = make_eval_loader(root, batch_size=5, num_workers=2)
    assert n == 24
    tfm = T.Compose([T.Resize((S, S)), T.ToTensor(), T.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])])
    maps, gts, names = {}, {}, []
    with torch.no_grad():
        for b in loader:
            x, gt = prepare_inputs(b, S)
            for i, name in enumerate(b.names):
                with Image.open(os.path.join(root, "Image", name + ".jpg")) as im:
                    want_x = tfm(im.convert("RGB"))
                assert torch.equal(x[i].cpu(), want_x), name     # Pillow resize, then ToTensor + Normalize exactly
                with Image.open(os.path.join(root, "Mask", name + ".png")) as im:
                    gts[name] = np.asarray(im.convert("L"))
                assert np.array_equal(gt.image(i).cpu().numpy(), gts[name])
            pred_s = SaliencyMetrics.quantize(model(x).float(), apply_sigmoid=True)[:, 0]
            pred = resize_u8(Ragged.stack(pred_s), gt.hw, _lib.SOD_RESIZE_BICUBIC)
            for i, name in enumerate(b.names):
                want = np.asarray(Image.fromarray(pred_s[i].cpu().numpy(), "L").resize(gts[name].shape[::-1]))
                got = pred.image(i).cpu().numpy()
                assert np.array_equal(got, want), name            # ToPILImage + .resize(gt.size), bit for bit
                maps[name] = got
            names += b.names
    assert sorted(names) == sorted(f"img_{i:03d}" for i in range(24))
    save = str(tmp_path / "pre")
    res = test_process(model, loader, length=n, wfm="host", input_size=S, save_dir=save)
    assert sorted(os.listdir(save)) == sorted(f"{k}.png" for k in names)
    tot = om.TotalMetric(n, with_wfm=True)
    for name in names:
        with Image.open(os.path.join(save, name + ".png")) as im:
            saved = np.asarray(im)
        assert saved.shape == gts[name].shape and np.array_equal(saved, maps[name]), name
        tot.update(*om.normalise(saved, gts[name]))
    want = tot.show()
    for k in ("MaxF", "MeanF", "MAE", "EM", "WFM"):
        assert res[k] == pytest.approx(float(want[k]), rel=1e-10), k
    assert res["SM"] == pytest.approx(float(want["SM"]), rel=2e-7)
    # the tuple form keeps working, its resize now Pillow-exact too
    x = torch.randn(2, 3, 64, 64, device="cuda")
    gt = torch.from_numpy(np.stack([gts[names[0]][:50, :70], gts[names[1]][:50, :70]])).cuda()
    res_t = test_process(model, [(x, gt)], length=2)
    with torch.no_grad():
        p8 = SaliencyMetrics.quantize(model(x).float(), apply_sigmoid=True)[:, 0].cpu().numpy()
    tot = om.TotalMetric(2, with_wfm=False)
    for i in range(2):
        tot.update(*om.normalise(np.asarray(Image.fromarray(p8[i], "L").resize((70, 50))), gt[i].cpu().numpy()))
    want = tot.show()
    for k in ("MaxF", "MeanF", "MAE", "EM"):
        assert res_t[k] == pytest.approx(float(want[k]), rel=1e-10), k


def test_cli_train_then_test_on_disk_sets(tmp_path):
    a = _write_set(str(tmp_path / "SETA"), n=7, seed=1)
    b = _write_set(str(tmp_path / "SETB"), n=5, seed=2)
    common = {"epoch_num": 1, "synthetic_iters_per_epoch": 2, "batch_size": 4, "print_freq": 0, "save_freq": 1,
              "is_distributed": False, "input_size": 112, "model": "res50", "output_name": "output_disk_eval",
              "val_freq": 0, "synthetic_eval": False, "num_workers": 2,
              "rgb_data": {"tr_data_path": "", "val_data_path": {"seta": a}, "te_data_list": {"seta": a, "setb": b}}}

    def run(script, cfg):
        env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
        return subprocess.run([sys.executable, os.path.join(ROOT, script)] + (["-ng", "1", "-p", "29711"] if script == "train.py" else []),
                              cwd=ROOT, env=env, capture_output=True, text=True, timeout=500)

    out = run("train.py", common)
    assert out.returncode == 0, out.stderr[-3000:]
    assert out.stdout.count("Results on the testset(") == 2
    from config import user_config
    from distributed_sod_project_b200.utils import construct_exp_name, construct_path_dict
    te_log = construct_path_dict(ROOT, construct_exp_name(dict(user_config, **common)), "x.xlsx")["te_log"]
    start = os.path.getsize(te_log)
    res = run("test.py", dict(common, resume_mode="test"))
    assert res.returncode == 0, res.stderr[-3000:]
    with open(te_log) as f:
        f.seek(start)
        logged = f.read()
    for text in (res.stdout, logged):
        dicts = [ast.literal_eval(m) for m in re.findall(r"\{'MaxF'[^}]*\}", text)]
        assert len(dicts) == 2
        for d in dicts:
            assert set(d) == {"MaxF", "MeanF", "WFM", "MAE", "SM", "EM"} and all(isinstance(v, float) for v in d.values())
    assert "(seta:" in logged and "7 images" in logged and "(setb:" in logged and "5 images" in logged
    missing = dict(common, resume_mode="test", rgb_data=dict(common["rgb_data"], te_data_list={"ghostset": str(tmp_path / "nope")}))
    bad = run("test.py", missing)
    assert bad.returncode != 0 and "ghostset" in bad.stderr
