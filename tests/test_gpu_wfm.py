"""The weighted F-measure on the GPU (csrc/wfm.cu through `metrics.wfm_sums*` and `SaliencyMetrics(wfm="gpu")`):
the nearest-foreground indices equal scipy's `distance_transform_edt(~gt, return_indices=True)` exactly, in every
launch regime oracle/wfm.py names on this device; Q is within 1e-10 of the host path (`metrics._wfm_host`, scipy) per
image; the sums are bit-identical from run to run and alone or in a batch; refusals touch nothing; and `test_process`
and the command line agree with the host path end to end."""
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
from scipy.ndimage import distance_transform_edt

from oracle import wfm as ow

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-10


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ragged(arrays):
    from distributed_sod_project_b200.pipeline import Ragged
    flat = torch.from_numpy(np.concatenate([a.reshape(-1) for a in arrays])).cuda()
    return Ragged(flat, torch.tensor([a.shape for a in arrays], dtype=torch.int32), 1)


def _head_ragged(p, g):
    from distributed_sod_project_b200 import _lib
    head = torch.empty((len(p), 8), dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().sod_saliency_head_ragged(p.data.data_ptr(), g.data.data_ptr(), len(p), p.off_d.data_ptr(),
                                                   p.hw_d.data_ptr(), head.data_ptr(), _lib.stream_ptr()))
    return head


def run_ragged(preds, gts):
    """(sums float64 [n, 4], nearest per image int32 [h, w, 2]) of the ragged entry"""
    from distributed_sod_project_b200.metrics import wfm_sums_ragged
    p, g = _ragged(preds), _ragged(gts)
    head = _head_ragged(p, g)
    px = sum(a.size for a in preds)
    near = torch.full((px, 2), -7, dtype=torch.int32, device="cuda")
    sums = wfm_sums_ragged(p, g, head, nearest=near)
    torch.cuda.synchronize()
    near_h = near.cpu().numpy()
    out, o = [], 0
    for a in preds:
        out.append(near_h[o:o + a.size].reshape(*a.shape, 2))
        o += a.size
    return sums.cpu().numpy(), out


def check_against_scipy(preds, gts, what=""):
    from distributed_sod_project_b200.metrics import _wfm_host, wfm_from_sums
    sums, near = run_ragged(preds, gts)
    for i, (p8, g8) in enumerate(zip(preds, gts)):
        fg = g8 / (g8.max() + 1e-8) > 0.5
        if fg.any():
            _, (iy, ix) = distance_transform_edt(~fg, return_indices=True)
            assert np.array_equal(near[i][..., 0], iy) and np.array_equal(near[i][..., 1], ix), (what, i, p8.shape)
        else:
            assert (near[i] == -1).all(), (what, i)
            assert (sums[i] == 0).all(), (what, i)
        assert sums[i, 2] == fg.sum() and sums[i, 3] == 0
        assert wfm_from_sums(*sums[i, :3]) == pytest.approx(_wfm_host(p8, g8), rel=TOL, abs=TOL), (what, i, p8.shape)
    return sums


def _content(rng, h, w):
    p8 = rng.integers(0, 256, (h, w)).astype(np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    g8 = (((yy - h * 0.4) ** 2 + (xx - w * 0.6) ** 2 <= (0.3 * min(h, w) + 1) ** 2) | (rng.random((h, w)) < 0.01))
    return p8, (g8 * 255).astype(np.uint8)


def test_nearest_indices_and_wfm_on_mask_families():
    rng = np.random.default_rng(1)
    fam = ow.mask_families(np.random.default_rng(0))
    gts = [(m * 255).astype(np.uint8) for _, m in fam]
    preds = [rng.integers(0, 256, m.shape).astype(np.uint8) for _, m in fam]
    check_against_scipy(preds, gts, "families")


@pytest.mark.parametrize("shape,kind", [((300, 420), "disc"), ((480, 350), "lattice"), ((333, 500), "random"),
                                        ((500, 500), "points")])
def test_nearest_indices_on_image_sized_masks(shape, kind):
    rng = np.random.default_rng(sum(shape))
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w]
    fg = {"disc": (yy - 150) ** 2 + (xx - 200) ** 2 <= 90 ** 2, "lattice": (yy % 37 == 5) & (xx % 29 == 3),
          "random": rng.random(shape) < 0.002, "points": (yy == 0) & (xx == 0) | (yy == h - 1) & (xx == w - 1)}[kind]
    check_against_scipy([rng.integers(0, 256, shape).astype(np.uint8)], [(fg * 200).astype(np.uint8)], kind)


_ran = set()


@pytest.mark.parametrize("cell", ow.REQUIRED, ids=lambda c: f"{c[0]}-{c[1].replace(' ', '_')}")
def test_every_launch_regime(cell):
    sm = _sm()
    hw = ow.select(cell, sm)
    assert cell in ow.cells(hw, sm)
    rng = np.random.default_rng(len(hw) * 1000 + hw[0][0])
    preds, gts = zip(*[_content(rng, h, w) for h, w in hw])
    check_against_scipy(list(preds), list(gts), cell)
    _ran.update(ow.cells(hw, sm))


def test_ragged_mixed_sizes_n1_and_fixed_entry():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.metrics import _wfm_host, wfm_from_sums, wfm_sums
    rng = np.random.default_rng(3)
    sizes = [(300, 400), (1, 1), (1, 90), (90, 1), (57, 83), (400, 300), (129, 257), (32, 32), (33, 31)]
    preds, gts = zip(*[_content(rng, h, w) for h, w in sizes])
    check_against_scipy(list(preds), list(gts), "mixed")
    check_against_scipy([preds[0]], [gts[0]], "n=1")
    # the fixed-size entry (update_batch's) equals the ragged one bit for bit
    h, w = 97, 130
    pr, gr = zip(*[_content(rng, h, w) for _ in range(5)])
    p = torch.from_numpy(np.stack(pr)).cuda()
    g = torch.from_numpy(np.stack(gr)).cuda()
    head = torch.empty((5, 8), dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib().sod_saliency_head(p.data_ptr(), g.data_ptr(), 5, h, w, head.data_ptr(), _lib.stream_ptr()))
    near = torch.empty((5, h, w, 2), dtype=torch.int32, device="cuda")
    fixed = wfm_sums(p, g, head, nearest=near).cpu().numpy()
    ragged, near_r = run_ragged(list(pr), list(gr))
    assert np.array_equal(fixed, ragged)
    assert np.array_equal(near.cpu().numpy(), np.stack(near_r))
    for i in range(5):
        assert wfm_from_sums(*fixed[i, :3]) == pytest.approx(_wfm_host(pr[i], gr[i]), rel=TOL, abs=TOL)


def test_special_cases():
    rng = np.random.default_rng(4)
    h, w = 70, 90
    yy, xx = np.mgrid[0:h, 0:w]
    disc = ((yy - 30) ** 2 + (xx - 40) ** 2 <= 400)
    noise = rng.integers(0, 256, (h, w)).astype(np.uint8)
    cases = {
        "constant prediction": (np.full((h, w), 133, np.uint8), (disc * 255).astype(np.uint8)),
        "constant zero prediction": (np.zeros((h, w), np.uint8), (disc * 255).astype(np.uint8)),
        "empty gt": (noise, np.zeros((h, w), np.uint8)),
        "gt below threshold": (noise, (disc * 255 // 2 + 40 * (~disc)).astype(np.uint8)),   # max 127: 2·40 < 127
        "full gt": (noise, np.full((h, w), 255, np.uint8)),
        "gt max 9": (noise, (disc * 9 + (rng.random((h, w)) < 0.1) * 4).astype(np.uint8)),
        # a binary prediction equal to the ground truth's complement inside the disc: Et = 1 there, EA = E = 1 in the
        # interior up to the rounding of the kernel's sum
        "EA == E ties": (((~disc) * 255).astype(np.uint8), (disc * 255).astype(np.uint8)),
        "EA == E ties, half plane": (np.where(yy < 35, 0, 255).astype(np.uint8), np.where(yy < 35, 255, 0).astype(np.uint8)),
    }
    preds, gts = zip(*cases.values())
    sums = check_against_scipy(list(preds), list(gts), "special")
    assert (sums[2] == 0).all()


def test_sums_are_deterministic_and_independent_of_the_batch():
    rng = np.random.default_rng(5)
    sizes = [(int(rng.integers(300, 501)), int(rng.integers(300, 501))) for _ in range(24)]
    preds, gts = zip(*[_content(rng, h, w) for h, w in sizes])
    a, na = run_ragged(list(preds), list(gts))
    b, nb = run_ragged(list(preds), list(gts))
    assert a.tobytes() == b.tobytes()
    assert all(np.array_equal(x, y) for x, y in zip(na, nb))
    for i in (0, 7, 23):
        alone, _ = run_ragged([preds[i]], [gts[i]])
        assert alone[0].tobytes() == a[i].tobytes(), i


def test_refusals_touch_nothing():
    from distributed_sod_project_b200 import _lib, metrics
    lib = _lib.lib()
    rng = np.random.default_rng(6)
    preds, gts = zip(*[_content(rng, 40, 50), _content(rng, 33, 20)])
    p, g = _ragged(list(preds)), _ragged(list(gts))
    head = _head_ragged(p, g)
    need = lib.sod_saliency_wfm_workspace_bytes(2, p.hw.data_ptr())
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    sums = torch.full((2, 4), 123.5, dtype=torch.float64, device="cuda")
    coef = metrics._wfm_coef_ptr()
    s = _lib.stream_ptr()

    def call(bytes_=need, hw_host=p.hw.data_ptr(), coef_=coef, ws_=ws.data_ptr()):
        return lib.sod_saliency_wfm_ragged(p.data.data_ptr(), g.data.data_ptr(), 2, p.off_d.data_ptr(), p.hw_d.data_ptr(),
                                           hw_host, head.data_ptr(), coef_, ws_, bytes_, sums.data_ptr(), None, s)
    assert call(bytes_=need - 1) == -3                                  # SOD_EWORKSPACE
    assert call(coef_=None) == -1 and call(hw_host=None) == -1 and call(ws_=None) == -1
    assert call(ws_=ws.data_ptr() + 8) == -2                            # SOD_EALIGN
    big = torch.tensor([[40, 50], [1 << 16, 1 << 15]], dtype=torch.int32)
    assert call(hw_host=big.data_ptr()) == -4                           # 2^31 pixels: SOD_EUNSUPPORTED
    wide = torch.tensor([[40, 50], [1, (1 << 21) + 1]], dtype=torch.int32)
    assert call(hw_host=wide.data_ptr()) == -4
    assert lib.sod_saliency_wfm_workspace_bytes(2, big.data_ptr()) == 0
    assert lib.sod_saliency_wfm(p.data.data_ptr(), g.data.data_ptr(), 1, 0, 5, head.data_ptr(), coef, ws.data_ptr(), need,
                                sums.data_ptr(), None, s) == -1
    torch.cuda.synchronize()
    assert (sums.cpu() == 123.5).all()
    assert call() == 0
    torch.cuda.synchronize()
    assert not (sums.cpu() == 123.5).any()
    with pytest.raises(_lib.SodError):
        metrics.wfm_sums(torch.zeros(1, 4, 4, dtype=torch.uint8), torch.zeros(1, 4, 4, dtype=torch.uint8),
                         torch.zeros(1, 8, dtype=torch.int64))
    with pytest.raises(_lib.SodError):
        metrics.SaliencyMetrics(wfm="gpu").update_batch(torch.zeros(1, 4, 4, dtype=torch.uint8),
                                                        torch.zeros(1, 4, 4, dtype=torch.uint8))
    with pytest.raises(ValueError):
        metrics.SaliencyMetrics(wfm="cuda")


def test_saliency_metrics_gpu_equals_host_for_batches_and_ragged():
    from distributed_sod_project_b200.metrics import SaliencyMetrics
    rng = np.random.default_rng(7)
    res = {}
    for mode in ("gpu", "host"):
        cal = SaliencyMetrics(num=11, wfm=mode)
        rng = np.random.default_rng(7)
        pr, gr = zip(*[_content(rng, 45, 61) for _ in range(4)])
        cal.update_batch(torch.from_numpy(np.stack(pr)).cuda(), torch.from_numpy(np.stack(gr)).cuda())
        pr, gr = zip(*[_content(rng, int(rng.integers(20, 200)), int(rng.integers(20, 200))) for _ in range(7)])
        cal.update_ragged(_ragged(list(pr)), _ragged(list(gr)))
        res[mode] = cal.show()
    for k in ("MaxF", "MeanF", "MAE", "SM", "EM"):
        assert res["gpu"][k] == res["host"][k], k
    assert res["gpu"]["WFM"] == pytest.approx(res["host"]["WFM"], rel=TOL, abs=TOL)


def _write_set(root, n, seed):
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "Image"))
    os.makedirs(os.path.join(root, "Mask"))
    for i in range(n):
        h, w = int(rng.integers(60, 140)), int(rng.integers(60, 140))
        img = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(root, "Image", f"img_{i:03d}.jpg"), quality=90)
        yy, xx = np.mgrid[0:h, 0:w]
        m = np.clip((0.3 * min(h, w) - np.sqrt((yy - h / 2) ** 2 + (xx - w / 3) ** 2)) * 40 + 128, 0, 255)
        Image.fromarray(m.astype(np.uint8), "L").save(os.path.join(root, "Mask", f"img_{i:03d}.png"))
    return root


def test_test_process_gpu_equals_host(tmp_path):
    from distributed_sod_project_b200.data import make_eval_loader
    from distributed_sod_project_b200.engine import Trainer
    from distributed_sod_project_b200.evaluate import test_process
    root = _write_set(str(tmp_path / "SET"), 13, 0)
    model = Trainer(model_name="res50", dtype=torch.float32, channels_last=True, report_items=False).model
    loader, n = make_eval_loader(root, batch_size=5, num_workers=0)
    res = {m: test_process(model, loader, length=n, wfm=m, input_size=96, save_dir=str(tmp_path / m)) for m in ("host", "gpu")}
    for name in os.listdir(tmp_path / "host"):                          # the same predictions went into both
        with Image.open(tmp_path / "host" / name) as a, Image.open(tmp_path / "gpu" / name) as b:
            assert np.array_equal(np.asarray(a), np.asarray(b)), name
    for k in ("MaxF", "MeanF", "MAE", "SM", "EM"):
        assert res["gpu"][k] == res["host"][k], k
    assert res["gpu"]["WFM"] == pytest.approx(res["host"]["WFM"], rel=TOL, abs=TOL)


def test_cli_default_wfm_impl_matches_host(tmp_path):
    from distributed_sod_project_b200.metrics import _wfm_host
    a = _write_set(str(tmp_path / "SETA"), 6, 1)
    common = {"epoch_num": 1, "synthetic_iters_per_epoch": 2, "batch_size": 4, "print_freq": 0, "save_freq": 1,
              "is_distributed": False, "input_size": 96, "model": "res50", "output_name": "output_wfm_gpu",
              "val_freq": 0, "synthetic_eval": False, "num_workers": 2,
              "rgb_data": {"tr_data_path": "", "val_data_path": {"seta": a}, "te_data_list": {"seta": a}}}

    def run(script, cfg):
        env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
        out = subprocess.run([sys.executable, os.path.join(ROOT, script)] + (["-ng", "1", "-p", "29731"] if script == "train.py" else []),
                             cwd=ROOT, env=env, capture_output=True, text=True, timeout=500)
        assert out.returncode == 0, out.stderr[-3000:]
        dicts = [ast.literal_eval(m) for m in re.findall(r"\{'MaxF'[^}]*\}", out.stdout)]
        assert len(dicts) == 1 and set(dicts[0]) == {"MaxF", "MeanF", "WFM", "MAE", "SM", "EM"}
        assert all(isinstance(v, float) for v in dicts[0].values())
        return dicts[0]

    from config import user_config
    from distributed_sod_project_b200.utils import construct_exp_name, construct_path_dict
    pre = os.path.join(construct_path_dict(ROOT, construct_exp_name(dict(user_config, **common)), "x.xlsx")["save"], "seta")

    def host_wfm():
        vals = []
        for name in sorted(os.listdir(pre)):
            with Image.open(os.path.join(pre, name)) as p, Image.open(os.path.join(a, "Mask", name)) as g:
                vals.append(_wfm_host(np.asarray(p), np.asarray(g.convert("L"))))
        assert len(vals) == 6
        return float(np.mean(vals))

    gpu = run("train.py", common)                                       # default wfm_impl: the kernels
    assert gpu["WFM"] == pytest.approx(host_wfm(), rel=TOL, abs=TOL)
    host = run("test.py", dict(common, resume_mode="test", wfm_impl="host"))
    assert host["WFM"] == pytest.approx(host_wfm(), rel=TOL, abs=TOL)


def test_zz_every_regime_cell_ran():
    missing = [c for c in ow.REQUIRED if c not in _ran]
    assert not missing, missing
