"""Training on on-disk SOD sets: the augmentation kernel (csrc/augment.cu) against Pillow and torchvision byte for byte,
the `TrainPrefetcher` batch against the reference's per-sample chain, and `train.py` with `"synthetic": false`."""
import itertools
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torchvision.transforms as T
import torchvision.transforms.functional as TF
from PIL import Image

from oracle import pipeline as opipe

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JIT = [TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation]
NORM = T.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])


def _pil_augment(img, mask, flip, angle, order, factor):
    """the reference's RandomHorizontallyFlip → RandomRotate → ColorJitter on PIL images, with given draws"""
    if flip:
        img, mask = img.transpose(Image.FLIP_LEFT_RIGHT), mask.transpose(Image.FLIP_LEFT_RIGHT)
    img, mask = img.rotate(angle, Image.BILINEAR), mask.rotate(angle, Image.NEAREST)
    for op in order:
        img = JIT[op](img, factor[op])
    return img, mask


def _content(rng, n, s):
    img = rng.integers(0, 256, (n, s, s, 3)).astype(np.uint8)
    img[:, : s // 3] = np.where(img[:, : s // 3] > 127, 255, 0)          # saturated band
    yy, xx = np.mgrid[0:s, 0:s]
    img[:, s // 3: 2 * s // 3] = ((xx + yy) * 255 // max(2 * s - 2, 1)).astype(np.uint8)[s // 3: 2 * s // 3, :, None]
    mask = (rng.random((n, s, s)) < 0.4).astype(np.uint8) * 255
    mask[:, : s // 4] = rng.integers(0, 256, (n, s // 4, s))
    return img, mask


def _check_kernel(n, s, seed, force=()):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import augment_u8, draw_augment_params
    rng = np.random.default_rng(seed)
    img, mask = _content(rng, n, s)
    p = draw_augment_params(n, s, torch.Generator().manual_seed(seed))
    for i, fn in force:
        fn(p, i)
    before = _lib.launches
    out, mout = augment_u8(torch.from_numpy(img).cuda(), torch.from_numpy(mask).cuda(), p)
    assert _lib.launches - before == 2                                   # rotate + pre-contrast ops, then contrast + rest
    out, mout = out.cpu().numpy(), mout.cpu().numpy()
    for i in range(n):
        wi, wm = _pil_augment(Image.fromarray(img[i], "RGB"), Image.fromarray(mask[i], "L"), p.flip[i], p.angle[i], p.order[i],
                              p.factor[i])
        assert np.array_equal(out[i], np.asarray(wi)), (s, i, p.angle[i], p.order[i])
        assert np.array_equal(mout[i], np.asarray(wm)), (s, i, p.angle[i])
    return p


def _set(attr, value):
    def fn(p, i):
        getattr(p, attr)[i] = value
    return fn


def test_augment_kernel_bs16_320_equals_pillow_and_torchvision():
    orders = list(itertools.permutations(range(3)))
    force = [(i, _set("order", list(orders[i % 6]))) for i in range(16)]
    force += [(i, _set("flip", bool(i % 2))) for i in range(16)]
    force += [(0, _set("angle", 0.0)), (1, _set("angle", 0.0)), (2, _set("angle", 10.0)), (3, _set("angle", -10.0)),
              (4, _set("angle", 1e-13)), (5, _set("angle", -1e-300)), (6, _set("factor", [1.0, 1.0, 1.0])),
              (7, _set("factor", [float(np.float32(0.9)), float(np.float32(1.1)), 1.0]))]
    p = _check_kernel(16, 320, 11, force)
    assert len({tuple(o) for o in p.order}) == 6 and len(set(p.angle)) >= 14


@pytest.mark.parametrize("s", [1, 2, 3, 37, 64, 257])
def test_augment_kernel_odd_sizes_equal_pillow(s):
    force = [(0, _set("angle", 0.0)), (1, _set("angle", 10.0)), (2, _set("angle", -10.0))]
    _check_kernel(5, s, s, force)


def test_augment_kernel_rejects_bad_arguments():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import draw_augment_params
    lib = _lib.lib()
    n, s = 2, 8
    img = torch.zeros((n, s, s, 3), dtype=torch.uint8, device="cuda")
    mask = torch.zeros((n, s, s), dtype=torch.uint8, device="cuda")
    io, mo = torch.empty_like(img), torch.empty_like(mask)
    ws_n = lib.sod_augment_u8_workspace_bytes(n)
    assert ws_n >= n * 80 + n * 8 and lib.sod_augment_u8_workspace_bytes(0) == 0 and lib.sod_augment_u8_workspace_bytes(-1) == 0
    ws = torch.empty(ws_n, dtype=torch.uint8, device="cuda")
    prm = draw_augment_params(n, s, torch.Generator().manual_seed(0)).c_array()
    args = [img.data_ptr(), mask.data_ptr(), io.data_ptr(), mo.data_ptr(), n, s, prm, ws.data_ptr(), ws_n, _lib.stream_ptr()]
    assert lib.sod_augment_u8(*args) == 0
    for i, bad in [(0, None), (1, None), (2, None), (3, None), (4, 0), (4, -1), (5, 0), (5, -3), (5, 16385), (6, None),
                   (7, None), (8, ws_n - 1), (8, 0)]:
        a = list(args)
        a[i] = bad
        assert lib.sod_augment_u8(*a) == -1, (i, bad)                   # SOD_EINVAL
    for ops in ([0, 1, 3], [0, -1, 2], [0, 0, 1], [2, 2, 2]):
        bad = draw_augment_params(n, s, torch.Generator().manual_seed(0)).c_array()
        bad[1].ops[:] = ops
        a = list(args)
        a[6] = bad
        assert lib.sod_augment_u8(*a) == -1, ops
    torch.cuda.synchronize()


def _write_set(root, n, seed=0):
    """JPEG images of 150–400 px in both orientations, PNG masks with soft edges, one all-black"""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "Image"))
    os.makedirs(os.path.join(root, "Mask"))
    for i in range(n):
        a, b = int(rng.integers(150, 401)), int(rng.integers(150, 401))
        h, w = (max(a, b), min(a, b)) if i % 2 else (min(a, b), max(a, b))
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        img = np.stack([(xx * 255 / w), (yy * 255 / h), rng.integers(0, 256, (h, w))], -1)
        img = np.clip(img + rng.normal(0, 20, img.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(root, "Image", f"img_{i:03d}.jpg"), quality=90)
        cy, cx, r = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w, rng.uniform(0.15, 0.35) * min(h, w)
        m = (np.clip((r - np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)) / 4.0 + 0.5, 0, 1) * 255).round().astype(np.uint8)
        if i == 3:
            m[:] = 0
        Image.fromarray(m, "L").save(os.path.join(root, "Mask", f"img_{i:03d}.png"))
    return root


@pytest.mark.parametrize("size_list", [None, [64, 112]])
def test_prefetched_disk_batch_equals_reference_chain(tmp_path, size_list):
    from distributed_sod_project_b200.data import make_train_loader
    from distributed_sod_project_b200.pipeline import TrainPrefetcher, draw_augment_params
    root = _write_set(str(tmp_path / "TR"), 12)
    S, bs = 96, 5
    pf = TrainPrefetcher(make_train_loader(root, bs, num_workers=2), S, size_list=size_list, seed=3)
    for epoch in (0, 1):
        pf.set_epoch(epoch)
        gen = torch.Generator()
        gen.set_state(pf.gen.get_state())                             # the same draws, replayed on the host
        sizes = __import__("random").Random(3 + epoch)
        n_batches = 0
        for x, m, names in pf:
            assert x.is_cuda and x.shape[0] == bs and m.shape[0] == bs
            p = draw_augment_params(bs, S, gen)
            size = sizes.choice(size_list) if size_list else None
            imgs, masks = [], []
            for i, name in enumerate(names):
                with Image.open(os.path.join(root, "Image", name + ".jpg")) as im:
                    img = im.convert("RGB").resize((S, S))                # JointResize: Pillow's default BICUBIC
                with Image.open(os.path.join(root, "Mask", name + ".png")) as im:
                    mask = im.convert("L").resize((S, S))
                img, mask = _pil_augment(img, mask, p.flip[i], p.angle[i], p.order[i], p.factor[i])
                imgs.append(np.asarray(img))
                masks.append(np.asarray(mask))
                if size is None:
                    assert torch.equal(x[i].cpu(), NORM(TF.to_tensor(img))), name
                    assert torch.equal(m[i].cpu(), TF.to_tensor(mask)), name
            if size is not None:
                wx, wm = opipe.preprocess(torch.from_numpy(np.stack(imgs)), torch.from_numpy(np.stack(masks)), size=size)
                assert x.shape[-1] == size and float((x.cpu() - wx).abs().max()) <= 4e-6
                assert torch.equal(m.cpu(), wm)
            n_batches += 1
        assert n_batches == len(pf) == 12 // bs


def _train(cfg, ngpus, port):
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
    return subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "-ng", str(ngpus), "-p", str(port)], cwd=ROOT, env=env,
                          capture_output=True, text=True, timeout=600)


def _cfg(tmp_path, root, **kw):
    cfg = {"synthetic": False, "epoch_num": 2, "batch_size": 8, "print_freq": 1, "save_freq": 0, "is_distributed": False,
           "input_size": 128, "model": "res50", "cuda_graph": True, "num_workers": 2, "final_test": False, "val_freq": 0,
           "proj_root": str(tmp_path), "rgb_data": {"tr_data_path": root, "val_data_path": {}, "te_data_list": {}}}
    cfg.update(kw)
    return cfg


def _check_run(out, cfg, tmp_path, iters):
    from config import user_config
    from distributed_sod_project_b200.utils import construct_exp_name, construct_path_dict
    assert out.returncode == 0, out.stderr[-3000:]
    assert "End Training" in out.stdout and out.stdout.count("[I:") == iters
    losses = [float(v) for v in re.findall(r"\|Cur:([^|]+)\|", out.stdout)]
    assert len(losses) == iters and all(math.isfinite(v) for v in losses)
    paths = construct_path_dict(str(tmp_path), construct_exp_name(dict(user_config, **cfg)), "x.xlsx")
    assert os.path.getsize(paths["final_full_net"]) > 0


@pytest.mark.parametrize("size_list", [None, [96, 128]])
def test_train_cli_from_disk(tmp_path, size_list):
    root = _write_set(str(tmp_path / "DUTS-TR"), 40, seed=7)
    cfg = _cfg(tmp_path, root, size_list=size_list)
    _check_run(_train(cfg, 1, 29721 if size_list is None else 29722), cfg, tmp_path, 2 * (40 // 8))


def test_train_cli_missing_training_set_names_it(tmp_path):
    ghost = str(tmp_path / "no-such-DUTS-TR")
    out = _train(_cfg(tmp_path, ghost), 1, 29723)
    assert out.returncode != 0 and "no-such-DUTS-TR" in out.stderr


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_train_cli_from_disk_two_gpus(tmp_path):
    root = _write_set(str(tmp_path / "DUTS-TR"), 40, seed=8)
    cfg = _cfg(tmp_path, root, is_distributed=True, batch_size=8)
    _check_run(_train(cfg, 2, 29724), cfg, tmp_path, 2 * (20 // 4))
