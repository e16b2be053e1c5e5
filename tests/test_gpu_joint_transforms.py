"""The reference's other joint transforms on the GPU (csrc/joint.cu, pipeline.py): NEAREST resize, window and Gaussian
blur against Pillow byte for byte in every launch regime of oracle/joint_geometry.py, their refusals, the
`TrainPrefetcher` batches of configured chains against the reference's per-sample PIL chain fed the same draws, and
`train.py` with a configured chain."""
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
from PIL import Image, ImageFilter

from oracle import joint_geometry as jg

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JIT = [TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation]
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
NORM = T.Normalize(MEAN, STD)
MODE = {1: "L", 3: "RGB"}


def _sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _images(rng, hws, ch):
    out = []
    for h, w in hws:
        a = rng.integers(0, 256, (h, w, ch) if ch == 3 else (h, w)).astype(np.uint8)
        a[: h // 3] = np.where(a[: h // 3] > 127, 255, 0)
        out.append(a)
    return out


def _ragged(imgs, ch):
    from distributed_sod_project_b200.pipeline import Ragged
    data = torch.from_numpy(np.concatenate([a.reshape(-1) for a in imgs])).cuda()
    return Ragged(data, torch.tensor([a.shape[:2] for a in imgs], dtype=torch.int32), ch)


def _cases():
    """ragged (src sizes, dst sizes) batches: many images, one large image in several grid-stride passes, an exact
    multiple of a pass, a single pixel, 1×N and N×1"""
    sm = _sm()
    rng = np.random.default_rng(0)
    many = [(int(a), int(b)) for a, b in rng.integers(17, 120, (300, 2))]
    span = jg.MAX_PER * jg.THREADS                                 # bytes of one pass at the largest per
    exact_side = int(math.isqrt(2 * span))                          # "L" side² = 2 passes exactly
    assert exact_side ** 2 == 2 * span and jg.per_of(1, 2 * span, sm) == jg.MAX_PER
    return [
        ("many", many, [(int(a), int(b)) for a, b in rng.integers(17, 120, (300, 2))]),
        ("one large", [(480, 640)], [(701, 933)]),
        ("exact passes", [(200, 300)], [(exact_side, exact_side)]),
        ("two small", [(5, 7), (19, 23)], [(20, 20), (3, 4)]),
        ("pixel and lines", [(1, 1), (1, 40), (40, 1), (9, 9)], [(7, 5), (3, 17), (17, 3), (1, 1)]),
        ("same size", [(37, 61), (61, 37)], [(37, 61), (61, 37)]),
    ]


def test_cases_reach_every_regime():
    sm = _sm()
    for ch in (1, 3):
        reached = set()
        for _, _, dst in _cases():
            reached |= jg.cells(len(dst), [h * w * ch for h, w in dst], sm)
        assert reached == set(jg.REGIMES), (ch, reached)


@pytest.mark.parametrize("ch", [1, 3])
def test_nearest_resize_equals_pillow(ch):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import resize_nearest_u8
    rng = np.random.default_rng(ch)
    for name, src_hw, dst_hw in _cases():
        imgs = _images(rng, src_hw, ch)
        before = _lib.launches
        out = resize_nearest_u8(_ragged(imgs, ch), dst_hw)
        assert _lib.launches - before == 2
        for i, (a, (h, w)) in enumerate(zip(imgs, dst_hw)):
            want = np.asarray(Image.fromarray(a, MODE[ch]).resize((w, h), Image.NEAREST))
            assert np.array_equal(out.image(i).cpu().numpy(), want), (name, i, a.shape, (h, w))


@pytest.mark.parametrize("ch", [1, 3])
def test_window_equals_pillow_crop(ch):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import window_u8
    rng = np.random.default_rng(10 + ch)
    for name, src_hw, dst_hw in _cases():
        imgs = _images(rng, src_hw, ch)
        off = [(int(rng.integers(-h, sh + 1)), int(rng.integers(-w, sw + 1))) for (sh, sw), (h, w) in zip(src_hw, dst_hw)]
        off[0] = (0, 0)
        before = _lib.launches
        out = window_u8(_ragged(imgs, ch), dst_hw, off)
        assert _lib.launches - before == 1
        for i, (a, (h, w), (dy, dx)) in enumerate(zip(imgs, dst_hw, off)):
            want = np.asarray(Image.fromarray(a, MODE[ch]).crop((dx, dy, dx + w, dy + h)))
            assert np.array_equal(out.image(i).cpu().numpy(), want), (name, i, (dy, dx))


BLUR_CASES = [  # (n, h, w): bs 16 at 320², one large image (grid-stride passes), an exact multiple, many small, lines
    (16, 320, 320), (1, 400, 333), (1, 256, 512), (300, 11, 13), (3, 1, 1), (3, 1, 2), (3, 3, 1), (2, 2, 3), (4, 23, 31)]


@pytest.mark.parametrize("ch", [1, 3])
def test_gaussian_blur_equals_pillow(ch):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import gaussian_blur_u8
    rng = np.random.default_rng(20 + ch)
    special = [0.0, 1e-30, 1e-7, 0.05, 0.5, 0.999, 0.99999999, 1.0, 1.7, 3.2, 7.5]
    reached = set()
    for n, h, w in BLUR_CASES:
        reached |= jg.cells(n, [h * w * ch] * n, _sm())
        imgs = _images(rng, [(h, w)] * n, ch)
        radii = [special[i] if i < len(special) and n > 2 else float(rng.random()) * (1 if i % 3 else 4) for i in range(n)]
        x = torch.from_numpy(np.stack(imgs)).cuda()
        before = _lib.launches
        out = gaussian_blur_u8(x, radii).cpu().numpy()
        assert _lib.launches - before == 6
        assert np.array_equal(x.cpu().numpy(), np.stack(imgs))                    # the source is only read
        for i, (a, r) in enumerate(zip(imgs, radii)):
            want = np.asarray(Image.fromarray(a, MODE[ch]).filter(ImageFilter.GaussianBlur(r)))
            assert np.array_equal(out[i], want), ((n, h, w), i, r)
    assert reached == {"one pass", "passes + tail", "passes exact"}          # equal sizes: the largest image sets per


def test_augment_identity_parameters_are_byte_identities():
    """the blur chain runs flip / rotate with jitter factors 1.0 and the jitter with the identity rotation: both must be
    byte identities of what they leave out"""
    from distributed_sod_project_b200.pipeline import AugmentParams, augment_u8, draw_augment_params
    rng = np.random.default_rng(3)
    for n, s in ((16, 320), (5, 37), (3, 1)):
        img = torch.from_numpy(np.stack(_images(rng, [(s, s)] * n, 3))).cuda()
        mask = torch.from_numpy(np.stack(_images(rng, [(s, s)] * n, 1))).cuda()
        p = draw_augment_params(n, s, torch.Generator().manual_seed(n))
        full_i, full_m = augment_u8(img, mask, p)
        ident = AugmentParams(s, [False] * n, [0.0] * n, p.order, [[1.0] * 3] * n)
        oi, om = augment_u8(img, mask, ident)
        assert torch.equal(oi, img) and torch.equal(om, mask)
        geo_i, geo_m = augment_u8(img, mask, AugmentParams(s, p.flip, p.angle, p.order, [[1.0] * 3] * n))
        jit_i, jit_m = augment_u8(geo_i, geo_m, AugmentParams(s, [False] * n, [0.0] * n, p.order, p.factor))
        assert torch.equal(jit_i, full_i) and torch.equal(jit_m, full_m) and torch.equal(geo_m, full_m)


def test_entries_refuse_bad_arguments():
    from distributed_sod_project_b200 import _lib
    lib = _lib.lib()
    EINVAL = -1
    n, ch = 2, 3
    imgs = _images(np.random.default_rng(0), [(8, 9), (5, 4)], ch)
    src = _ragged(imgs, ch)
    dst = _ragged(_images(np.random.default_rng(1), [(6, 7), (6, 7)], ch), ch)
    s_hw = src.hw.contiguous()
    d_hw = dst.hw.contiguous()
    # NEAREST
    ws_n = lib.sod_resize_nearest_u8_workspace_bytes(n, s_hw.data_ptr(), d_hw.data_ptr(), ch)
    assert ws_n >= 4 * (13 + 13)
    assert lib.sod_resize_nearest_u8_workspace_bytes(0, s_hw.data_ptr(), d_hw.data_ptr(), ch) == 0
    assert lib.sod_resize_nearest_u8_workspace_bytes(n, None, d_hw.data_ptr(), ch) == 0
    assert lib.sod_resize_nearest_u8_workspace_bytes(n, s_hw.data_ptr(), d_hw.data_ptr(), 2) == 0
    bad_hw = torch.tensor([[6, 7], [0, 7]], dtype=torch.int32)
    assert lib.sod_resize_nearest_u8_workspace_bytes(n, s_hw.data_ptr(), bad_hw.data_ptr(), ch) == 0
    ws = torch.empty(ws_n, dtype=torch.uint8, device="cuda")
    args = [src.data.data_ptr(), src.off_d.data_ptr(), src.hw_d.data_ptr(), dst.data.data_ptr(), dst.off_d.data_ptr(),
            dst.hw_d.data_ptr(), s_hw.data_ptr(), d_hw.data_ptr(), n, ch, ws.data_ptr(), ws_n, _lib.stream_ptr()]
    assert lib.sod_resize_nearest_u8(*args) == 0
    for i, bad in [(0, None), (1, None), (2, None), (3, None), (4, None), (5, None), (6, None), (7, None), (7, bad_hw.data_ptr()),
                   (8, 0), (8, -1), (9, 2), (9, 4), (10, None), (11, ws_n - 1), (11, 0)]:
        a = list(args)
        a[i] = bad
        assert lib.sod_resize_nearest_u8(*a) == EINVAL, (i, bad)
    # window
    ws_w = lib.sod_window_u8_workspace_bytes(n)
    assert ws_w >= 8 * n and lib.sod_window_u8_workspace_bytes(0) == 0 and lib.sod_window_u8_workspace_bytes(-2) == 0
    wsw = torch.empty(ws_w, dtype=torch.uint8, device="cuda")
    off = torch.tensor([[1, -2], [0, 3]], dtype=torch.int32)
    args = [src.data.data_ptr(), src.off_d.data_ptr(), src.hw_d.data_ptr(), dst.data.data_ptr(), dst.off_d.data_ptr(),
            dst.hw_d.data_ptr(), d_hw.data_ptr(), off.data_ptr(), n, ch, wsw.data_ptr(), ws_w, _lib.stream_ptr()]
    assert lib.sod_window_u8(*args) == 0
    for i, bad in [(0, None), (1, None), (2, None), (3, None), (4, None), (5, None), (6, None), (6, bad_hw.data_ptr()),
                   (7, None), (8, 0), (8, -1), (9, 0), (9, 2), (10, None), (11, ws_w - 1), (11, 0)]:
        a = list(args)
        a[i] = bad
        assert lib.sod_window_u8(*a) == EINVAL, (i, bad)
    # blur
    h, w = 6, 7
    x = torch.zeros((n, h, w, ch), dtype=torch.uint8, device="cuda")
    y = torch.empty_like(x)
    ws_b = lib.sod_gaussian_blur_u8_workspace_bytes(n, h, w, ch)
    assert ws_b >= n * h * w * ch + 12 * n
    for bad in [(0, h, w, ch), (n, 0, w, ch), (n, h, -1, ch), (n, h, w, 2), (n, h, w, 4)]:
        assert lib.sod_gaussian_blur_u8_workspace_bytes(*bad) == 0, bad
    wsb = torch.empty(ws_b, dtype=torch.uint8, device="cuda")
    prm = (_lib.sod_blur_param * n)()
    for p in prm:
        p.radius, p.ww, p.fw = 0, 1 << 24, 0
    args = [x.data_ptr(), y.data_ptr(), n, h, w, ch, prm, wsb.data_ptr(), ws_b, _lib.stream_ptr()]
    assert lib.sod_gaussian_blur_u8(*args) == 0
    for i, bad in [(0, None), (1, None), (2, 0), (2, -1), (3, 0), (4, 0), (5, 2), (6, None), (7, None), (8, ws_b - 1), (8, 0)]:
        a = list(args)
        a[i] = bad
        assert lib.sod_gaussian_blur_u8(*a) == EINVAL, (i, bad)
    for radius, ww, fw in [(-1, 1 << 24, 0), (1025, 1, 0), (0, 0, 0), (0, (1 << 24) + 1, 0), (1, 1 << 23, 0), (0, 1 << 24, 1)]:
        badp = (_lib.sod_blur_param * n)()
        for p in badp:
            p.radius, p.ww, p.fw = 0, 1 << 24, 0
        badp[1].radius, badp[1].ww, badp[1].fw = radius, ww, fw
        a = list(args)
        a[6] = badp
        assert lib.sod_gaussian_blur_u8(*a) == EINVAL, (radius, ww, fw)
    torch.cuda.synchronize()


# ---- TrainPrefetcher with configured chains --------------------------------------------------------------------------
def _write_set(root, n, seed=0):
    """JPEG images of 150–400 px in both orientations and squares, PNG masks with soft edges"""
    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(root, "Image"))
    os.makedirs(os.path.join(root, "Mask"))
    for i in range(n):
        a, b = int(rng.integers(150, 401)), int(rng.integers(150, 401))
        h, w = [(max(a, b), min(a, b)), (min(a, b), max(a, b)), (a, a)][i % 3]
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
        img = np.stack([(xx * 255 / w), (yy * 255 / h), rng.integers(0, 256, (h, w))], -1)
        img = np.clip(img + rng.normal(0, 20, img.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img, "RGB").save(os.path.join(root, "Image", f"img_{i:03d}.jpg"), quality=90)
        cy, cx, r = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w, rng.uniform(0.15, 0.35) * min(h, w)
        m = (np.clip((r - np.sqrt((yy - cy) ** 2 + (xx - cx) ** 2)) / 4.0 + 0.5, 0, 1) * 255).round().astype(np.uint8)
        Image.fromarray(m, "L").save(os.path.join(root, "Mask", f"img_{i:03d}.png"))
    return root


def _ref_chain(img, mask, chain, jp, i):
    """the reference's joint transforms (utils/joint_transforms.py), restated with its Pillow calls, fed draw i of `jp`,
    then ColorJitter with the drawn order and factors"""
    a = jp.augment
    for name, *args in chain:
        if name == "JointResize":
            img, mask = img.resize((args[0], args[0])), mask.resize((args[0], args[0]))
        elif name == "ScaleCenterCrop":
            s = args[0]
            w, h = img.size
            if w > h:
                oh = s
                ow = int(1.0 * w * oh / h)
            else:
                ow = s
                oh = int(1.0 * h * ow / w)
            img, mask = img.resize((ow, oh), Image.BILINEAR), mask.resize((ow, oh), Image.NEAREST)
            w, h = img.size
            x1, y1 = int(round((w - s) / 2.0)), int(round((h - s) / 2.0))
            img, mask = img.crop((x1, y1, x1 + s, y1 + s)), mask.crop((x1, y1, x1 + s, y1 + s))
        elif name == "PaddingSquare":
            x, y = np.asarray(img), np.asarray(mask)
            h, w, c = x.shape
            size = max(h, w)
            ph, pw = (size - h) // 2, (size - w) // 2
            tx, ty = np.zeros((size, size, c)), np.zeros((size, size))
            tx[ph:h + ph, pw:w + pw, :] = x
            ty[ph:h + ph, pw:w + pw] = y
            img = Image.fromarray(tx.astype(np.uint8)).resize((args[0], args[0]))
            mask = Image.fromarray(ty.astype(np.uint8)).resize((args[0], args[0]))
        elif name == "RandomScaleCrop":
            s, (o, x1, y1) = args[0], jp.crop[i]
            img, mask = img.resize((o, o), Image.BILINEAR), mask.resize((o, o), Image.NEAREST)
            img, mask = img.crop((x1, y1, x1 + s, y1 + s)), mask.crop((x1, y1, x1 + s, y1 + s))
        elif name == "RandomHorizontallyFlip":
            if a.flip[i]:
                img, mask = img.transpose(Image.FLIP_LEFT_RIGHT), mask.transpose(Image.FLIP_LEFT_RIGHT)
        elif name == "RandomRotate":
            img, mask = img.rotate(a.angle[i], Image.BILINEAR), mask.rotate(a.angle[i], Image.NEAREST)
        elif name == "RandomGaussianBlur":
            if jp.blur[i] != 0.0:
                img = img.filter(ImageFilter.GaussianBlur(radius=jp.blur[i]))
    for op in a.order[i]:
        img = JIT[op](img, a.factor[i][op])
    return img, mask


S = 96
CHAINS = {
    "default": [["JointResize", S], ["RandomHorizontallyFlip"], ["RandomRotate", 10]],
    "scale_crop_blur": [["JointResize", S], ["RandomScaleCrop", S, 1.5], ["RandomHorizontallyFlip"], ["RandomRotate", 10],
                        ["RandomGaussianBlur"]],
    "scale_center_crop": [["ScaleCenterCrop", S]],
    "padding_square": [["PaddingSquare", S], ["RandomHorizontallyFlip"], ["RandomRotate", 10]],
    "blur_only": [["JointResize", S], ["RandomGaussianBlur"]],
}


@pytest.fixture(scope="module")
def train_set(tmp_path_factory):
    return _write_set(str(tmp_path_factory.mktemp("joint") / "TR"), 15, seed=4)


@pytest.mark.parametrize("chain", list(CHAINS))
def test_prefetched_batch_equals_reference_chain(train_set, chain):
    from distributed_sod_project_b200.data import make_train_loader
    from distributed_sod_project_b200.pipeline import TrainPrefetcher, draw_joint_params
    bs = 5
    pf = TrainPrefetcher(make_train_loader(train_set, bs, num_workers=2), S, seed=3, joint_transforms=CHAINS[chain])
    blurred = cropped = 0
    for epoch in (0, 1):
        pf.set_epoch(epoch)
        gen = torch.Generator()
        gen.set_state(pf.gen.get_state())                             # the same draws, replayed on the host
        n_batches = 0
        for x, m, names in pf:
            jp = draw_joint_params(bs, pf.chain, gen)
            xs, ms = x.cpu(), m.cpu()
            for i, name in enumerate(names):
                with Image.open(os.path.join(train_set, "Image", name + ".jpg")) as im:
                    img = im.convert("RGB")
                with Image.open(os.path.join(train_set, "Mask", name + ".png")) as im:
                    mask = im.convert("L")
                img, mask = _ref_chain(img, mask, CHAINS[chain], jp, i)
                want_u8 = torch.from_numpy(np.asarray(img).copy()).permute(2, 0, 1)
                got_u8 = ((xs[i] * torch.tensor(STD)[:, None, None] + torch.tensor(MEAN)[:, None, None]) * 255).round().to(torch.uint8)
                assert torch.equal(got_u8, want_u8), (chain, name)               # the 8-bit image before Normalize
                assert torch.equal((ms[i, 0] * 255).round().to(torch.uint8), torch.from_numpy(np.asarray(mask).copy()))
                assert torch.equal(xs[i], NORM(TF.to_tensor(img))), (chain, name)
                assert torch.equal(ms[i], TF.to_tensor(mask)), (chain, name)
            blurred += sum(r > 0 for r in jp.blur) if jp.blur else 0
            cropped += sum(o > S for o, _, _ in jp.crop) if jp.crop else 0
            n_batches += 1
        assert n_batches == len(pf) == 15 // bs
    if "blur" in chain:
        assert blurred >= 3
    if "crop_blur" in chain:
        assert cropped >= 3


def test_explicit_default_chain_is_the_reference_path(train_set):
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.data import make_train_loader
    from distributed_sod_project_b200.pipeline import TrainPrefetcher

    def run(chain):
        pf = TrainPrefetcher(make_train_loader(train_set, 5, num_workers=0), S, seed=1, joint_transforms=chain)
        pf.set_epoch(2)
        before = _lib.launches
        out = [(x.cpu(), m.cpu(), names) for x, m, names in pf]
        return out, _lib.launches - before

    a, la = run(None)
    b, lb = run(CHAINS["default"])
    assert la == lb == 3 * (3 + 3 + 2 + 1)                                # resize ×2, augment, preprocess per batch
    for (xa, ma, na), (xb, mb, nb) in zip(a, b):
        assert na == nb and torch.equal(xa, xb) and torch.equal(ma, mb)


def test_train_cli_with_a_configured_chain(tmp_path):
    root = _write_set(str(tmp_path / "DUTS-TR"), 24, seed=9)
    cfg = {"synthetic": False, "epoch_num": 1, "batch_size": 8, "print_freq": 1, "save_freq": 0, "is_distributed": False,
           "input_size": 128, "model": "res50", "cuda_graph": True, "num_workers": 2, "final_test": False, "val_freq": 1,
           "synthetic_eval": False, "save_pre": False, "proj_root": str(tmp_path),
           "joint_transforms": [["JointResize", 128], ["RandomScaleCrop", 128, 1.5], ["RandomHorizontallyFlip"],
                                ["RandomRotate", 10], ["RandomGaussianBlur"]],
           "rgb_data": {"tr_data_path": root, "val_data_path": {"dtr": root}, "te_data_list": {}}}
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "-ng", "1", "-p", "29731"], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "End Training" in out.stdout and out.stdout.count("[I:") == 24 // 8
    losses = [float(v) for v in re.findall(r"\|Cur:([^|]+)\|", out.stdout)]
    assert len(losses) == 3 and all(math.isfinite(v) for v in losses)
    assert "Results on the valset(dtr:" in out.stdout


def test_train_cli_refuses_a_bad_chain(tmp_path):
    root = _write_set(str(tmp_path / "DUTS-TR"), 8, seed=10)
    cfg = {"synthetic": False, "epoch_num": 1, "batch_size": 8, "is_distributed": False, "input_size": 128, "model": "res50",
           "num_workers": 0, "final_test": False, "val_freq": 0, "proj_root": str(tmp_path),
           "joint_transforms": [["RandomHorizontallyFlip"], ["JointResize", 128]],
           "rgb_data": {"tr_data_path": root, "val_data_path": {}, "te_data_list": {}}}
    env = dict(os.environ, SOD_CONFIG_JSON=json.dumps(cfg))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "train.py"), "-ng", "1", "-p", "29732"], cwd=ROOT, env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode != 0 and "joint_transforms[0]" in out.stderr and "accepted order" in out.stderr
