"""On-disk training data, host side: oracle/pil_augment.py (the numpy restatement the GPU augmentation kernel is checked
against) equals Pillow's `rotate` and torchvision's ColorJitter operations byte for byte; the host parameter draw has
the reference's distributions; the training sampler is `DistributedSampler`'s."""
import ctypes
import itertools
import math
import os

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as TF
from PIL import Image

from oracle import pil_augment as pa

ANGLES = [10.0, -10.0, 0.0, 1e-12, -1e-12, 1e-300, -1e-300, 0.5, -0.5, 3.3, -7.77, 9.999999, -9.9999999]
SIZES = [(1, 1), (2, 2), (3, 3), (37, 37), (64, 64), (257, 257), (320, 320), (37, 64), (64, 37)]
JIT = [TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation]


def _content(rng, h, w, ch=3):
    """noise with a band saturated at 0 and one at 255"""
    a = rng.integers(0, 256, (h, w, ch) if ch > 1 else (h, w)).astype(np.uint8)
    a[: h // 3] = 0
    a[h // 3: 2 * h // 3] = np.where(a[h // 3: 2 * h // 3] > 100, 255, a[h // 3: 2 * h // 3])
    return a


@pytest.mark.parametrize("hw", SIZES)
def test_rotate_oracle_equals_pillow(hw):
    h, w = hw
    rng = np.random.default_rng(h * 1009 + w)
    for angle in ANGLES + [float(a) for a in rng.uniform(-10, 10, 4)]:
        img, mask = _content(rng, h, w), _content(rng, h, w, 1)
        m, ident = pa.rotate_matrix(angle, w, h)
        got = img.copy() if ident else pa.rotate_bilinear(img, m)
        got_m = mask.copy() if ident else pa.rotate_nearest(mask, m)
        assert np.array_equal(got, np.asarray(Image.fromarray(img, "RGB").rotate(angle, Image.BILINEAR))), (hw, angle)
        assert np.array_equal(got_m, np.asarray(Image.fromarray(mask, "L").rotate(angle, Image.NEAREST))), (hw, angle)


def test_luma_and_blend_oracle_equal_pillow():
    rng = np.random.default_rng(3)
    img = _content(rng, 50, 70)
    assert np.array_equal(pa.luma(img), np.asarray(Image.fromarray(img, "RGB").convert("L")))
    deg = rng.integers(0, 256, img.shape).astype(np.uint8)
    for f in (0.0, 0.3, 0.9, 1.0, 1.1, float(np.float32(1.0999999)), float(np.float32(0.9000001))):
        want = np.asarray(Image.blend(Image.fromarray(deg, "RGB"), Image.fromarray(img, "RGB"), f))
        assert np.array_equal(pa.blend(deg, img, f), want), f


@pytest.mark.parametrize("order", list(itertools.permutations(range(3))))
def test_color_jitter_oracle_equals_torchvision(order):
    rng = np.random.default_rng(sum((i + 1) * o for i, o in enumerate(order)))
    for hw in [(1, 1), (3, 2), (37, 41), (64, 64), (320, 320)]:
        img = _content(rng, *hw)
        factors = [float(np.float32(f)) for f in rng.uniform(0.9, 1.1, 3)]
        for fs in (factors, [1.0, 1.0, 1.0], [float(np.float32(0.9)), float(np.float32(1.1)), 1.0]):
            pil = Image.fromarray(img, "RGB")
            for op in order:
                pil = JIT[op](pil, fs[op])
            got = img
            for op in order:
                got = pa.jitter_op(got, op, fs[op])
            assert np.array_equal(got, np.asarray(pil)), (hw, fs)


@pytest.mark.parametrize("hw", [(37, 37), (64, 64), (320, 320), (37, 64)])
def test_whole_augmentation_oracle_equals_reference_chain(hw):
    """flip → rotate → ColorJitter as the reference's transforms run them on PIL images"""
    h, w = hw
    rng = np.random.default_rng(h + 7 * w)
    for k, order in enumerate(itertools.permutations(range(3))):
        img, mask = _content(rng, h, w), _content(rng, h, w, 1)
        flip, angle = bool(k % 2), float(rng.uniform(-10, 10))
        factors = [float(np.float32(f)) for f in rng.uniform(0.9, 1.1, 3)]
        pi, pm = Image.fromarray(img, "RGB"), Image.fromarray(mask, "L")
        if flip:
            pi, pm = pi.transpose(Image.FLIP_LEFT_RIGHT), pm.transpose(Image.FLIP_LEFT_RIGHT)
        pi, pm = pi.rotate(angle, Image.BILINEAR), pm.rotate(angle, Image.NEAREST)
        for op in order:
            pi = JIT[op](pi, factors[op])
        gi, gm = pa.augment(img, mask, flip, angle, order, factors)
        assert np.array_equal(gi, np.asarray(pi)) and np.array_equal(gm, np.asarray(pm)), (hw, order)


def test_rotate_matrix_is_pillows():
    from distributed_sod_project_b200.pipeline import rotate_matrix
    for angle in ANGLES + [360.0, -360.0, 720.0]:
        for w, h in [(320, 320), (37, 64), (1, 1)]:
            assert rotate_matrix(angle, w, h) == pa.rotate_matrix(angle, w, h)
    assert rotate_matrix(0.0, 5, 5)[1] and rotate_matrix(-360.0, 5, 5)[1] and not rotate_matrix(1e-300, 5, 5)[1]


def test_parameter_draw_support_frequencies_and_seeding():
    from distributed_sod_project_b200 import _lib
    from distributed_sod_project_b200.pipeline import draw_augment_params, rotate_matrix
    n = 24000
    p = draw_augment_params(n, 320, torch.Generator().manual_seed(5))
    assert len(p) == n and p.size == 320
    flips = np.array(p.flip, dtype=np.float64)
    assert abs(flips.mean() - 0.5) < 4 * math.sqrt(0.25 / n)
    ang = np.array(p.angle)
    assert ang.min() >= -10.0 and ang.max() < 10.0 and ang.min() < -9.99 and ang.max() > 9.99
    assert abs(ang.mean()) < 4 * 20 / math.sqrt(12 * n)
    fac = np.array(p.factor, dtype=np.float32)
    assert fac.min() >= np.float32(0.9) and fac.max() <= np.float32(1.1)
    assert np.all(np.abs(fac.mean(0) - 1.0) < 4 * 0.2 / math.sqrt(12 * n))
    orders = [tuple(o) for o in p.order]
    counts = {o: orders.count(o) for o in itertools.permutations(range(3))}
    assert sum(counts.values()) == n and all(abs(c - n / 6) < 4 * math.sqrt(n * (1 / 6) * (5 / 6)) for c in counts.values())
    q = draw_augment_params(n, 320, torch.Generator().manual_seed(5))
    assert (q.flip, q.angle, q.order, q.factor) == (p.flip, p.angle, p.order, p.factor)
    r = draw_augment_params(n, 320, torch.Generator().manual_seed(6))
    assert r.angle != p.angle
    # the C array the kernel reads
    small = draw_augment_params(4, 37, torch.Generator().manual_seed(1))
    small.angle[0] = 0.0
    arr = small.c_array()
    assert ctypes.sizeof(_lib.sod_augment_param) == 80
    for i, e in enumerate(arr):
        m, ident = rotate_matrix(small.angle[i], 37, 37)
        assert list(e.rot) == m and e.identity == int(ident) and e.flip == int(small.flip[i])
        assert list(e.ops) == small.order[i] and list(e.factor) == small.factor[i]
    assert arr[0].identity == 1 and isinstance(arr[0], _lib.sod_augment_param)


def _write_tiny_set(root, n):
    os.makedirs(os.path.join(root, "Image"))
    os.makedirs(os.path.join(root, "Mask"))
    for i in range(n):
        Image.fromarray(np.full((4 + i % 3, 5, 3), i, np.uint8), "RGB").save(os.path.join(root, "Image", f"s{i:03d}.jpg"))
        Image.fromarray(np.full((4 + i % 3, 5), i, np.uint8), "L").save(os.path.join(root, "Mask", f"s{i:03d}.png"))
    return root


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_training_shards_are_distributed_samplers(tmp_path, world):
    from distributed_sod_project_b200.data import list_pairs, make_train_loader
    n, bs = 29, 2
    root = _write_tiny_set(str(tmp_path / "TR"), n)
    names = [os.path.basename(m)[:-4] for _, m in list_pairs(root)]
    for epoch in (0, 3):
        shards = []
        for rank in range(world):
            loader = make_train_loader(root, bs, world, rank, num_workers=0)
            loader.sampler.set_epoch(epoch)
            idx = list(loader.sampler)
            want = torch.utils.data.DistributedSampler(range(n), num_replicas=world, rank=rank, shuffle=True, seed=0)
            want.set_epoch(epoch)
            assert idx == list(want)
            shards.append(idx)
            batches = list(loader)
            assert len(batches) == len(loader) == len(idx) // bs
            for k, b in enumerate(batches):
                assert b.names == [names[j] for j in idx[k * bs:(k + 1) * bs]]
                assert b.img.dtype == torch.uint8 and b.img_hw.tolist() == [[4 + j % 3, 5] for j in idx[k * bs:(k + 1) * bs]]
        # the epoch's permutation padded to a multiple of the world size, dealt out rank by rank: disjoint positions
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(epoch)).tolist()
        padded = perm + perm[:math.ceil(n / world) * world - n]
        assert all(shards[r] == padded[r::world] for r in range(world))
        assert sorted(i for s in shards for i in s) == sorted(padded) and set(padded) == set(range(n))
    assert make_train_loader(root, bs, world, 0).sampler.seed == 0


def test_missing_or_too_small_training_set_is_an_error(tmp_path):
    from distributed_sod_project_b200.data import make_train_loader
    with pytest.raises(FileNotFoundError, match="nowhere"):
        make_train_loader(str(tmp_path / "nowhere"), 4)
    root = _write_tiny_set(str(tmp_path / "TR"), 3)
    with pytest.raises(ValueError, match="no batch"):
        make_train_loader(root, 4)
