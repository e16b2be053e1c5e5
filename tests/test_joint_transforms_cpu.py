"""The reference's other joint transforms (utils/joint_transforms.py:51-137), host side: oracle/pil_joint.py (the numpy
restatement the GPU kernels of csrc/joint.cu are checked against) equals Pillow byte for byte; each transform composed
from the oracle's pieces and the pipeline's geometry equals the reference's own Pillow calls; the `joint_transforms`
chain is validated; and the parameter draws keep the reference chain's numbers."""
import math

import numpy as np
import pytest
import torch
from PIL import Image, ImageFilter

from oracle import pil_joint as pj
from oracle import pil_resize as pr

NEAREST_SIZES = [((17, 23), (31, 29)), ((40, 57), (13, 11)), ((1, 1), (5, 9)), ((1, 1), (1, 1)), ((1, 9), (4, 3)),
                 ((9, 1), (3, 4)), ((5, 7), (1, 1)), ((1, 40), (1, 17)), ((40, 1), (17, 1)), ((33, 33), (33, 33)),
                 ((300, 400), (320, 320)), ((320, 320), (479, 479)), ((320, 320), (321, 320)), ((100, 640), (37, 320)),
                 ((640, 480), (320, 427)), ((37, 61), (61, 37))]
BLUR_RADII = [0.0, 1e-30, 1e-7, 0.05, 0.3, 0.5, 0.77, 0.999, 0.99999999, 1.0, 1.7, 3.2, 7.5]
BLUR_SIZES = [(1, 1), (1, 2), (5, 1), (2, 3), (3, 3), (4, 2), (23, 31), (64, 37)]


def _img(rng, h, w, mode):
    a = rng.integers(0, 256, (h, w, 3) if mode == "RGB" else (h, w)).astype(np.uint8)
    a[: h // 3] = np.where(a[: h // 3] > 127, 255, 0)            # hard edges, saturated values
    return a


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("src,dst", NEAREST_SIZES)
def test_nearest_oracle_equals_pillow(src, dst, mode):
    rng = np.random.default_rng(src[0] * 7 + dst[1])
    a = _img(rng, *src, mode)
    want = np.asarray(Image.fromarray(a, mode).resize((dst[1], dst[0]), Image.NEAREST))
    assert np.array_equal(pj.resize_nearest(a, (dst[1], dst[0])), want)


def test_nearest_table_is_accumulated_not_a_product():
    """Pillow's repeated addition and `int((x + 0.5)·in/out)` differ at some sizes: the oracle is the former"""
    differ = 0
    for n_in in range(17, 200, 7):
        for n_out in (n_in * 3 // 2, n_in + 5, 2 * n_in + 3, max(n_in // 3, 1)):
            prod = np.array([int((x + 0.5) * (n_in / n_out)) for x in range(n_out)])
            differ += not np.array_equal(pj.nearest_table(n_in, n_out), prod)
            a = np.arange(n_in, dtype=np.uint8)[None]
            assert np.array_equal(pj.resize_nearest(a, (n_out, 1)), np.asarray(Image.fromarray(a, "L").resize((n_out, 1), Image.NEAREST)))
    assert differ > 0


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("hw", BLUR_SIZES)
def test_blur_oracle_equals_pillow(hw, mode):
    rng = np.random.default_rng(hw[0] * 31 + hw[1])
    a = _img(rng, *hw, mode)
    for r in BLUR_RADII + [float(v) for v in rng.random(4)]:
        want = np.asarray(Image.fromarray(a, mode).filter(ImageFilter.GaussianBlur(r)))
        assert np.array_equal(pj.gaussian_blur(a, r), want), (hw, mode, r)


def test_blur_parameters_of_the_product_equal_the_oracle():
    from distributed_sod_project_b200.pipeline import blur_param
    rng = np.random.default_rng(5)
    for r in BLUR_RADII + [float(v) for v in rng.random(200)] + [float(v) for v in rng.uniform(1, 50, 50)]:
        assert blur_param(r) == pj.blur_params(r), r
    radius, ww, fw = blur_param(0.0)
    assert (radius, ww, fw) == (0, 1 << 24, 0)
    for r in rng.random(100):                                     # RandomGaussianBlur's radii: a 3-tap box at most
        radius, ww, fw = blur_param(float(r))
        assert radius == 0 and (2 * radius + 1) * ww + 2 * fw <= 1 << 24


@pytest.mark.parametrize("hw", [(30, 50), (50, 30), (40, 40), (1, 7), (7, 1)])
def test_window_crop_and_pad_equal_pillow_and_numpy(hw):
    h, w = hw
    rng = np.random.default_rng(h + 100 * w)
    for mode in ("L", "RGB"):
        a = _img(rng, h, w, mode)
        for (x1, y1, cw, ch) in [(0, 0, w, h), (1, 2, max(w - 3, 1), max(h - 4, 1)), (w - 1, h - 1, 1, 1), (-3, -2, w + 6, h + 4),
                                 (w // 2, h // 2, w, h)]:
            want = np.asarray(Image.fromarray(a, mode).crop((x1, y1, x1 + cw, y1 + ch)))
            assert np.array_equal(pj.window(a, (ch, cw), y1, x1), want), (mode, x1, y1, cw, ch)
        from distributed_sod_project_b200.pipeline import padding_square_geometry
        side, (dy, dx) = padding_square_geometry(h, w)
        size = max(h, w)
        pad = np.zeros((size, size) + a.shape[2:])                  # the reference's PaddingSquare, in numpy
        pad[(size - h) // 2: h + (size - h) // 2, (size - w) // 2: w + (size - w) // 2] = a
        assert np.array_equal(pj.window(a, (side, side), dy, dx), pad.astype(np.uint8))


# ---- the reference's transforms, restated with their own Pillow calls, against the composed pieces ------------------
def _ref_random_scale_crop(img, mask, s, o, x1, y1):
    img, mask = img.resize((o, o), Image.BILINEAR), mask.resize((o, o), Image.NEAREST)
    box = (x1, y1, x1 + s, y1 + s)
    return img.crop(box), mask.crop(box)


def _ref_scale_center_crop(img, mask, s):
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
    box = (x1, y1, x1 + s, y1 + s)
    return img.crop(box), mask.crop(box)


def _ref_padding_square(img, mask, s):
    x, y = np.asarray(img), np.asarray(mask)
    h, w, c = x.shape
    size = max(h, w)
    ph, pw = (size - h) // 2, (size - w) // 2
    tx, ty = np.zeros((size, size, c)), np.zeros((size, size))
    tx[ph:h + ph, pw:w + pw, :] = x
    ty[ph:h + ph, pw:w + pw] = y
    return Image.fromarray(tx.astype(np.uint8)).resize((s, s)), Image.fromarray(ty.astype(np.uint8)).resize((s, s))


def _pair(rng, h, w):
    return _img(rng, h, w, "RGB"), _img(rng, h, w, "L")


@pytest.mark.parametrize("s,f", [(24, 1.5), (31, 1.0), (17, 2.0)])
def test_random_scale_crop_composed_equals_reference(s, f):
    rng = np.random.default_rng(s)
    a, m = _pair(rng, s, s)
    for o in sorted({s, int(s * f), (s + int(s * f)) // 2}):
        for x1, y1 in {(0, 0), (o - s, o - s), (o - s, 0), ((o - s) // 2, (o - s) // 3)}:
            wi, wm = _ref_random_scale_crop(Image.fromarray(a, "RGB"), Image.fromarray(m, "L"), s, o, x1, y1)
            gi = pj.window(pr.resize(a, (o, o), pr.BILINEAR), (s, s), y1, x1)
            gm = pj.window(pj.resize_nearest(m, (o, o)), (s, s), y1, x1)
            assert np.array_equal(gi, np.asarray(wi)) and np.array_equal(gm, np.asarray(wm)), (o, x1, y1)


@pytest.mark.parametrize("hw", [(30, 47), (47, 30), (36, 36), (21, 64), (33, 32)])
@pytest.mark.parametrize("s", [16, 25])
def test_scale_center_crop_composed_equals_reference(hw, s):
    from distributed_sod_project_b200.pipeline import scale_center_crop_geometry
    rng = np.random.default_rng(hw[0] * s)
    a, m = _pair(rng, *hw)
    wi, wm = _ref_scale_center_crop(Image.fromarray(a, "RGB"), Image.fromarray(m, "L"), s)
    (oh, ow), (y1, x1) = scale_center_crop_geometry(*hw, s)
    gi = pj.window(pr.resize(a, (ow, oh), pr.BILINEAR), (s, s), y1, x1)
    gm = pj.window(pj.resize_nearest(m, (ow, oh)), (s, s), y1, x1)
    assert np.array_equal(gi, np.asarray(wi)) and np.array_equal(gm, np.asarray(wm))


def test_scale_center_crop_rounds_half_to_even():
    from distributed_sod_project_b200.pipeline import scale_center_crop_geometry
    assert scale_center_crop_geometry(10, 15, 10) == ((10, 15), (0, 2))       # (15 − 10) / 2 = 2.5 → 2
    assert scale_center_crop_geometry(10, 17, 10) == ((10, 17), (0, 4))       # 3.5 → 4
    assert scale_center_crop_geometry(13, 10, 10) == ((13, 10), (2, 0))       # 1.5 → 2


@pytest.mark.parametrize("hw", [(30, 47), (47, 30), (36, 36), (1, 9)])
def test_padding_square_composed_equals_reference(hw):
    from distributed_sod_project_b200.pipeline import padding_square_geometry
    rng = np.random.default_rng(hw[1])
    a, m = _pair(rng, *hw)
    s = 24
    wi, wm = _ref_padding_square(Image.fromarray(a, "RGB"), Image.fromarray(m, "L"), s)
    side, (dy, dx) = padding_square_geometry(*hw)
    gi = pr.resize(pj.window(a, (side, side), dy, dx), (s, s), pr.BICUBIC)
    gm = pr.resize(pj.window(m, (side, side), dy, dx), (s, s), pr.BICUBIC)       # the mask too: Pillow's default filter
    assert np.array_equal(gi, np.asarray(wi)) and np.array_equal(gm, np.asarray(wm))


# ---- the chain -----------------------------------------------------------------------------------------------------
def test_default_chain_and_parse():
    from distributed_sod_project_b200.pipeline import default_joint_transforms, parse_joint_transforms
    assert parse_joint_transforms(None, 320) == [["JointResize", 320], ["RandomHorizontallyFlip"], ["RandomRotate", 10]]
    assert parse_joint_transforms(default_joint_transforms(64), 64) == default_joint_transforms(64)
    for chain in ([["ScaleCenterCrop", 64]], [["PaddingSquare", 64], ["RandomHorizontallyFlip"], ["RandomRotate", 5]],
                  [["JointResize", 64], ["RandomScaleCrop", 64, 1.5], ["RandomHorizontallyFlip"], ["RandomRotate", 10],
                   ["RandomGaussianBlur"]],
                  [["JointResize", 64], ["RandomGaussianBlur"]], (("JointResize", 64), ("RandomRotate", 2.5))):
        assert parse_joint_transforms(chain, 64) == [list(e) for e in chain]


@pytest.mark.parametrize("chain,entry", [
    ([], None),
    ("JointResize", None),
    ([["RandomHorizontallyFlip"], ["JointResize", 64]], "joint_transforms[0]"),
    ([["JointResize", 64], ["ScaleCenterCrop", 64]], "joint_transforms[1]"),
    ([["JointResize", 64], ["RandomRotate", 10], ["RandomHorizontallyFlip"]], "joint_transforms[2]"),
    ([["JointResize", 64], ["RandomGaussianBlur"], ["RandomScaleCrop", 64, 1.5]], "joint_transforms[2]"),
    ([["JointResize", 64], ["RandomHorizontallyFlip"], ["RandomHorizontallyFlip"]], "joint_transforms[2]"),
    ([["JointResize", 64], ["RandomCrop", 64]], "joint_transforms[1]"),
    ([["JointResize"]], "joint_transforms[0]"),
    ([["JointResize", 64, 64]], "joint_transforms[0]"),
    ([["JointResize", [64, 64]]], "joint_transforms[0]"),
    ([["JointResize", 0]], "joint_transforms[0]"),
    ([["JointResize", True]], "joint_transforms[0]"),
    ([["JointResize", 32]], "joint_transforms[0]"),
    ([["PaddingSquare", 96]], "joint_transforms[0]"),
    ([["ScaleCenterCrop", 64.0]], "joint_transforms[0]"),
    ([["JointResize", 48], ["RandomScaleCrop", 48, 1.5]], "joint_transforms[0]"),
    ([["JointResize", 64], ["RandomScaleCrop", 48, 1.5]], "joint_transforms[1]"),
    ([["JointResize", 64], ["RandomScaleCrop", 64, 0.5]], "joint_transforms[1]"),
    ([["JointResize", 64], ["RandomRotate", float("nan")]], "joint_transforms[1]"),
    ([["JointResize", 64], ["RandomRotate", "10"]], "joint_transforms[1]"),
    ([["JointResize", 64], ["RandomHorizontallyFlip", 0.5]], "joint_transforms[1]"),
    ([["JointResize", 64], 7], "joint_transforms[1]"),
])
def test_chain_validation_names_the_entry(chain, entry):
    from distributed_sod_project_b200.pipeline import parse_joint_transforms
    with pytest.raises(ValueError) as e:
        parse_joint_transforms(chain, 64)
    msg = str(e.value)
    assert "size step first" in msg or "input_size" in msg or "must be" in msg
    if entry is not None:
        assert entry in msg and repr(chain[int(entry[-2])]) in msg
    if entry is not None and "takes" not in msg and "must be" not in msg and "needs a square" not in msg:
        assert "accepted order" in msg


def _same_augment(a, b):
    return (a.size, a.flip, a.angle, a.order, a.factor) == (b.size, b.flip, b.angle, b.order, b.factor)


def test_default_chain_draws_the_reference_numbers():
    from distributed_sod_project_b200.pipeline import default_joint_transforms, draw_augment_params, draw_joint_params
    for seed in range(5):
        g1, g2 = torch.Generator().manual_seed(seed), torch.Generator().manual_seed(seed)
        for n in (1, 5, 16):
            jp = draw_joint_params(n, default_joint_transforms(96), g1)
            assert _same_augment(jp.augment, draw_augment_params(n, 96, g2)) and jp.crop is None and jp.blur is None
        assert torch.equal(g1.get_state(), g2.get_state())


def test_added_steps_keep_the_reference_draws_and_follow_them():
    from distributed_sod_project_b200.pipeline import default_joint_transforms, draw_augment_params, draw_joint_params
    s, f, n = 64, 1.5, 400
    chain = [["JointResize", s], ["RandomScaleCrop", s, f], ["RandomHorizontallyFlip"], ["RandomRotate", 10],
             ["RandomGaussianBlur"]]
    g1, g2 = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
    jp = draw_joint_params(n, chain, g1)
    assert _same_augment(jp.augment, draw_augment_params(n, s, g2))
    u = torch.rand(n, 3, generator=g2, dtype=torch.float64).tolist()         # then the crop triples, then the blur
    on = (torch.rand(n, generator=g2, dtype=torch.float64) < 0.5).tolist()
    rad = torch.rand(n, generator=g2, dtype=torch.float64).tolist()
    hi = int(s * f)
    for (o, x1, y1), (u0, u1, u2) in zip(jp.crop, u):
        assert o == s + math.floor(u0 * (hi - s + 1)) and x1 == math.floor(u1 * (o - s + 1)) and y1 == math.floor(u2 * (o - s + 1))
        assert s <= o <= hi and 0 <= x1 <= o - s and 0 <= y1 <= o - s
    assert {o for o, _, _ in jp.crop} == set(range(s, hi + 1))                # both ends reached
    assert jp.blur == [r if b else 0.0 for b, r in zip(on, rad)]
    assert 150 < sum(b > 0 for b in jp.blur) < 250
    # no flip / rotate in the chain: the draws are still made, and the flips and angles are the identity
    g3, g4 = torch.Generator().manual_seed(4), torch.Generator().manual_seed(4)
    jp = draw_joint_params(8, [["ScaleCenterCrop", s]], g3)
    ref = draw_augment_params(8, s, g4)
    assert jp.augment.flip == [False] * 8 and jp.augment.angle == [0.0] * 8
    assert (jp.augment.order, jp.augment.factor) == (ref.order, ref.factor)
    assert torch.equal(g3.get_state(), g4.get_state())
    # another degree: r·2·degree − degree of the same r
    g5, g6 = torch.Generator().manual_seed(6), torch.Generator().manual_seed(6)
    jp = draw_joint_params(8, default_joint_transforms(s)[:2] + [["RandomRotate", 30]], g5)
    ref = draw_augment_params(8, s, g6)
    assert [a * 3 for a in ref.angle] == pytest.approx(jp.augment.angle, abs=1e-12)
