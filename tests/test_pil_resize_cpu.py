"""oracle/pil_resize.py (the numpy restatement the GPU resize kernel is checked against) equals Pillow's `Image.resize`
byte for byte: "L" with BICUBIC and BILINEAR, "RGB" with BILINEAR, over up- and downscales by more than 6×, 1×N and N×1
outputs, one-axis-only changes and the identity."""
import numpy as np
import pytest
from PIL import Image

from oracle import pil_resize as pr

# (in_h, in_w) → (out_h, out_w)
SIZES = [
    ((300, 400), (320, 320)), ((400, 300), (320, 320)), ((1000, 1400), (320, 320)), ((320, 320), (300, 400)),
    ((320, 320), (500, 375)), ((37, 53), (320, 320)), ((320, 320), (41, 29)), ((20, 15), (160, 130)),
    ((320, 320), (1, 77)), ((320, 320), (77, 1)), ((1, 1), (9, 5)), ((1, 60), (30, 1)), ((64, 48), (64, 300)),
    ((64, 48), (7, 48)), ((57, 83), (57, 83)), ((2, 3), (2, 3)), ((700, 90), (5, 640)),
]


@pytest.mark.parametrize("src,dst", SIZES)
@pytest.mark.parametrize("mode,resample", [("L", Image.BICUBIC), ("L", Image.BILINEAR), ("RGB", Image.BILINEAR)])
def test_oracle_equals_pillow(src, dst, mode, resample):
    rng = np.random.default_rng(src[0] * 7919 + dst[1])
    shape = src if mode == "L" else (*src, 3)
    # smooth content with sharp edges: every tap weight and the clipping at 0 and 255 matter
    a = rng.integers(0, 256, shape).astype(np.uint8)
    a[: src[0] // 2] = np.where(a[: src[0] // 2] > 127, 255, 0)
    want = np.asarray(Image.fromarray(a, mode).resize((dst[1], dst[0]), resample))
    got = pr.resize(a, (dst[1], dst[0]), resample)
    assert got.dtype == np.uint8 and got.shape == want.shape
    assert np.array_equal(got, want)


def test_bicubic_is_the_default_of_image_resize():
    """the reference calls `.resize(gt.size)` with no filter: Pillow's default for "L" is BICUBIC"""
    a = np.random.default_rng(0).integers(0, 256, (50, 70)).astype(np.uint8)
    assert np.array_equal(np.asarray(Image.fromarray(a, "L").resize((33, 81))), pr.resize(a, (33, 81), pr.BICUBIC))
