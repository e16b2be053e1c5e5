"""The weighted F-measure's oracle without a GPU (oracle/wfm.py): its restatement of scipy's feature transform equals
`scipy.ndimage.distance_transform_edt(~fg, return_indices=True)` index for index, ties included; the column kernel's
stackless pass 1 is the envelope with R ≡ 0; the per-image metric equals `metrics._wfm_host` and the unmodified
reference's golden values; the product's host-side Q formula and coefficients are the oracle's; and the launch
geometry's constants are the kernels' and every regime cell is reachable."""
import os
import re

import numpy as np
import pytest
from scipy.ndimage import distance_transform_edt

from oracle import wfm as ow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_feature_transform_equals_scipy_index_for_index():
    for name, fg in ow.mask_families(np.random.default_rng(0)):
        dst, (iy, ix) = distance_transform_edt(~fg, return_indices=True)
        my, mx, md = ow.feature_transform(fg)
        assert np.array_equal(my, iy) and np.array_equal(mx, ix), name
        assert np.array_equal(md, dst), name


@pytest.mark.parametrize("shape,kind", [((300, 420), "disc"), ((480, 350), "lattice"), ((333, 500), "random")])
def test_feature_transform_equals_scipy_on_image_sized_masks(shape, kind):
    rng = np.random.default_rng(sum(shape))
    h, w = shape
    yy, xx = np.mgrid[0:h, 0:w]
    fg = {"disc": (yy - 150) ** 2 + (xx - 200) ** 2 <= 90 ** 2, "lattice": (yy % 37 == 5) & (xx % 29 == 3),
          "random": rng.random(shape) < 0.002}[kind]
    dst, (iy, ix) = distance_transform_edt(~fg, return_indices=True)
    my, mx, md = ow.feature_transform(fg)
    assert np.array_equal(my, iy) and np.array_equal(mx, ix) and np.array_equal(md, dst)


def test_column_pass_is_the_envelope_without_perpendicular_distance():
    for name, fg in ow.mask_families(np.random.default_rng(1)):
        h, w = fg.shape
        want = np.full((h, w), -1, dtype=np.int64)
        for x in range(w):
            pos = np.nonzero(fg[:, x])[0]
            if len(pos):
                want[:, x] = pos[ow.envelope_1d(pos, np.zeros(len(pos), dtype=np.int64), h)]
        assert np.array_equal(ow.column_nearest(fg), want), name


def test_oracle_wfm_equals_host_path_and_reference(golden):
    from distributed_sod_project_b200.metrics import _wfm_host, wfm_from_sums
    g = golden("metrics_kat.npz")
    for i in range(int(g["n"])):
        p8, g8 = g[f"pred{i}"], g[f"gt{i}"]
        mine = ow.wfm(p8, g8)
        assert mine == pytest.approx(_wfm_host(p8, g8), rel=1e-12, abs=1e-12), i
        assert mine == pytest.approx(float(g["wfm"][i]), rel=1e-10, abs=1e-10), i
        assert wfm_from_sums(*ow.wfm_sums(p8, g8)) == mine, i
    rng = np.random.default_rng(2)
    for trial in range(20):
        h, w = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        p8 = rng.integers(0, 256, (h, w)).astype(np.uint8)
        if trial % 4 == 0:
            p8[:] = 77                                          # max == min: u / 255
        g8 = ((rng.random((h, w)) < rng.uniform(0, 0.7)) * int(rng.integers(1, 256))).astype(np.uint8)
        assert ow.wfm(p8, g8) == pytest.approx(_wfm_host(p8, g8), rel=1e-12, abs=1e-12), trial


def test_product_coefficients_are_the_oracles():
    import ctypes
    from distributed_sod_project_b200 import metrics
    assert np.array_equal(metrics.wfm_gaussian(), ow.gaussian_kernel())
    got = np.ctypeslib.as_array((ctypes.c_double * 50).from_address(metrics._wfm_coef_ptr()))
    assert np.array_equal(got, ow.coefficients())
    assert metrics.wfm_from_sums(0.0, 0.0, 0.0) == 0.0


def test_geometry_constants_are_the_kernels():
    src = open(os.path.join(ROOT, "distributed_sod_project_b200", "csrc", "wfm.cu")).read()
    const = {}
    for k, v in re.findall(r"constexpr int (k\w+) = ([^;]+);", src):
        const[k] = int(eval(v, {}, dict(const)))
    assert const["kColThreads"] == ow.COL_THREADS and const["kRowThreads"] == ow.ROW_THREADS
    assert const["kChunk"] == ow.ROW_CHUNK and const["kTile"] == ow.TILE and const["kTileThreads"] == ow.TILE_THREADS
    assert const["kMaxWidth"] == ow.MAX_WIDTH


@pytest.mark.parametrize("sm", [1, 114, 132, 148])
def test_every_regime_cell_is_reachable(sm):
    for cell in ow.REQUIRED:
        assert cell in ow.cells(ow.select(cell, sm), sm), cell
