"""The launch-geometry model of the data-side kernels (oracle/data_geometry.py) and the pre-processing and metric
oracles it is used with, on the CPU.

The GPU regime tests (test_gpu_data_regimes.py) pick their shapes with this model for the device they run on.  Here:
the model's constants are the ones in csrc/pipeline.cu, csrc/resize.cu and csrc/augment.cu; the grid-stride loops visit
every element once; every regime cell is reachable on 1, 114, 132 and 148 SMs with the selected shape landing in its
cell; and the spot values of a 132-SM H100 SXM hold.  The bilinear source coordinate is pinned to torch's CPU
`interpolate` (rounded once) at the rows of real training geometries where rounding twice would differ, and the
metric kernels' integer binarisation `2·g > gmax` to the reference's `g / (gmax + 1e-8) > 0.5` for every byte pair.
"""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import data_geometry as geo
from oracle import pipeline as opipe

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sod_project_b200", "csrc")
SM_COUNTS = (1, 114, 132, 148)

# (n_in, n_out, output rows where one rounding of scale·(o + ½) − ½ and two roundings differ)
TWO_ROUNDING_ROWS = ((320, 224, (1, 22, 179)), (320, 288, (14, 115, 230)), (256, 384, (3, 12, 48, 192)),
                     (384, 416, (17, 277)))


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_constants_match_the_kernel_sources():
    src = _src("pipeline.cu")
    assert "__launch_bounds__(256) preprocess_kernel" in src and "__launch_bounds__(256) metric_hist_kernel" in src
    assert f"const long long cap = {geo.PREP_CTAS_PER_SM}ll * dev_info().sm_count;" in src
    assert f"const long long cap = {geo.QUANT_CTAS_PER_SM}ll * dev_info().sm_count;" in src
    assert src.count("long long blocks = (total + 255) / 256;") == 1 and src.count("long long blocks = (n + 255) / 256;") == 1
    assert src.count("i += static_cast<long long>(gridDim.x) * blockDim.x)") == 2          # preprocess, quantize
    assert f"__launch_bounds__({geo.HEAD_THREADS}) metric_head_kernel" in src
    assert f"metric_head_kernel<<<n, {geo.HEAD_THREADS}, 0," in src
    assert src.count("for (int i = threadIdx.x; i < h * w; i += blockDim.x)") == 2           # head's two loops
    assert "i < h * w; i += gridDim.x * blockDim.x)" in src                                  # hist
    assert f"int per = (h * w + 256 * 16 - 1) / (256 * 16);" in src and 256 * 16 == geo.HIST_PX_PER_CTA
    assert f"int per = ({geo.HIST_RAGGED_CTAS_PER_SM} * dev_info().sm_count + n - 1) / n;" in src
    assert src.count(f"if (per > {geo.HIST_MAX_PER}) per = {geo.HIST_MAX_PER};") == 2
    assert "metric_hist_kernel<<<dim3(per, n), 256, 0," in src
    src = _src("resize.cu")
    assert f"constexpr int kThreads = {geo.THREADS};" in src
    assert f"int per = ({geo.RESIZE_CTAS_PER_SM} * dev_info().sm_count + n - 1) / n;" in src
    assert f"per = per < 1 ? 1 : (per > {geo.RESIZE_MAX_PER} ? {geo.RESIZE_MAX_PER} : per);" in src
    assert "r += gridDim.y)" in src and "yy += gridDim.y)" in src
    src = _src("augment.cu")
    assert f"constexpr int kThreads = {geo.THREADS};" in src and f"constexpr int kPixelsPerCta = {geo.AUG_PIXELS_PER_CTA};" in src
    assert "p.rows_per_tile = size >= kPixelsPerCta ? 1 : kPixelsPerCta / size;" in src
    assert "const int tiles = (size + p.rows_per_tile - 1) / p.rows_per_tile;" in src


@pytest.mark.parametrize("kernel", ["preprocess", "quantize"])
@pytest.mark.parametrize("sm_count", [1, 3])
def test_grid_stride_loops_visit_every_element_once(kernel, sm_count):
    full = geo.full_pass(kernel, sm_count)
    for total in sorted({1, 255, 257, full - 1, full, full + 1, 2 * full, 2 * full + 7, 3 * full - 5}):
        seen = np.concatenate([np.asarray(r) for r in geo.thread_elements(kernel, total, sm_count)])
        assert np.array_equal(np.sort(seen), np.arange(total)), total


@pytest.mark.parametrize("sm_count", SM_COUNTS)
@pytest.mark.parametrize("kernel", geo.KERNELS)
def test_every_cell_is_reachable(kernel, sm_count):
    got = set()
    for cell in sorted(geo.required(kernel, sm_count), key=str):
        shape = geo.select(kernel, cell, sm_count)
        assert cell in geo.cells(kernel, shape, sm_count), (cell, shape)
        got |= geo.cells(kernel, shape, sm_count)
        if kernel in ("preprocess", "quantize") and cell[0] == "wave":
            total = shape[0] if kernel == "quantize" else shape[0] * shape[3] * shape[4]
            if cell[1] == "partial":
                assert geo.grid(kernel, total, sm_count) >= 2 and total % geo.THREADS != 0
            else:            # the smallest: one element (pre-processing: one 8×8 image) less leaves the cell
                assert geo.wave(kernel, total - (64 if kernel == "preprocess" else 1), sm_count) != cell[1]
            if kernel == "preprocess":
                assert geo.prep_mode(*shape[1:]) == cell[2] and min(shape) >= 1
        if kernel in ("hist_ragged", "resize") and cell[0] == "per":
            n = shape[0] if kernel == "resize" else len(shape)
            per_cell = geo.resize_cell if kernel == "resize" else geo.hist_ragged_cell
            assert n == 1 or per_cell(n - 1, sm_count) != cell[1]
    assert geo.required(kernel, sm_count) <= got


def test_spot_values_on_132_sms():
    sm = 132
    assert geo.full_pass("preprocess", sm) == 540_672 and geo.full_pass("quantize", sm) == 270_336
    assert geo.wave("preprocess", 16 * 320 * 320, sm) == ">=2 ragged"          # bs 16 at 320²: 1,638,400 px
    assert [geo.hist_ragged_per(n, sm) for n in (1, 8, 9, 527, 528)] == [64, 64, 59, 2, 1]
    assert [geo.resize_per(n, sm) for n in (1, 8, 9, 1055, 1056)] == [128, 128, 118, 2, 1]
    assert geo.hist_fixed_per(258_048) == 63 and geo.hist_fixed_per(258_049) == 64
    assert geo.hist_fixed_cell(258_048) == "mid" and geo.hist_fixed_cell(258_049) == "cap"
    assert geo.aug_grid(16, 320) == (16, 107) and geo.aug_grid(1, 1024) == (1, 1024)
    assert geo.head_cell(511) == "idle" and geo.head_cell(512_000) == ">=1000"
    assert geo.hist_ragged_per(1, 1) == 4 and geo.resize_per(1, 1) == 8      # one SM: the caps are out of reach


@pytest.mark.parametrize("n_in, n_out, rows", TWO_ROUNDING_ROWS)
def test_bilinear_coordinate_is_rounded_once_as_torch_cpu_does(n_in, n_out, rows):
    """λ of torch's CPU bilinear interpolate is the once-rounded coordinate's at every output row, and at the listed
    rows the twice-rounded coordinate gives a different λ (so a kernel rounding twice is caught there)"""
    i0, i1, lam = opipe.bilinear_taps(n_in, n_out)
    _, _, lam2 = opipe.bilinear_taps(n_in, n_out, fused=False)
    assert sorted(int(r) for r in np.nonzero(lam != lam2)[0]) == list(rows)
    for o in rows:
        x = torch.zeros(1, 1, n_in, 2)
        x[0, 0, i1[o]] = 1.0                               # the output at row o is λ exactly
        got = F.interpolate(x, size=(n_out, 2), mode="bilinear", align_corners=False)[0, 0, o, 0].item()
        assert got == lam[o] != lam2[o], (o, got, lam[o], lam2[o])
    # every row: an image whose row i holds i / 1024 (exact) interpolates to (1 − λ)·i0 + λ·i1 rounded once
    x = (torch.arange(n_in, dtype=torch.float32) / 1024)[None, None, :, None].expand(1, 1, n_in, 2).contiguous()
    got = F.interpolate(x, size=(n_out, 2), mode="bilinear", align_corners=False)[0, 0, :, 0].double().numpy()
    want = ((1 - lam) * i0 + lam * i1) / 1024
    assert np.abs(got - want).max() <= 2.0 ** -24 * n_in / 1024 * 2


@pytest.mark.parametrize("n_in, n_out", [(320, 224), (5, 7), (7, 5), (1, 9), (9, 1), (64, 80)])
def test_nearest_index_matches_torch(n_in, n_out):
    x = torch.arange(n_in, dtype=torch.float32)[None, None, :, None]
    got = F.interpolate(x, size=(n_out, 1), mode="nearest")[0, 0, :, 0].long().numpy()
    assert np.array_equal(got, opipe.nearest_index(n_in, n_out))


def test_normalise_table_is_torch_to_tensor_normalize():
    u = torch.arange(256, dtype=torch.uint8)
    img = u[:, None, None].expand(256, 1, 3).numpy()
    import torchvision.transforms.functional as TF
    want = TF.normalize(TF.to_tensor(img), opipe.MEAN, opipe.STD)[:, :, 0]
    assert torch.equal(opipe.normalise_table(), want)


def test_integer_binarisation_is_the_reference_threshold():
    """for every (g, gmax) byte pair: 2·g > gmax (gmax > 0) is exactly g / (gmax + 1e-8) > 0.5 in float64"""
    g = np.arange(256, dtype=np.float64)[:, None]
    gmax = np.arange(256, dtype=np.float64)[None, :]
    ref = g / (gmax + 1e-8) > 0.5
    kernel = (2 * g > gmax) & (gmax > 0)
    valid = g <= gmax
    assert np.array_equal(ref[valid], kernel[valid])
