"""The launch-geometry model of the resampling kernels (oracle/resample_geometry.py) and the fp32 replay of `sod_colsum`,
on the CPU.

The GPU regime tests (test_gpu_resample_regimes.py) pick their shapes with this model for the device they run on.
Here: the model's constants are the ones in csrc/resample.cu, csrc/maxpool.cu and csrc/nearest.cu; the grid-stride loops and the colsum
row loop visit every packet / row exactly once; every regime cell is reachable on a 132-SM H100 SXM and a 114-SM H100
PCIe; and the replay of the colsum order equals an exact sum on integer data.
"""
import math
import os
import re

import numpy as np
import pytest

from oracle import resample_geometry as geo

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sod_project_b200", "csrc")
SM_COUNTS = (132, 114)


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_constants_match_the_kernel_sources():
    for name in ("resample.cu", "maxpool.cu", "nearest.cu"):
        src = _src(name)
        assert int(re.search(r"constexpr int kThreads = (\d+);", src).group(1)) == geo.K_THREADS
        body = re.search(r"static unsigned grid_for\(long long packets\) \{(.*?)\n\}", src, re.S).group(1)
        assert "(packets + kThreads - 1) / kThreads" in body
        assert f"const long long cap = {geo.K_CTAS_PER_SM}ll * dev_info().sm_count;" in body
        assert "if (b < 1) b = 1;" in body
        # every grid-stride loop starts at blockIdx.x·kThreads + threadIdx.x and strides by gridDim.x·kThreads
        assert src.count("idx += static_cast<long long>(gridDim.x) * kThreads)") == (4 if name == "resample.cu" else 2)
    src = _src("resample.cu")
    assert f"__launch_bounds__({geo.COLSUM_THREADS}) colsum_kernel" in src
    assert f"(rows + static_cast<long long>(R) * {geo.COLSUM_PASSES} - 1) / (static_cast<long long>(R) * {geo.COLSUM_PASSES})" in src
    assert f"const long long cap = {geo.COLSUM_CTAS_PER_SM}ll * dev_info().sm_count;" in src
    assert f"if (grid > {geo.COLSUM_MAX_GRID}) grid = {geo.COLSUM_MAX_GRID};" in src
    assert f"c <= {geo.COLSUM_MAX_C}" in src and "(L & (L - 1)) == 0" in src
    # the summation order colsum_replay restates
    assert "for (; r + 3 * step < rows; r += 4 * step)" in src
    assert "a[k] += (v0[k] + v1[k]) + (v2[k] + v3[k]);" in src
    assert "for (; r < rows; r += step)" in src
    assert "for (int rr = 0; rr < R; ++rr) t += s_acc[(rr * L + ll) * 8 + k];" in src
    assert "for (unsigned b = 0; b < gridDim.x; ++b) t += __ldcg(partial + static_cast<size_t>(b) * C + ch);" in src
    # the packets each launch writes: (h, w) of the input for the up-sample, of the output for the average pool
    assert "packets = static_cast<long long>(n) * 2 * h * 2 * w * (c / 8);" in src
    assert "packets = static_cast<long long>(n) * 2 * h_out * 2 * w_out * (c / 8);" in src
    assert "packets = static_cast<long long>(n) * ho * wo * (c / 8);" in _src("maxpool.cu")
    # the nearest kernels: one thread per input packet, forward and backward
    src = _src("nearest.cu")
    assert src.count("const long long packets = static_cast<long long>(n) * h * w * (c / 8);") == 2
    assert src.count("<<<grid_for(packets), kThreads, 0, s>>>") == 2


@pytest.mark.parametrize("sm_count", [1, 3, 132])
def test_grid_stride_loops_visit_every_packet_once(sm_count):
    full = geo.K_CTAS_PER_SM * sm_count * geo.K_THREADS
    for p in sorted({1, 255, 256, 257, full - 1, full, full + 1, 2 * full, 2 * full + 3, 3 * full - 5}):
        if p > 600_000 and sm_count > 3:
            continue
        seen = np.concatenate(geo.thread_packets(p, sm_count))
        assert np.array_equal(np.sort(seen), np.arange(p)), p
        counts = geo.passes(p, sm_count)
        assert int(counts.sum()) == p and counts.max() - counts[counts > 0].min() <= 1
        assert geo.classify(p, sm_count) == ("partial" if p < full else "1" if p == full else "1+ragged" if p < 2 * full
                                             else ">=2 exact" if p % full == 0 else ">=2 ragged")


@pytest.mark.parametrize("sm_count", SM_COUNTS)
def test_every_wave_cell_is_reachable(sm_count):
    for kernel in geo.GRID_STRIDE_KERNELS:
        for wave in geo.WAVES:
            shape = geo.select(kernel, wave, sm_count)
            p = geo.packets(kernel, shape)
            assert geo.classify(p, sm_count) == wave, (kernel, wave, shape)
            n, c, h, w = shape
            assert c % 8 == 0 and min(shape) >= 1
            if kernel.startswith("avgpool"):
                assert h % 2 == 0 and w % 2 == 0
            if wave == "partial":
                assert geo.grid_for(p, sm_count) >= 2 and p % geo.K_THREADS != 0
            # the smallest: one packet (four for the ×2 side) less leaves the cell
            m = 4 if kernel in ("upsample_fwd", "avgpool_bwd") else 1
            if wave != "partial":
                assert geo.classify(p - m, sm_count) != wave


@pytest.mark.parametrize("sm_count", [1, 2, 5, 132])
@pytest.mark.parametrize("L", geo.LANES)
def test_colsum_rows_are_each_read_once(sm_count, L):
    R = geo.COLSUM_THREADS // L
    cap = min(geo.COLSUM_CTAS_PER_SM * sm_count, geo.COLSUM_MAX_GRID)
    for rows in sorted({1, 2, R - 1, R, R + 1, 8 * R, 8 * R + 1, 8 * R * cap - 1, 8 * R * cap + 3, 11 * R * cap + 7}):
        if rows < 1 or rows > 400_000:
            continue
        g = geo.colsum_launch(rows, 8 * L, sm_count)
        seen = np.concatenate(list(geo.colsum_thread_rows(g).values()))
        assert np.array_equal(np.sort(seen), np.arange(rows)), rows
        assert int(g.q.sum()) == rows


@pytest.mark.parametrize("sm_count", SM_COUNTS)
def test_every_colsum_cell_is_reachable(sm_count):
    got = set()
    for want in geo.COLSUM_SPECS:
        rows = geo.select_colsum(want, sm_count)
        assert rows is not None, (want, sm_count)
        g = geo.colsum_launch(rows, 8 * want["L"], sm_count)
        cls = geo.classify_colsum(g)
        assert all(cls[k] == v for k, v in want.items())
        if rows > 1:                                # the smallest row count with these properties
            assert not all(v == geo.classify_colsum(geo.colsum_launch(rows - 1, 8 * want["L"], sm_count))[k]
                           for k, v in want.items())
        got |= geo.colsum_cells(g)
    assert not geo.required_colsum_cells() - got, sorted(geo.required_colsum_cells() - got, key=str)


@pytest.mark.parametrize("sm_count", [1, 3, 132])
@pytest.mark.parametrize("rows, c", [(1, 8), (3, 64), (37, 2048), (1000, 16), (5000, 8), (40_001, 64), (70_000, 8)])
def test_colsum_replay_is_exact_on_integers(sm_count, rows, c):
    """integer data whose every partial sum stays below 2²⁴: the replay must be the exact column sum"""
    rng = np.random.default_rng(rows * 7 + c + sm_count)
    x = rng.integers(-64, 65, size=(rows, c)).astype(np.float32)
    got = geo.colsum_replay(x, sm_count)
    want = np.array([math.fsum(col) for col in x.T.astype(np.float64)])
    assert np.array_equal(got.astype(np.float64), want)


def test_colsum_replay_follows_the_kernel_order():
    """on data where fp32 addition is not associative the replay differs from a plain sequential sum (the order is what
    the GPU test compares bit for bit) and stays within fp32 rounding of the float64 sum"""
    rng = np.random.default_rng(5)
    rows, c, sm = 9 * 2 * 3 * 256 + 77, 8, 3
    x = (rng.standard_normal((rows, c)) * np.exp2(rng.integers(-12, 12, (rows, c)))).astype(np.float32)
    got = geo.colsum_replay(x, sm)
    seq = np.zeros(c, np.float32)
    for r in range(rows):
        seq = seq + x[r]
    assert not np.array_equal(got, seq)
    assert np.allclose(got, x.astype(np.float64).sum(0), rtol=0, atol=1e-5 * np.abs(x).astype(np.float64).sum(0).max())
