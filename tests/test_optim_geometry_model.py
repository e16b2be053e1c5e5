"""oracle/optim_geometry.py against csrc/sgd.cu and include/sod_b200.h: the constants, exactly-once coverage of every
grid-stride loop, and every regime cell reachable on 1, 114, 132 and 148 SMs (CPU only)."""
import os
import re

import pytest

from oracle import optim_geometry as geo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = (1, 114, 132, 148)


def _src(rel):
    with open(os.path.join(ROOT, rel)) as f:
        return f.read()


def test_constants_match_the_sources():
    cu = _src("distributed_sod_project_b200/csrc/sgd.cu")
    h = _src("include/sod_b200.h")
    assert re.search(r"constexpr int kThreads = (\d+);", cu).group(1) == str(geo.STEP_THREADS)
    assert re.search(r"constexpr int kUnroll = (\d+);", cu).group(1) == str(geo.STEP_UNROLL)
    assert "const long long cap = 2ll * dev_info().sm_count;" in cu and geo.STEP_CTAS_PER_SM == 2
    assert re.search(r"kGatherChunk = (\d+);", cu).group(1) == str(geo.GATHER_CHUNK)
    assert re.search(r"kCheckChunk = (\d+);", cu).group(1) == str(geo.CHECK_CHUNK)
    assert re.search(r"#define SOD_GATHER_MAX_ITEMS (\d+)", h).group(1) == str(geo.GATHER_MAX_ITEMS)
    assert re.search(r"#define SOD_CHECK_MAX_RANGES (\d+)", h).group(1) == str(geo.CHECK_MAX_RANGES)
    assert "const unsigned cap = 8u * static_cast<unsigned>(dev_info().sm_count);" in cu
    assert "const unsigned cap = 4u * static_cast<unsigned>(dev_info().sm_count);" in cu
    assert "grad_gather16_kernel(const __grid_constant__ GatherTable t" in cu and "for (unsigned i = threadIdx.x; i < nv; i += 256)" in cu
    assert "if (blocks > 4ll * dev_info().sm_count) blocks = 4ll * dev_info().sm_count;" in cu      # nonfinite
    assert "if (blocks > 8ll * dev_info().sm_count) blocks = 8ll * dev_info().sm_count;" in cu      # merge
    assert cu.count("long long blocks = (nvec + 1023) / 1024;") == 2 and cu.count("<<<static_cast<unsigned>(blocks), 256, 0,") == 2
    assert (geo.GATHER_CTAS_PER_SM, geo.CHECK_CTAS_PER_SM, geo.NONFINITE_CTAS_PER_SM, geo.MERGE_CTAS_PER_SM) == (8, 4, 4, 8)


@pytest.mark.parametrize("sm", [1, 3])
@pytest.mark.parametrize("cell", geo.STEP_CELLS)
def test_step_visits_every_vector_once(sm, cell):
    nvec = geo.select("step", cell, sm)
    seen = [0] * nvec
    for v in geo.step_visits(nvec, sm):
        assert v == sorted(v)                    # the segment cursor only moves forward
        for i in v:
            seen[i] += 1
    assert seen == [1] * nvec


@pytest.mark.parametrize("kind", ["nonfinite", "merge"])
@pytest.mark.parametrize("sm", [1, 2])
def test_flat_visits_every_vector_once(kind, sm):
    for cell in geo.FLAT_CELLS:
        nvec = geo.select(kind, cell, sm)
        seen = [0] * nvec
        for r in geo.flat_visits(kind, nvec, sm):
            for i in r:
                seen[i] += 1
        assert seen == [1] * nvec


def test_gather_and_check_cover_every_element_once():
    for sm in (1, 2):
        numels = [1, 7, 8, 13, 8192, 8193, 3 * 8192 + 5] * 30
        cta = geo.gather_chunk_cta(numels, sm)
        assert len(cta) == sum(geo.cdiv(x, geo.GATHER_CHUNK) for x in numels)
        for li, (items, c0, grid) in enumerate(geo.gather_launches(numels, sm)):
            assert len(items) <= geo.GATHER_MAX_ITEMS and grid == min(c0[-1], 8 * sm)
        for x in (1, 7, 8, 13, 8192, 8193, 3 * 8192 + 5):
            for mis in (0, 2, 14):
                seen = []
                for vecs, tail in geo.gather_elements(x, mis):
                    seen += [i for r in vecs for i in r] + tail
                assert sorted(seen) == list(range(x)) and len(seen) == x
        lengths = [0, 5, 4096, 4097, 0] * 60
        total = 0
        for launch in geo.check_launches(lengths, sm):
            if launch is not None:
                live, c0, grid = launch
                total += sum(lengths[i] for i in live)
                assert grid == min(c0[-1], 4 * sm) and all(lengths[i] > 0 for i in live)
        assert total == sum(lengths)


@pytest.mark.parametrize("sm", SMS)
def test_every_cell_is_reachable(sm):
    for cell in geo.STEP_CELLS:
        nvec = geo.select("step", cell, sm)
        assert cell in geo.step_cells(nvec, sm)
    big = geo.select("step", ">=2 passes ragged", sm) + 7
    for cls in geo.EDGE_CLASSES:
        b = geo.edge_at(cls, big, sm)
        assert b is not None and geo.edge_class(b, big, sm) == cls, (cls, sm)
    for kind in ("nonfinite", "merge"):
        for cell in geo.FLAT_CELLS:
            assert geo.flat_cells(kind, geo.select(kind, cell, sm), sm) == {cell}
    for cell in geo.GATHER_CELLS:
        shape = geo.select("gather", cell, sm)
        assert cell in geo.gather_cells(shape, [2] if cell == "misaligned" else [0], sm)
    for cell in geo.CHECK_CELLS:
        assert cell in geo.check_cells(geo.select("check", cell, sm), sm)


def test_spot_values_on_132_sms():
    assert geo.step_grid(6_228_000, 132) == 264 and geo.step_stride(6_228_000, 132) == 135_168
    assert geo.select("step", "cap 1 pass", 132) == 540_672
    assert geo.step_cells(540_673, 132) == {">=2 passes ragged"}
    assert geo.edge_class(135_168, 540_673, 132) == "T" and geo.edge_class(540_672, 600_000, 132) == "pass"
    assert geo.edge_class(512, 600_000, 132) == "cta" and geo.edge_class(5, 600_000, 132) == "unroll"
    assert geo.edge_class(3 * 135_168 + 5, 600_000, 132) is None           # last quarter: advances between groups
    assert geo.gather_launches([8192 * 1057], 132)[0][2] == 1056
    assert [x[2] for x in geo.gather_launches([8] * 161, 132)] == [160, 1]
    assert geo.check_launches([4096 * 529], 132)[0][2] == 528 and geo.check_launches([0] * 128, 132) == [None]
    assert geo.flat_grid("nonfinite", 1 << 20, 132) == 528 and geo.flat_grid("merge", 1 << 20, 132) == 1024
    assert geo.flat_cells("nonfinite", 540_673, 132) == {"cap"}
