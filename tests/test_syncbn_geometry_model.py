"""The SyncBN launch-geometry model (oracle/syncbn_geometry.py) and its covering set, on the CPU.

The GPU regime tests (test_gpu_syncbn_regimes.py) pick their shapes with this model for the device they run on.  Here:
the model's constants are the ones in csrc/syncbn.cu, and on a 132-SM H100 and a 148-SM part alike every kernel
instance reaches every regime axis value (chunks per strip 1, NS-1, NS, NS+1, 2NS+1; last strip equal, 1 chunk, NS+1
chunks or otherwise shorter; full / partial last chunk; 1, a few, grid-filling strips; C = 8 … 2048).
"""
import os
import re

import pytest

from oracle import syncbn_geometry as geo

H100_SMEM_OPTIN = 232448           # cudaDevAttrMaxSharedMemoryPerBlockOptin of sm_90 (and of sm_100)
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sod_project_b200", "csrc", "syncbn.cu")


def test_constants_match_the_kernel_source():
    src = open(SRC).read()
    const = {m.group(1): m.group(2) for m in re.finditer(r"constexpr int (k\w+) = ([^;]+);", src)}
    assert int(const["kThreads"]) == geo.K_THREADS
    assert int(const["kMaxC"]) == geo.K_MAX_C
    assert int(const["kMaxStages"]) == geo.K_MAX_STAGES
    assert int(const["kMaxGrid"]) == geo.K_MAX_GRID
    assert int(const["kRedBytes"]) == geo.K_RED_BYTES
    assert const["kSmemFixed"].split("/*")[0].strip() == "256" and "kRedBytes + 3 * kMaxC * 4" in const["kSmemFixed"]
    assert "nstream * chunk_bytes > 49152" in src and "residual ? 16384 : 32768" in src
    assert "const int nstream = 2 + (pre_add ? 1 : 0) + ((relu && !xmask) ? 1 : 0);" in src


def test_stage_counts_on_hopper():
    """the four ring configurations of the issue table: NS 4 (one 32 KB stream, or two / four smaller), 3, 9"""
    ns = lambda site: geo.make_geom(1, 64, 4, *site, 132, H100_SMEM_OPTIN).nstage  # noqa: E731
    assert ns(geo.fwd_site(False, False)) == 4 and ns(geo.fwd_site(True, False)) == 4
    assert ns(geo.fwd_site(False, True)) == 9 and ns(geo.fwd_site(True, True)) == 4
    assert ns(geo.bwd_site(False, False, False)) == 4 and ns(geo.bwd_site(False, True, False)) == 3
    assert ns(geo.bwd_site(True, True, False)) == 4 and ns(geo.bwd_site(True, True, True)) == 3


@pytest.mark.parametrize("sm_count", [132, 148])
def test_every_instance_reaches_every_regime(sm_count, capsys):
    got, rows = set(), {}
    for case in geo.covering_cases():
        g = geo.resolve(case, sm_count, H100_SMEM_OPTIN)
        assert g is not None, f"{case.id}: {geo.SPECS[case.spec]} unreachable on {sm_count} SMs"
        cls = geo.classify(g, sm_count)
        assert geo.matches(cls, geo.SPECS[case.spec])
        cells = geo.cells(case, g, sm_count)
        got |= cells
        for inst, axis, value in cells:
            rows.setdefault(inst, {}).setdefault((axis, value), 0)
            rows[inst][(axis, value)] += 1
    missing = geo.required_cells(got) - got
    assert not missing, sorted(missing)
    cols = [(a, v) for a, vals in geo.AXES.items() for v in vals]
    with capsys.disabled():
        print(f"\n{sm_count} SMs: cases per instance x regime cell")
        print(" " * 52 + " ".join(f"{a}={v}"[:9].rjust(9) for a, v in cols))
        for inst in sorted(rows):
            print(inst[:51].ljust(52) + " ".join(str(rows[inst].get(c, 0)).rjust(9) for c in cols))


def test_selector_returns_the_smallest_shape():
    """a brute-force scan over row counts never finds a smaller tensor with the requested regime"""
    for want, site in ((dict(n="NS+1", C=64), geo.fwd_site(False, False)), (dict(n="NS", strips="few"), geo.bwd_site(True, True, False)),
                       (dict(n="1", strips="grid", C=16), geo.bwd_site(False, False, False))):
        g = geo.select(want, 2, *site, 132, H100_SMEM_OPTIN)
        assert g is not None and geo.matches(geo.classify(g, 132), want)
        for rows in range(1, g.rows):
            h = geo.make_geom(rows, g.C, 2, *site, 132, H100_SMEM_OPTIN)
            assert not geo.matches(geo.classify(h, 132), want), (want, rows)
