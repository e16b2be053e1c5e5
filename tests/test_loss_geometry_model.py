"""The launch-geometry model of the fused BCE+CEL kernels (oracle/loss_geometry.py) and its covering set, on the CPU.

The GPU regime tests (test_gpu_loss_regimes.py) pick their sizes with this model for the device they run on.  Here: the
model's constants are the ones in csrc/loss.cu; on a 132-SM H100 and a 148-SM part alike each of the ten kernel
instances (five (logits, mask) dtype pairs × resident / ring-streamed kernel) reaches every regime value it can have;
the array form used by the selector agrees with the per-CTA restatement; the selector returns the smallest n; and no
CTA is ever left without elements.
"""
import os
import re

import numpy as np
import pytest

from oracle import loss_geometry as geo

H100_SMEM_OPTIN = 232448           # cudaDevAttrMaxSharedMemoryPerBlockOptin of sm_90
SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sod_project_b200", "csrc", "loss.cu")


def test_constants_match_the_kernel_source():
    src = open(SRC).read()
    const = {m.group(1): m.group(2) for m in re.finditer(r"constexpr int (k\w+) = ([^;]+);", src)}
    assert int(const["kThreads"]) == geo.K_THREADS
    assert int(const["kChunk"]) == geo.K_CHUNK
    assert int(const["kMaxResident"]) == geo.K_MAX_RESIDENT
    assert int(const["kMaxStreamStages"]) == geo.K_MAX_STREAM_STAGES
    assert int(const["kMaxGrid"]) == geo.K_MAX_GRID
    assert "static_cast<size_t>(dv.max_smem_optin) - 128 - 1024" in src and geo.RESIDENT_RESERVE == 128 + 1024
    assert "static_cast<size_t>(dv.max_smem_optin) - 256 - 1024" in src and geo.STREAM_RESERVE == 256 + 1024
    assert "per_cta = (per_cta + 7) & ~7ll;" in src and "if (grid > dv.sm_count) grid = dv.sm_count;" in src
    assert "if (mode == 2) resident = 0;" in src and "if (mode == 1 && need > resident) return SOD_EUNSUPPORTED;" in src


def test_resident_limit_and_stage_count_on_hopper():
    """7 chunks for fp32/fp32, 9 for 2-byte logits with an fp32 mask, 12 when both are 2 bytes: in both kernels"""
    for (sx, sm), k in (((4, 4), 7), ((2, 4), 9), ((2, 2), 12)):
        assert geo.resident_limit(sx, sm, H100_SMEM_OPTIN) == k
        assert geo.stream_stages(sx, sm, H100_SMEM_OPTIN) == k


@pytest.mark.parametrize("sm_count", [132, 148])
def test_every_instance_reaches_every_regime(sm_count, capsys):
    got, table = set(), {}
    for case in geo.covering_cases():
        n, g = geo.resolve(case, sm_count, H100_SMEM_OPTIN)
        assert g is not None, f"{case.id}: {geo.SPECS[case.spec]} unreachable on {sm_count} SMs"
        assert geo.matches(geo.classify(g, sm_count), geo.SPECS[case.spec]), case.id
        for cell in geo.cells(case, g, sm_count):
            got.add(cell)
            table.setdefault(cell[0], {}).setdefault(cell[1:], 0)
            table[cell[0]][cell[1:]] += 1
    missing = geo.required_cells() - got
    assert not missing, sorted(missing)
    assert len(table) == 10
    cols = [(a, v) for a, vals in geo.AXES.items() if a != "kernel" for v in vals]
    with capsys.disabled():
        print(f"\n{sm_count} SMs, {H100_SMEM_OPTIN} B: cases per kernel instance x regime cell (-: unreachable)")
        print(" " * 38 + " ".join(f"{a}={v}"[:10].rjust(10) for a, v in cols))
        for inst in sorted(table):
            kernel = "resident" if inst.startswith("loss_bce_cel_kernel") else "streamed"
            print(inst.ljust(38) + " ".join((str(table[inst].get(c, 0)) if geo.reachable(kernel, *c) else "-").rjust(10)
                                            for c in cols))


def _scalar_codes(n, sx, sm, mode, sm_count, smem):
    cls = geo.classify(geo.launch(n, sx, sm, mode, sm_count, smem), sm_count)
    return {a: (-1 if v is None else geo._code(a, v)) for a, v in cls.items()}


@pytest.mark.parametrize("sm_count, smem", [(3, 3 * 32768 + 1280), (5, 5 * 24576 + 1280), (132, H100_SMEM_OPTIN)])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_array_form_agrees_with_the_per_cta_model(sm_count, smem, mode):
    """`regimes` (CTA 0 and the last CTA only) classifies like `classify(launch(n))`, every n on small devices and a
    sample of n around every chunk boundary on an H100"""
    for sx, sm in ((4, 4), (2, 4), (2, 2)):
        top = sm_count * geo.K_CHUNK * (3 * geo.stream_stages(sx, sm, smem) + 2)
        if sm_count < 10:
            ns = np.arange(1, top + 1)
        else:
            ks = np.arange(0, top // geo.K_CHUNK, sm_count // 4) * geo.K_CHUNK
            ns = np.unique(np.clip((ks[:, None] + np.arange(-40, 41)[None, :]).ravel(), 1, None))
        r = geo.regimes(ns, sx, sm, mode, sm_count, smem)
        pick = ns if sm_count >= 10 else ns[:: max(1, ns.size // 4000)]
        for n in pick:
            i = int(np.searchsorted(ns, n))
            want = _scalar_codes(int(n), sx, sm, mode, sm_count, smem)
            assert {a: int(r[a][i]) for a in want} == want, (int(n), sx, sm)


@pytest.mark.parametrize("sm_count", [1, 2, 3, 7, 132, 148])
def test_no_cta_is_ever_empty(sm_count):
    """for n ≥ 8 every CTA of the grid owns at least one element of the 16-byte-packet part (checked per CTA on small
    grids, through the last CTA's element count up to 40 chunks per CTA on large ones)"""
    if sm_count < 10:
        for n in range(8, sm_count * geo.K_CHUNK * 3):
            g = geo.launch(n, 4, 4, 0, sm_count, H100_SMEM_OPTIN)
            assert min(g.chunks) >= 1, n
    step = 1 << 20
    for start in range(8, sm_count * geo.K_CHUNK * 40, step):
        n = np.arange(start, start + step, dtype=np.int64)
        grid = np.clip(-(-n // geo.K_CHUNK), 1, sm_count)
        per = ((-(-n // grid)) + 7) & ~7
        assert bool(((grid - 1) * per < (n & ~7)).all())


@pytest.mark.parametrize("sm_count, smem", [(3, 3 * 32768 + 1280), (132, H100_SMEM_OPTIN)])
def test_selector_returns_the_smallest_n(sm_count, smem):
    """a plain scan over n with the per-CTA model never finds a smaller n with the requested regime"""
    wants = [dict(kernel="resident", ctas="few", last="partial", tail="1-7"),
             dict(kernel="streamed", mode=2, ctas="few", last="equal"),
             dict(kernel="resident", chunks="2..limit-1", last="fewer", tail="1-7"),
             dict(kernel="streamed", mode=2, chunks="NS-1", last="fewer", tail="1-7")]
    if sm_count < 10:
        wants += [dict(kernel="streamed", chunks="NS+1", last="equal", tail="0"),
                  dict(kernel="streamed", chunks="2NS+1", last="fewer", tail="1-7"),
                  dict(kernel="streamed", mode=2, chunks=">=3NS", last="partial", tail="1-7")]
    for want in wants:
        for sx, sm in ((4, 4), (2, 2)):
            n = geo.select(want, sx, sm, sm_count, smem)
            assert n is not None, want
            mode = want.get("mode", 0)
            g = geo.launch(n, sx, sm, mode, sm_count, smem)
            assert geo.matches(geo.classify(g, sm_count), want)
            # on a large device the scan starts where CTA 0 first has the chunk count of n: chunks only grow with n
            lo = 1
            if sm_count > 10 and g.chunks[0] > 1:
                lo = sm_count * (g.chunks[0] - 1) * geo.K_CHUNK - 8 * sm_count
                assert geo.launch(lo, sx, sm, mode, sm_count, smem).chunks[0] < g.chunks[0]
            for m in range(lo, n):
                cls = geo.classify(geo.launch(m, sx, sm, mode, sm_count, smem), sm_count)
                assert not geo.matches(cls, want), (want, m, n)
