"""The launch-geometry model of the peer-memory collectives (oracle/comm_geometry.py), on the CPU.

tests/test_gpu_virtual_world.py sizes its W-rank cases with this model and checks every launch's grid against it.
Here: the model's constants and formulas are the ones in csrc/sgd.cu and include/sod_b200.h, the shard restatement agrees
with `FusedOptimizer.shard_bounds`, the case selector returns the smallest n of each regime and only co-resident cases,
and on a 132-SM H100 (and other SM counts) every regime the co-residency rule admits is reached at W = 2, 3, 4 and 8.
"""
import os
import re

import pytest

from oracle import comm_geometry as geo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SGD = os.path.join(ROOT, "distributed_sod_project_b200", "csrc", "sgd.cu")
HDR = os.path.join(ROOT, "include", "sod_b200.h")
COMMON = os.path.join(ROOT, "distributed_sod_project_b200", "csrc", "common.cuh")
WORLDS = (2, 3, 4, 8)


def test_constants_match_the_kernel_source():
    src = open(SGD).read()
    const = {m.group(1): m.group(2) for m in re.finditer(r"constexpr int (k\w+) = ([^;]+);", src)}
    assert int(const["kThreads"]) == geo.K_THREADS
    assert int(const["kUnroll"]) == geo.K_UNROLL
    hdr = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define (SOD_\w+) (\d+)", open(HDR).read())}
    assert hdr["SOD_MAX_WORLD"] == geo.SOD_MAX_WORLD
    assert hdr["SOD_COMM_MAX_BLOCKS"] == geo.SOD_COMM_MAX_BLOCKS
    assert hdr["SOD_COMM_CHANNELS"] == geo.SOD_COMM_CHANNELS
    # comm_grid, the shard, the one-shot cap and the algo-0 choice, as the host writes them
    assert "(vecs_per_rank + static_cast<long long>(kThreads) * kUnroll - 1) / (static_cast<long long>(kThreads) * kUnroll)" in src
    assert "dev_info().sm_count < SOD_COMM_MAX_BLOCKS ? dev_info().sm_count : SOD_COMM_MAX_BLOCKS" in src
    assert "if (blocks < 1) blocks = 1;" in src and "if (blocks > cap) blocks = cap;" in src
    assert src.count("const long long shard = (nvec + c.world - 1) / c.world;") == 2
    assert "const unsigned grid = comm_grid((nvec + c.world - 1) / c.world);" in src
    assert "static_cast<long long>(kThreads) * kUnroll *" in src and "if (algo == 1 && nvec > one_shot_cap) return SOD_EUNSUPPORTED;" in src
    assert "if (algo == 0) algo = (!has_mc && n * 4 <= (256 << 10)) ? 1 : 2;" in src and geo.ONE_SHOT_AUTO_BYTES == 256 << 10
    assert "if (algo == 1) {\n        const unsigned grid = comm_grid(nvec);" in src
    # barrier channels and the two barriers per CTA and launch
    assert src.count("comm_block_barrier(c, 0, blockIdx.x)") == geo.BARRIERS_PER_LAUNCH          # the step kernel
    assert src.count("comm_block_barrier(c, 3, blockIdx.x)") == 2 * geo.BARRIERS_PER_LAUNCH      # one- and two-shot
    assert "uint32_t* slot = c.block_seq + channel * SOD_COMM_MAX_BLOCKS + block;" in open(COMMON).read()


@pytest.mark.parametrize("world", WORLDS)
def test_shards_tile_the_buffer_like_the_host(world):
    """the model's shards are disjoint, ordered and cover every vector; FusedOptimizer.shard_bounds says the same"""
    from distributed_sod_project_b200.optim import FusedOptimizer

    class Flat:
        pass
    for nvec in list(range(1, 40)) + [2048 * world + 1, 123457]:
        bounds = [geo.shard_bounds(r, nvec, world) for r in range(world)]
        assert bounds[0][0] == 0 and bounds[-1][1] == nvec
        assert all(a[1] == b[0] for a, b in zip(bounds, bounds[1:]))
        opt = object.__new__(FusedOptimizer)
        opt.flat = Flat()
        opt.flat.numel = 4 * nvec
        assert [opt.shard_bounds(r, world) for r in range(world)] == [(4 * lo, 4 * hi) for lo, hi in bounds]


@pytest.mark.parametrize("sm_count", [132, 114, 148, 16])
def test_grids(sm_count):
    cap = min(sm_count, 1024)
    assert geo.comm_grid(0, sm_count) == 1 and geo.comm_grid(1, sm_count) == 1
    assert geo.comm_grid(2048, sm_count) == 1 and geo.comm_grid(2049, sm_count) == 2
    assert geo.comm_grid(10 ** 9, sm_count) == cap
    assert geo.one_shot_cap(sm_count) == 2048 * cap
    assert geo.allreduce_grid(4 * (geo.one_shot_cap(sm_count) + 1), 2, 1, sm_count) is None
    assert geo.allreduce_grid(4 * geo.one_shot_cap(sm_count), 2, 1, sm_count) == cap
    assert geo.auto_algo(65536) == 1 and geo.auto_algo(65540) == 2 and geo.auto_algo(4, has_mc=True) == 2
    assert geo.allreduce_grid(65536, 8, 0, sm_count) == geo.comm_grid(16384, sm_count)
    assert geo.allreduce_grid(65540, 8, 0, sm_count) == geo.comm_grid(geo.shard(16385, 8), sm_count)
    # the one-shot grid grows with the whole buffer: W full grids never fit, so the cap is only reachable as a refusal
    assert not geo.coresident([[geo.allreduce_grid(4 * geo.one_shot_cap(sm_count), 2, 1, sm_count)]] * 2, sm_count)


@pytest.mark.parametrize("sm_count", [132, 114, 148, 20])
@pytest.mark.parametrize("algo", [1, 2])
@pytest.mark.parametrize("world", WORLDS)
def test_selector_returns_the_smallest_coresident_n(world, algo, sm_count):
    reached = set()
    for name in geo.REGIMES:
        n = geo.select(name, world, algo, sm_count)
        if n is None:
            continue
        reached.add(name)
        g = geo.allreduce_grid(n, world, algo, sm_count)
        assert g is not None and geo.coresident([[g]] * world, sm_count), (name, n)
        if name == "max":
            # one more CTA's worth no longer fits
            bigger = n + 4 * geo.VEC_PER_CTA * (1 if algo == 1 else world)
            assert not geo.coresident([[geo.allreduce_grid(bigger, world, algo, sm_count)]] * world, sm_count)
            continue
        assert name in geo.regime(n, world, algo, sm_count)
        assert not any(name in geo.regime(m, world, algo, sm_count) for m in range(4, n, 4)), (name, n)
    # every regime of the issue that the rule admits: an empty shard needs W ≥ 3 (ceil(nvec/2) never leaves rank 1
    # without vectors once nvec > 1)
    want = set(geo.REGIMES) - ({"empty_shard"} if world == 2 else set())
    if sm_count // world < 2:
        want -= {"ragged_block"}
    assert reached == want


def test_table_on_an_h100(capsys):
    """the selected all-reduce sizes on 132 SMs (printed for the record)"""
    rows = []
    for world in WORLDS:
        for algo in (1, 2):
            ns = {name: geo.select(name, world, algo, 132) for name in geo.REGIMES}
            rows.append((world, algo, ns))
            assert ns["max"] == (132 // world) * 2048 * 4 * (1 if algo == 1 else world)
    with capsys.disabled():
        print("\n132 SMs: smallest co-resident n (elements) per all-reduce regime")
        for world, algo, ns in rows:
            print(f"W={world} algo={algo}: " + "  ".join(f"{k}={v}" for k, v in ns.items()))
