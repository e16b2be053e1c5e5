"""ORACLE (test infrastructure only): the launch geometry of the peer-memory collectives, restated from csrc/sgd.cu.

The host side of `sod_allreduce_f32`, `sod_allreduce_sgd` and `sod_allreduce_adam` with the SM count as an argument
instead of a device query, so the tests can say in advance how many CTAs every rank launches:

* `comm_grid`: ⌈vectors / (kThreads·kUnroll)⌉ clamped to [1, min(#SMs, SOD_COMM_MAX_BLOCKS)];
* `shard`: rank r owns float4 vectors [r·⌈nvec/W⌉, min((r+1)·⌈nvec/W⌉, nvec)) in the two-shot and step kernels;
* `one_shot_cap`: the largest nvec the one-shot kernel takes (each thread keeps at most kUnroll vectors in registers);
* `auto_algo`: what algo 0 picks without a multicast mapping (one-shot up to 256 KB, else two-shot);
* `allreduce_grid` / `step_grid`: the grid of one launch, or None where the host refuses it (SOD_EUNSUPPORTED).

W virtual ranks on one GPU can only run side by side if every CTA of every rank is resident at once (the barriers spin
on peers).  At one CTA per SM — the step kernels' 512 threads × ~100 registers leave room for one, and nothing in the
argument needs more — that is `coresident`: Σ over ranks of the largest grid the rank launches ≤ #SMs.

`regime` / `select` classify an all-reduce size and find the smallest n (elements, a multiple of 4) of a regime that
the co-residency rule admits, or the largest for "max".
"""
from __future__ import annotations

K_THREADS = 512
K_UNROLL = 4
SOD_MAX_WORLD = 8
SOD_COMM_MAX_BLOCKS = 1024
SOD_COMM_CHANNELS = 4
CH_STEP, CH_ALLREDUCE = 0, 3              # barrier channels of the step kernels and of the plain all-reduce
BARRIERS_PER_LAUNCH = 2                   # every comm kernel passes comm_block_barrier twice per CTA
ONE_SHOT_AUTO_BYTES = 256 << 10
VEC_PER_CTA = K_THREADS * K_UNROLL

REGIMES = ("n4", "empty_shard", "ragged", "ragged_block", "max")


def grid_cap(sm_count):
    return min(sm_count, SOD_COMM_MAX_BLOCKS)


def comm_grid(vecs_per_rank, sm_count):
    return max(1, min(-(-vecs_per_rank // VEC_PER_CTA), grid_cap(sm_count)))


def shard(nvec, world):
    return -(-nvec // world)


def shard_bounds(rank, nvec, world):
    """[lo, hi) in float4 vectors; empty (lo == hi) when the ceiling division leaves rank `rank` nothing"""
    s = shard(nvec, world)
    return min(rank * s, nvec), min((rank + 1) * s, nvec)


def one_shot_cap(sm_count):
    return VEC_PER_CTA * grid_cap(sm_count)


def auto_algo(n, has_mc=False):
    return 1 if (not has_mc and n * 4 <= ONE_SHOT_AUTO_BYTES) else 2


def allreduce_grid(n, world, algo, sm_count, has_mc=False):
    """CTAs of one sod_allreduce_f32 launch on every rank; None when the host returns SOD_EUNSUPPORTED"""
    nvec = n // 4
    if algo == 0:
        algo = auto_algo(n, has_mc)
    if algo == 1:
        return None if nvec > one_shot_cap(sm_count) else comm_grid(nvec, sm_count)
    return comm_grid(shard(nvec, world), sm_count)


def step_grid(n, world, sm_count):
    """CTAs of one sod_allreduce_sgd / sod_allreduce_adam launch on every rank"""
    return comm_grid(shard(n // 4, world), sm_count)


def coresident(grids_per_rank, sm_count):
    """grids_per_rank[r]: the grids rank r launches (None for launches that never wait on a peer)"""
    return sum(max((g for g in gs if g is not None), default=0) for gs in grids_per_rank) <= sm_count


def regime(n, world, algo, sm_count):
    """the regime classes an all-reduce of n elements belongs to (a size can be in several)"""
    nvec = n // 4
    out = set()
    if nvec == 1:
        out.add("n4")
    if nvec > 1 and any(lo == hi for lo, hi in (shard_bounds(r, nvec, world) for r in range(world))):
        out.add("empty_shard")
    if nvec % world and shard_bounds(world - 1, nvec, world)[1] > shard_bounds(world - 1, nvec, world)[0]:
        out.add("ragged")                 # every rank owns vectors, the last fewer than the others
    per = nvec if algo == 1 else shard(nvec, world)
    if per > VEC_PER_CTA and per % VEC_PER_CTA:
        out.add("ragged_block")           # more than one CTA and the last one only partly filled
    return out


def max_n(world, algo, sm_count):
    """the largest n whose W grids are co-resident"""
    per_rank = sm_count // world
    vecs = per_rank * VEC_PER_CTA
    return (vecs if algo == 1 else vecs * world) * 4


def select(name, world, algo, sm_count):
    """smallest n (largest for "max") of regime `name` whose launch is co-resident; None when unreachable"""
    if name == "max":
        n = max_n(world, algo, sm_count)
        return n if n > 0 and allreduce_grid(n, world, algo, sm_count) * world <= sm_count else None
    top = max_n(world, algo, sm_count)
    for n in range(4, top + 1, 4):
        if name in regime(n, world, algo, sm_count):
            g = allreduce_grid(n, world, algo, sm_count)
            if g is not None and g * world <= sm_count:
                return n
    return None
