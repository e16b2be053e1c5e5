"""The world > 1 collective kernels on ONE GPU: W = 2, 3, 4 and 8 virtual ranks run side by side.

A rank of the peer-memory collectives is nothing but a `sod_comm`: `peer[q]` holds arena q's base address, `block_seq`
and `error_flag` are device pointers, and every wait is bounded by `timeout_cycles`.  So W arenas on one device and W
communicators pointing at them form a world; each virtual rank's calls go to its own stream, and the ranks run
concurrently.  Peer loads and stores (`ld/st.relaxed.sys`, `st.release.sys`) are ordinary global accesses there.

Harness (`VirtualWorld`): per rank a zeroed arena of `sod_comm_flag_bytes() + payload` bytes, a zeroed `block_seq`, an
error word, `timeout_cycles` = 2·10⁹ (about a second: a protocol failure shows up as a set error flag, quickly), and a
stream.  `run` synchronizes the device, enqueues each rank's whole call sequence on its stream (ranks in the order
0..W−1, reversed, or interleaved call by call) without a host sync in between, so the ranks drift apart and reuse
slots and sequence numbers under skew, then synchronizes and requires every return code and every error flag to be 0.

* Co-residency.  The spin-wait kernels only finish if every CTA of every rank is resident at once.  One CTA per SM is
  assumed, which is what the kernels get: the step kernels run 512 threads at ~100 registers, the SyncBN kernels take
  ≈227 KB of shared memory.  Before anything is enqueued the harness asserts Σ over ranks of the largest grid the rank
  launches ≤ #SMs, with the grids taken from the models (oracle/comm_geometry.py, oracle/syncbn_geometry.py).  Stream
  order keeps one kernel per rank in flight; nothing here uses PDL or a cooperative launch.
* Grids.  After a run, every rank's `block_seq` must have advanced by exactly 2 per barrier channel slot for each launch
  whose grid covers that slot, and the SyncBN debug stamps must count the model's strips: a change of `comm_grid` or
  `make_geom` fails here instead of quietly testing something else.
* The first launch of a kernel instance may load it lazily, and loading may wait for the device to go idle, which a
  rank spinning on a peer that is not launched yet never does.  A sequence whose ranks are enqueued one after the other
  is therefore run once interleaved first, every time: the ranks' sequences are aligned call by call, so in that order
  every kernel a spinning one waits for is already enqueued when the next kernel is loaded.  (Skipping that warm-up once
  the SyncBN kernels were loaded let a first `add_` on an int32 tensor load while rank 0 spun: both ranks timed out.)
* The timeout is a safety net: no case aims at it or at the error flag, and no case depends on luck to be co-resident.
  The module is skipped when launches are serialised (CUDA_LAUNCH_BLOCKING=1, a kernel-serialising tool injected).

Oracles.
* `sod_allreduce_f32`: both kernels add in rank order (acc = x₀; acc += x_q), then multiply by `scale`; numpy float32
  does the same, so the check is bit for bit on every rank.
* `sod_allreduce_sgd` / `sod_allreduce_adam`: a difference test against the world-1 kernels (`sod_sgd_momentum`,
  `sod_adam`) run on the rank-order fp32 sum of the ranks' gradients (for SOD_SEG_GRAD16 ranges the bf16 values summed in
  fp32 from 0, as `reduce_vec16` does) with `inv_scale` = fp32(inv_scale)/fp32(W), which is what the host passes.  Both
  call the same `Rule::update` on the same operands, so parameters, the owner's slice of the optimizer state and Adam's
  step words must be equal bit for bit; an fp64 run of oracle/sgd.py / oracle/adam.py makes the check absolute.
* SyncBN: oracle/syncbn.py's formulas over the W per-rank lists in fp64, with the tolerances derived in the docstring of
  test_gpu_syncbn_regimes.py.  World > 1 adds one fp32 merge of W per-rank terms: forward, the rank-order sum of the W
  (mean, M2) pairs (mean = Σ m_q / W, var = Σ (M2_q + n·(m_q − mean)²) / (n·W)); backward, the rank-order sums of Σdy and
  Σdy·(z − mean).  Each adds at most W·2⁻²⁴ ≤ 2⁻²¹ of the summed magnitudes, inside the 1e-5 relative bound of the
  statistics and inside the 2⁻¹⁸ of |terms| the column means already carry, so the world-1 bounds stand with every
  statistic taken over all W·rows rows — with one addition: the merge forms m_q − mean from per-rank means rounded to
  fp32 (2⁻²⁴·|m_q| each), so the variance also carries 2⁻²¹·mean_q(|m_q|·|m_q − mean|) absolute, which dominates where
  a channel's variance is far below its squared mean (a few rows per rank); invstd gets half of it relative to var + eps.
  Saved mean / invstd, running statistics and num_batches_tracked must be
  bit-identical on every rank; dγ, dβ and the folded conv-bias gradient are per-rank local sums.  `exchange_moments`
  assumes every rank contributes the same number of rows (syncbn.cu: "every rank contributes the same number of rows"),
  and so do these cases.

Out of scope here (they stay with the ≥ 2-GPU tests in test_gpu_multi.py and test_gpu_adam_multi.py):
* NVLS multicast: `kMulticast = true`, the SyncBN `use_mc` path and SOD_ALGO_FORCE_MULTIMEM need real peers;
* grid-stride passes past the first: the step kernels reach `i0 += stride·kUnroll` only when a rank's grid is capped at
  the SM count, and W such grids cannot be co-resident on one GPU; the SyncBN "grid" strip class likewise;
* unequal per-rank row counts in SyncBN (see above);
* real multi-process behaviour: the symmetric-memory rendezvous and the `gather_state` / checkpoint collectives.
"""
import ctypes as C
import os
import zlib
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from oracle import adam as oadam
from oracle import comm_geometry as cgeo
from oracle import sgd as osgd
from oracle import syncbn_geometry as bgeo

_SERIAL = os.environ.get("CUDA_LAUNCH_BLOCKING") == "1" or bool(os.environ.get("CUDA_INJECTION64_PATH"))
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(_SERIAL, reason="serialised kernel launches cannot run virtual ranks side by side")]

WORLDS = (2, 3, 4, 8)
ORDERS = ("forward", "reversed", "interleaved")
TIMEOUT_CYCLES = 2_000_000_000
SEQ_WORDS = cgeo.SOD_COMM_CHANNELS * cgeo.SOD_COMM_MAX_BLOCKS
EPS, MOMENTUM = 1e-5, 0.1
STAMP_BYTES = bgeo.K_MAX_GRID * 64
SOD_ECOMM, SOD_EALIGN, SOD_EUNSUPPORTED = -5, -2, -4


def L():
    from distributed_sod_project_b200 import _lib
    return _lib.lib()


def _lib():
    from distributed_sod_project_b200 import _lib as m
    return m


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def smem_optin():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).shared_memory_per_block_optin


def stream_ptr():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# harness
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class Launch:
    fn: object                      # () -> return code (C-ABI call) or None (a torch op on the rank's stream)
    grid: int | None = None         # CTAs of a launch that waits on peers, from the model
    channel: int | None = None      # barrier channel of a comm kernel (its block_seq slots are counted)
    stamps: object = None           # (workspace, offset) of a SyncBN launch with SOD_DEBUG_TIMING


@dataclass
class VirtualWorld:
    world: int
    payload: int
    arenas: list = field(default_factory=list)
    seqs: list = field(default_factory=list)
    errs: list = field(default_factory=list)
    comms: list = field(default_factory=list)
    streams: list = field(default_factory=list)

    def __post_init__(self):
        lib = _lib()
        self.flag_bytes = int(L().sod_comm_flag_bytes())
        self.nbytes = self.flag_bytes + (self.payload + 255) // 256 * 256
        for r in range(self.world):
            self.arenas.append(torch.zeros(self.nbytes, dtype=torch.uint8, device="cuda"))
            self.seqs.append(torch.zeros(SEQ_WORDS, dtype=torch.int32, device="cuda"))
            self.errs.append(torch.zeros(1, dtype=torch.int32, device="cuda"))
            self.streams.append(torch.cuda.Stream())
        for r in range(self.world):
            c = lib.sod_comm()
            c.rank, c.world = r, self.world
            for q in range(lib.SOD_MAX_WORLD):
                c.peer[q] = self.arenas[q].data_ptr() if q < self.world else 0
            c.mc = 0
            c.arena_bytes = self.nbytes
            c.error_flag = self.errs[r].data_ptr()
            c.timeout_cycles = TIMEOUT_CYCLES
            c.block_seq = self.seqs[r].data_ptr()
            self.comms.append(c)
        self._top = self.flag_bytes
        self._tag = 0
        torch.cuda.synchronize()

    def alloc(self, nbytes, align=256):
        off = (self._top + align - 1) // align * align
        assert off + nbytes <= self.nbytes, "arena too small for the case"
        self._top = off + nbytes
        return off

    def view(self, r, off, numel, dtype):
        esz = torch.empty((), dtype=dtype).element_size()
        return self.arenas[r][off:off + numel * esz].view(dtype)

    def ref(self, r):
        return C.byref(self.comms[r])

    def tag(self):
        """host-style SyncBN tag: unique among every call of the world (0 would match a zeroed slot)"""
        self._tag += 1
        return self._tag

    def seed_sequences(self, value):
        """every rank's block_seq and signal area at `value`, as if that many barriers had completed everywhere"""
        v = int(np.array(value, dtype=np.uint32).view(np.int32))
        for r in range(self.world):
            self.seqs[r].fill_(v)
            self.arenas[r][:self.flag_bytes].view(torch.int32).fill_(v)
        torch.cuda.synchronize()

    def _enqueue(self, calls, order):
        W = self.world
        rcs = [[] for _ in range(W)]

        def go(r, k):
            with torch.cuda.stream(self.streams[r]):
                rc = calls[r][k].fn()
            if isinstance(rc, int):         # a C-ABI return code (torch ops return tensors or None)
                rcs[r].append(rc)
        if order == "interleaved":
            for k in range(max(len(c) for c in calls)):
                for r in range(W):
                    if k < len(calls[r]):
                        go(r, k)
        else:
            for r in (range(W) if order == "forward" else reversed(range(W))):
                for k in range(len(calls[r])):
                    go(r, k)
        torch.cuda.synchronize()
        assert all(rc == 0 for rr in rcs for rc in rr), f"return codes per rank: {rcs}"
        errs = [int(e.item()) & 0xFFFFFFFF for e in self.errs]
        assert errs == [0] * W, f"error flags: {[hex(e) for e in errs]}"

    def run(self, make, order="interleaved"):
        """`make()` (re)initialises the case and returns W call lists, aligned call by call across the ranks"""
        if order != "interleaved":
            self._run_once(make(), "interleaved")      # loads every kernel the sequence launches, torch's included
        self._run_once(make(), order)

    def _run_once(self, calls, order):
        W = self.world
        assert len(calls) == W
        grids = [[c.grid for c in calls[r] if c.grid is not None] for r in range(W)]
        assert cgeo.coresident(grids, sm_count()), f"grids {grids} are not co-resident on {sm_count()} SMs"
        torch.cuda.synchronize()
        before = [s.to(torch.int64) & 0xFFFFFFFF for s in self.seqs]
        stamp_areas = {}
        for r in range(W):
            for c in calls[r]:
                if c.stamps is not None:
                    ws, off = c.stamps
                    ws[off:off + STAMP_BYTES].zero_()
                    key = (ws.data_ptr(), off)
                    stamp_areas[key] = (ws, off, max(stamp_areas.get(key, (None, None, 0))[2], c.grid))
        self._enqueue(calls, order)
        for r in range(W):
            want = torch.zeros(SEQ_WORDS, dtype=torch.int64)
            for c in calls[r]:
                if c.channel is not None:
                    base = c.channel * cgeo.SOD_COMM_MAX_BLOCKS
                    want[base:base + c.grid] += cgeo.BARRIERS_PER_LAUNCH
            got = ((self.seqs[r].to(torch.int64) & 0xFFFFFFFF) - before[r]) & 0xFFFFFFFF
            bad = (got.cpu() != want).nonzero().flatten().tolist()
            assert not bad, (f"rank {r}: block_seq advanced {got.cpu()[bad[:4]].tolist()} at slots {bad[:4]}, "
                             f"the model says {want[bad[:4]].tolist()}")
        for ws, off, grid in stamp_areas.values():
            n = int((ws[off:off + STAMP_BYTES].view(torch.int64).view(bgeo.K_MAX_GRID, 8)[:, 0] != 0).sum())
            assert n == grid, f"SyncBN grid {n} != model {grid}"


def rng_for(*parts):
    return np.random.default_rng(zlib.crc32(repr(parts).encode()))


def spread(rng, n, lo=-8, hi=8):
    """fp32 values over several binades, so that the order of a sum shows in its rounding"""
    return (rng.standard_normal(n) * np.exp2(rng.integers(lo, hi, n))).astype(np.float32)


def rank_order_sum(xs):
    acc = xs[0].astype(np.float32).copy()
    for x in xs[1:]:
        acc += x.astype(np.float32)
    return acc


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).numpy()


# ---------------------------------------------------------------------------------------------------------------------
# (a) sod_allreduce_f32
# ---------------------------------------------------------------------------------------------------------------------
def allreduce_launch(vw, r, off, n, scale, algo, flags=0):
    world = vw.world
    g = cgeo.allreduce_grid(n, world, algo, sm_count())
    return Launch(lambda: L().sod_allreduce_f32(vw.ref(r), off, n, scale, algo, flags, stream_ptr()), grid=g,
                  channel=cgeo.CH_ALLREDUCE)


def check_allreduce(vw, off, n, xs, scale):
    want = rank_order_sum(xs) * np.float32(scale)
    for r in range(vw.world):
        got = vw.view(r, off, n, torch.float32)
        assert np.array_equal(bits(got), want.view(np.int32)), \
            f"rank {r}: {int((bits(got) != want.view(np.int32)).sum())} of {n} elements differ from the rank-order sum"


AR_CASES = [(w, a, reg) for w in WORLDS for a in (1, 2) for reg in cgeo.REGIMES if not (w == 2 and reg == "empty_shard")]


@pytest.mark.parametrize("world,algo,regime", AR_CASES, ids=[f"W{w}-algo{a}-{r}" for w, a, r in AR_CASES])
def test_allreduce_f32_is_the_rank_order_sum(world, algo, regime):
    n = cgeo.select(regime, world, algo, sm_count())
    assert n is not None
    vw = VirtualWorld(world, 4 * n)
    off = vw.alloc(4 * n)
    scale = float(np.float32(1.0 / world))
    xs = [spread(rng_for("ar", world, algo, n, r), n) for r in range(world)]

    def make():
        for r in range(world):
            vw.view(r, off, n, torch.float32).copy_(torch.from_numpy(xs[r]))
        return [[allreduce_launch(vw, r, off, n, scale, algo)] for r in range(world)]
    vw.run(make, ORDERS[(world + algo) % 3])
    check_allreduce(vw, off, n, xs, scale)


@pytest.mark.parametrize("world", WORLDS)
def test_allreduce_f32_auto_picks_one_shot_up_to_256_kb_without_multicast(world):
    """algo 0 with mc == 0: one-shot up to 256 KB, two-shot above; the grids (block_seq slots) tell which ran"""
    sizes = (65536, 65540)
    assert [cgeo.auto_algo(n) for n in sizes] == [1, 2]
    vw = VirtualWorld(world, 4 * sum(sizes) + 512)
    offs = [vw.alloc(4 * n) for n in sizes]
    xs = [[spread(rng_for("auto", world, n, r), n) for r in range(world)] for n in sizes]

    def make():
        for i, n in enumerate(sizes):
            for r in range(world):
                vw.view(r, offs[i], n, torch.float32).copy_(torch.from_numpy(xs[i][r]))
        return [[allreduce_launch(vw, r, offs[i], n, 0.5, 0) for i, n in enumerate(sizes)] for r in range(world)]
    assert [cgeo.allreduce_grid(n, world, 0, sm_count()) for n in sizes] != \
           [cgeo.allreduce_grid(n, world, a, sm_count()) for n, a in zip(sizes, (2, 1))]
    vw.run(make, "interleaved")
    for i, n in enumerate(sizes):
        check_allreduce(vw, offs[i], n, xs[i], 0.5)


# ---------------------------------------------------------------------------------------------------------------------
# (b) the fused reduce-scatter + optimizer step + all-gather
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class StepCase:
    id: str
    world: int
    rule: str                 # "sgd", "nesterov", "adam"
    segs: str                 # "inside": boundaries inside shards, a frozen segment = one whole shard; "gap16": a gap, 16 segments
    wire16: bool = True       # grad16 passed (SOD_SEG_GRAD16 ranges next to fp32 ranges); False: grad16_off = 0
    lr_dev: bool = True
    zero_grad: bool = True
    shadow: bool = True
    skip_step: int = -1       # index of the step that runs with *found_inf != 0
    steps: int = 3
    order: str = "interleaved"


def _step_cases():
    out = []
    for i, w in enumerate(WORLDS):
        for j, rule in enumerate(("sgd", "nesterov", "adam")):
            k = i + j
            out.append(StepCase(f"W{w}-{rule}-inside", w, rule, "inside", order=ORDERS[k % 3]))
            out.append(StepCase(f"W{w}-{rule}-gap16-nolr-nozero", w, rule, "gap16", wire16=k % 2 == 0, lr_dev=False,
                                zero_grad=False, shadow=k % 2 == 1, order=ORDERS[(k + 1) % 3]))
            out.append(StepCase(f"W{w}-{rule}-found-inf", w, rule, "inside" if k % 2 else "gap16", skip_step=1,
                                wire16=k % 2 == 1, order=ORDERS[(k + 2) % 3]))
        out.append(StepCase(f"W{w}-sgd-fp32-wire", w, "sgd", "inside", wire16=False, steps=2))
        out.append(StepCase(f"W{w}-adam-all-skipped", w, "adam", "inside", skip_step=0, steps=1))
    return out


STEP_CASES = _step_cases()


def seg_table(case, nvec, world, rng):
    """[(begin, end, flags, k)] in elements; k indexes the hyper-parameters"""
    lib = _lib()
    G16 = lib.SOD_SEG_GRAD16
    if case.segs == "inside":
        lo1, hi1 = cgeo.shard_bounds(1, nvec, world)
        cuts = [0, lo1 - 5, lo1, hi1, min(hi1 + 37, nvec), nvec]
        flags = [0, G16, lib.SOD_SEG_FROZEN, G16, 0]
    else:
        cuts = sorted(set([0, nvec] + [int(c) for c in rng.choice(np.arange(1, nvec), 16, replace=False)]))
        assert len(cuts) == 18                         # 17 pieces: 16 segments and one gap
        flags = [(G16 if i % 3 == 1 else 0) | (lib.SOD_SEG_FROZEN if i == 5 else 0) for i in range(17)]
    out = []
    gap = -1 if case.segs == "inside" else 9
    for i in range(len(cuts) - 1):
        if i == gap or cuts[i] == cuts[i + 1]:
            continue
        f = flags[i]
        if case.rule == "nesterov" and i % 2 == 0:
            f |= lib.SOD_SEG_NESTEROV
        out.append((4 * cuts[i], 4 * cuts[i + 1], f, i))
    assert len(out) <= lib.SOD_MAX_SEGMENTS
    return out


def hyper(rule, k):
    lrs = (0.05, 0.01, 0.2, 0.003)
    if rule == "adam":
        betas = ((0.9, 0.999), (0.8, 0.99), (0.95, 0.9999), (0.5, 0.9))
        return dict(lr=lrs[k % 4] * 0.1, wd=(5e-4, 0.0, 1e-2)[k % 3], b1=betas[k % 4][0], b2=betas[k % 4][1],
                    eps=(1e-8, 1e-6)[k % 2])
    return dict(lr=lrs[k % 4], wd=(5e-4, 0.0, 1e-2)[k % 3], mu=(0.9, 0.0, 0.5)[k % 3])


def make_segs(rule, table, lr_scale=1.0):
    lib = _lib()
    if rule == "adam":
        arr = (lib.sod_adam_segment * len(table))()
        for i, (b, e, f, k) in enumerate(table):
            h = hyper(rule, k)
            arr[i] = lib.sod_adam_segment(b, e, h["lr"] * lr_scale, h["wd"], h["b1"], h["b2"], h["eps"], f)
    else:
        arr = (lib.sod_sgd_segment * len(table))()
        for i, (b, e, f, k) in enumerate(table):
            h = hyper(rule, k)
            arr[i] = lib.sod_sgd_segment(b, e, h["lr"] * lr_scale, h["wd"], h["mu"], f)
    return arr


def step_size_of(case):
    """vectors per rank a little over two CTAs' worth, ragged across ranks"""
    return case.world * 2 * cgeo.VEC_PER_CTA + 3 * case.world + 1


@pytest.mark.parametrize("case", STEP_CASES, ids=[c.id for c in STEP_CASES])
def test_allreduce_step_equals_the_world1_step(case):
    lib = _lib()
    W, K = case.world, case.steps
    nvec = step_size_of(case)
    n = 4 * nvec
    rng = rng_for("step", case.id)
    table = seg_table(case, nvec, W, rng)
    nseg = len(table)
    segs = make_segs(case.rule, table)
    adam = case.rule == "adam"
    G16 = lib.SOD_SEG_GRAD16
    in16 = np.zeros(n, bool)
    upd = np.zeros(n, bool)
    for b, e, f, _ in table:
        in16[b:e] = case.wire16 and bool(f & G16)
        upd[b:e] = not (f & lib.SOD_SEG_FROZEN)
    # inputs: identical parameters and step counts everywhere, per-rank gradients and a fresh set per step
    p0 = spread(rng, n, -3, 3)
    st0 = [spread(rng, n, -4, 0)] + ([np.abs(spread(rng, n, -12, -4))] if adam else [])
    step0 = np.zeros(lib.SOD_ADAM_STEP_WORDS, np.int32)
    step0[:nseg] = rng.integers(0, 6, nseg)
    g32 = [[spread(rng, n, -6, 2) for _ in range(W)] for _ in range(K)]
    g16 = [[torch.from_numpy(spread(rng, n, -6, 2)).to(torch.bfloat16) for _ in range(W)] for _ in range(K)]
    shadow0 = torch.full((n,), 0x7F7F, dtype=torch.int16).view(torch.bfloat16)
    inv_scale = float(np.float32(3.0 / 1024))
    lr_vals = np.array([hyper(case.rule, k)["lr"] * 0.5 for *_, k in table], np.float32)
    lr_dev = torch.from_numpy(lr_vals).cuda() if case.lr_dev else None
    finf = [torch.tensor([1 if k == case.skip_step else 0], dtype=torch.int32, device="cuda") for k in range(K)]
    flags = (lib.SOD_SGD_ZERO_GRAD if case.zero_grad else 0) | lib.SOD_ALGO_NO_MULTIMEM

    vw = VirtualWorld(W, 4 * n * 2 + 2 * n + 1024)
    p_off, g_off, h_off = vw.alloc(4 * n), vw.alloc(4 * n), vw.alloc(2 * n)
    state = {}
    grid = cgeo.step_grid(n, W, sm_count())
    g32_dev = [[torch.from_numpy(g).cuda() for g in gk] for gk in g32]
    g16_dev = [[g.cuda() for g in gk] for gk in g16]

    def make():
        st = [[torch.from_numpy(s).cuda() for s in st0] for _ in range(W)]
        steps = [torch.from_numpy(step0).cuda() for _ in range(W)]
        shadows = [shadow0.cuda() for _ in range(W)] if case.shadow else [None] * W
        state.update(st=st, steps=steps, shadows=shadows)
        calls = []
        for r in range(W):
            vw.view(r, p_off, n, torch.float32).copy_(torch.from_numpy(p0))
            seq = []
            for k in range(K):
                def fill(r=r, k=k):
                    vw.view(r, g_off, n, torch.float32).copy_(g32_dev[k][r])
                    vw.view(r, h_off, n, torch.bfloat16).copy_(g16_dev[k][r])
                seq.append(Launch(fill))
                sh = shadows[r].data_ptr() if case.shadow else None
                h = h_off if case.wire16 else 0
                lrp = lr_dev.data_ptr() if lr_dev is not None else None
                if adam:
                    fn = (lambda r=r, k=k, sh=sh, h=h, lrp=lrp: L().sod_allreduce_adam(
                        vw.ref(r), g_off, h, p_off, st[r][0].data_ptr(), st[r][1].data_ptr(), sh, n, segs, nseg, lrp,
                        steps[r].data_ptr(), inv_scale, finf[k].data_ptr(), flags, stream_ptr()))
                else:
                    fn = (lambda r=r, k=k, sh=sh, h=h, lrp=lrp: L().sod_allreduce_sgd(
                        vw.ref(r), g_off, h, p_off, st[r][0].data_ptr(), sh, n, segs, nseg, lrp, inv_scale,
                        finf[k].data_ptr(), flags, stream_ptr()))
                seq.append(Launch(fn, grid=grid, channel=cgeo.CH_STEP))
            calls.append(seq)
        return calls
    vw.run(make, case.order)

    # ---- world-1 reference: the same rule on the reduced gradient ----------------------------------------------------
    scale1 = float(np.float32(inv_scale) / np.float32(W))
    p1 = torch.from_numpy(p0).cuda()
    st1 = [torch.from_numpy(s).cuda() for s in st0]
    steps1 = torch.from_numpy(step0).cuda()
    sh1 = shadow0.cuda()
    p64, st64, steps64 = p0.astype(np.float64), [s.astype(np.float64) for s in st0], list(step0[:nseg])
    o_segs = []
    for i, (b, e, f, k) in enumerate(table):
        h = hyper(case.rule, k)
        lr = float(lr_vals[i]) if case.lr_dev else float(np.float32(h["lr"]))
        fz = bool(f & lib.SOD_SEG_FROZEN)
        if adam:
            o_segs.append(oadam.Segment(b, e, lr, float(np.float32(h["wd"])), h["b1"], h["b2"], float(np.float32(h["eps"])), fz))
        else:
            o_segs.append(osgd.Segment(b, e, lr, float(np.float32(h["wd"])), float(np.float32(h["mu"])), fz,
                                       bool(f & lib.SOD_SEG_NESTEROV)))
    for k in range(K):
        gsum = rank_order_sum(g32[k])
        if case.wire16:
            b16 = np.zeros(n, np.float32)
            for r in range(W):
                b16 += g16[k][r].float().numpy()
            gsum = np.where(in16, b16, gsum)
        g1 = torch.from_numpy(gsum).cuda()
        lrp = lr_dev.data_ptr() if lr_dev is not None else None
        if adam:
            rc = L().sod_adam(p1.data_ptr(), st1[0].data_ptr(), st1[1].data_ptr(), g1.data_ptr(), None, sh1.data_ptr(), n, segs,
                              nseg, lrp, steps1.data_ptr(), scale1, finf[k].data_ptr(), 0, stream_ptr())
        else:
            rc = L().sod_sgd_momentum(p1.data_ptr(), st1[0].data_ptr(), g1.data_ptr(), None, sh1.data_ptr(), n, segs, nseg,
                                      lrp, scale1, finf[k].data_ptr(), 0, stream_ptr())
        assert rc == 0
        if k != case.skip_step:
            if adam:
                p64, m64, v64, steps64 = oadam.adam_step_f64(p64, st64[0], st64[1], gsum, o_segs, steps64, scale1)
                st64 = [m64, v64]
            else:
                p64, v64 = osgd.sgd_step_f64(p64, st64[0], gsum, o_segs, scale1)
                st64 = [v64]
    torch.cuda.synchronize()

    p_want = bits(p1)
    for r in range(W):
        p = vw.view(r, p_off, n, torch.float32)
        assert np.array_equal(bits(p), p_want), f"rank {r}: parameters differ from the world-1 step"
        lo, hi = (4 * x for x in cgeo.shard_bounds(r, nvec, W))
        for i, (got, want, init) in enumerate(zip(state["st"][r], st1, st0)):
            g = got.cpu().numpy()
            assert np.array_equal(g[lo:hi].view(np.int32), bits(want)[lo:hi]), f"rank {r}: state {i} of the shard"
            outside = np.ones(n, bool)
            outside[lo:hi] = False
            assert np.array_equal(g[outside].view(np.int32), init[outside].view(np.int32)), f"rank {r}: state {i} off-shard"
        if adam:
            assert state["steps"][r].tolist() == steps1.tolist(), f"rank {r}: Adam step words"
            # and, independently of the world-1 kernel (which shares the epilogue): one count per step that was not
            # skipped, for every segment that is not frozen; the ticket word re-armed
            taken = sum(k != case.skip_step for k in range(K))
            want_steps = [int(step0[i]) + (0 if table[i][2] & lib.SOD_SEG_FROZEN else taken) for i in range(nseg)]
            assert state["steps"][r].tolist()[:nseg] == want_steps, f"rank {r}: Adam step counts"
            assert state["steps"][r][lib.SOD_MAX_SEGMENTS].item() == 0
        # gradients: cleared everywhere with SOD_SGD_ZERO_GRAD (also on a skipped step), except the fp32 buffer of
        # SOD_SEG_GRAD16 ranges, which those ranges neither read nor clear
        g = vw.view(r, g_off, n, torch.float32).cpu().numpy()
        h = vw.view(r, h_off, n, torch.bfloat16).float().cpu().numpy()
        last32, last16 = g32[K - 1][r], g16[K - 1][r].float().numpy()
        if case.zero_grad:
            assert np.array_equal(g[in16], last32[in16]), f"rank {r}: fp32 gradients of GRAD16 ranges must be untouched"
            assert not g[~in16].any(), f"rank {r}: fp32 gradients not cleared"
            if case.wire16:
                assert not h.any(), f"rank {r}: bf16 gradients not cleared"
            else:
                assert np.array_equal(h, last16), f"rank {r}: grad16 without grad16_off is not the kernel's"
        else:
            assert np.array_equal(g, last32) and np.array_equal(h, last16), f"rank {r}: gradients changed"
        if case.shadow:
            # world > 1 refreshes the whole shadow from the all-gathered parameters, frozen ranges and gaps included
            sh = state["shadows"][r]
            stepped = any(k != case.skip_step for k in range(K))
            want = p.to(torch.bfloat16) if stepped else shadow0.cuda()
            assert torch.equal(sh.view(torch.int16), want.view(torch.int16)), f"rank {r}: shadow"
    # world 1 refreshes the shadow of updated elements only
    stepped = any(k != case.skip_step for k in range(K))
    s1 = sh1.view(torch.int16).cpu().numpy()
    want_upd = p1.to(torch.bfloat16).view(torch.int16).cpu().numpy() if stepped else shadow0.view(torch.int16).numpy()
    assert np.array_equal(s1[upd], want_upd[upd])
    assert np.array_equal(s1[~upd], shadow0.view(torch.int16).numpy()[~upd])
    # fp64: the world-1 result, and so every rank's, is the exact step up to fp32 rounding
    pg = p1.double().cpu().numpy()
    tol = 1e-5 * (np.abs(p64) + np.abs(p64 - p0)) + 1e-30
    assert bool((np.abs(pg - p64) <= tol).all()), f"fp64 oracle: worst {float((np.abs(pg - p64) / tol).max()):.3g}x"


def test_world1_adds_grad16_outside_grad16_ranges_and_world2_does_not():
    """pinned: with grad16 passed, a range without SOD_SEG_GRAD16 adds the bf16 gradient to the fp32 one at world 1
    (the per-tensor "cast" of amp), and ignores it at world > 1 — the host folds it in first with sod_grad_merge_bf16
    whenever a range can hold both (optim.py step())"""
    lib = _lib()
    n = 4096
    rng = rng_for("pin16")
    p0, g = spread(rng, n, -3, 3), spread(rng, n, -6, 2)
    h = torch.from_numpy(spread(rng, n, -6, 2)).to(torch.bfloat16)
    segs = (lib.sod_sgd_segment * 1)(lib.sod_sgd_segment(0, n, 0.1, 0.0, 0.0, 0))
    outs = {}
    for name, g1, h1 in (("sum", g + h.float().numpy(), None), ("grad16", g, h), ("fp32", g, None)):
        p, v = torch.from_numpy(p0).cuda(), torch.zeros(n, device="cuda")
        gg, hh = torch.from_numpy(g1).cuda(), (h1.cuda() if h1 is not None else None)
        rc = L().sod_sgd_momentum(p.data_ptr(), v.data_ptr(), gg.data_ptr(), hh.data_ptr() if hh is not None else None, None, n,
                                  segs, 1, None, 1.0, None, 0, stream_ptr())
        assert rc == 0
        outs[name] = p
    torch.cuda.synchronize()
    assert torch.equal(outs["sum"], outs["grad16"]) and not torch.equal(outs["fp32"], outs["grad16"])
    # world 2: the same bf16 values on the wire are not read for the fp32 range
    vw = VirtualWorld(2, 4 * n * 2 + 2 * n + 1024)
    p_off, g_off, h_off = vw.alloc(4 * n), vw.alloc(4 * n), vw.alloc(2 * n)
    moms = [torch.zeros(n, device="cuda") for _ in range(2)]

    def make():
        for r in range(2):
            vw.view(r, p_off, n, torch.float32).copy_(torch.from_numpy(p0))
            vw.view(r, g_off, n, torch.float32).copy_(torch.from_numpy(g))
            vw.view(r, h_off, n, torch.bfloat16).copy_(h)
        return [[Launch(lambda r=r: L().sod_allreduce_sgd(vw.ref(r), g_off, h_off, p_off, moms[r].data_ptr(), None, n, segs, 1,
                                                          None, 1.0, None, lib.SOD_ALGO_NO_MULTIMEM, stream_ptr()),
                        grid=cgeo.step_grid(n, 2, sm_count()), channel=cgeo.CH_STEP)] for r in range(2)]
    vw.run(make)
    for r in range(2):       # (g + g)·0.5 = g exactly: the world-1 step on the fp32 gradient alone
        assert torch.equal(vw.view(r, p_off, n, torch.float32), outs["fp32"]), f"rank {r} read grad16 of an fp32 range"



# ---------------------------------------------------------------------------------------------------------------------
# (d) protocol sequences on one set of arenas
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", WORLDS)
def test_mixed_sequence_across_the_sequence_wrap_in_every_launch_order(world):
    """all-reduces (channel 3) and SGD steps (channel 0) alternate with grids changing from launch to launch, so
    blocks sit out launches; before every run (the warm-up included) every rank's block_seq and signal area are set to
    0xFFFFFFF8, so the signed-difference wait of comm_block_barrier crosses 2³² in each of the three launch orders.
    Every all-reduce is the rank-order sum, the parameters equal the world-1 steps on the summed gradients, and the bytes
    do not depend on the order.  (Momentum 0: the shards move with n from launch to launch, so a rank's momentum buffer
    only holds what that rank owned last time; with μ = 0 the update does not read it.)"""
    lib = _lib()
    sm = sm_count()
    per_rank = sm // world
    grids = [g for g in (1, 3, 2, per_rank, 1, 2) if g <= per_rank]
    sizes = [4 * (world * (g - 1) * cgeo.VEC_PER_CTA + 5 * world) for g in grids]
    assert [cgeo.step_grid(n, world, sm) for n in sizes] == grids
    nmax = max(sizes)
    vw = VirtualWorld(world, 2 * 4 * nmax + 4 * sum(sizes) + 256 * len(sizes) + 4096)
    p_off, g_off = vw.alloc(4 * nmax), vw.alloc(4 * nmax)
    a_offs = [vw.alloc(4 * n) for n in sizes]
    rng = rng_for("seq", world)
    xs = [[spread(rng, n) for _ in range(world)] for n in sizes]
    gs = [[spread(rng, n, -6, 0) for _ in range(world)] for n in sizes]
    p0 = spread(rng, nmax, -3, 3)
    moms = [torch.zeros(nmax, device="cuda") for _ in range(world)]
    xs_dev = [[torch.from_numpy(x).cuda() for x in xk] for xk in xs]
    gs_dev = [[torch.from_numpy(x).cuda() for x in gk] for gk in gs]
    segs = [(lib.sod_sgd_segment * 1)(lib.sod_sgd_segment(0, n, 0.05, 1e-3, 0.0, 0)) for n in sizes]

    def make():
        vw.seed_sequences(0xFFFFFFF8)      # block 0 of both channels passes 12 barriers per run
        calls = []
        for r in range(world):
            moms[r].zero_()
            vw.view(r, p_off, nmax, torch.float32).copy_(torch.from_numpy(p0))
            seq = []
            for i, n in enumerate(sizes):
                def fill(r=r, i=i, n=n):
                    vw.view(r, a_offs[i], n, torch.float32).copy_(xs_dev[i][r])
                    vw.view(r, g_off, n, torch.float32).copy_(gs_dev[i][r])
                seq.append(Launch(fill))
                seq.append(allreduce_launch(vw, r, a_offs[i], n, 1.0, 2))
                seq.append(Launch(lambda r=r, i=i, n=n: L().sod_allreduce_sgd(
                    vw.ref(r), g_off, 0, p_off, moms[r].data_ptr(), None, n, segs[i], 1, None, 1.0, None,
                    lib.SOD_SGD_ZERO_GRAD | lib.SOD_ALGO_NO_MULTIMEM, stream_ptr()), grid=grids[i], channel=cgeo.CH_STEP))
            calls.append(seq)
        return calls
    # world-1 reference: the same steps on the rank-order sums, inv_scale = fp32(1)/fp32(W)
    p1, v1 = torch.from_numpy(p0).cuda(), torch.zeros(nmax, device="cuda")
    for i, n in enumerate(sizes):
        g1 = torch.from_numpy(rank_order_sum(gs[i])).cuda()
        assert L().sod_sgd_momentum(p1.data_ptr(), v1.data_ptr(), g1.data_ptr(), None, None, n, segs[i], 1, None,
                                    float(np.float32(1.0) / np.float32(world)), None, 0, stream_ptr()) == 0
    torch.cuda.synchronize()
    for order in ORDERS:
        vw.run(make, order)
        for ch in (cgeo.CH_STEP, cgeo.CH_ALLREDUCE):
            wrapped = [int(s[ch * cgeo.SOD_COMM_MAX_BLOCKS].item()) & 0xFFFFFFFF for s in vw.seqs]
            assert all(w < 0xFFFFFFF8 for w in wrapped), f"{order}: block 0 of channel {ch} did not cross 2^32"
        for i, n in enumerate(sizes):
            check_allreduce(vw, a_offs[i], n, xs[i], 1.0)
        for r in range(world):
            assert torch.equal(vw.view(r, p_off, nmax, torch.float32), p1), f"{order}: rank {r} parameters"


# ---------------------------------------------------------------------------------------------------------------------
# (e) argument contract: refused before any launch
# ---------------------------------------------------------------------------------------------------------------------
def test_comm_argument_contract_returns_before_any_launch():
    lib = _lib()
    n = 64
    vw = VirtualWorld(2, 65536)
    fb = vw.flag_bytes
    off = vw.alloc(4 * n)
    mom = torch.zeros(n, device="cuda")
    m2 = torch.zeros(n, device="cuda")
    steps = torch.zeros(lib.SOD_ADAM_STEP_WORDS, dtype=torch.int32, device="cuda")
    sgd_segs = (lib.sod_sgd_segment * 1)(lib.sod_sgd_segment(0, n, 0.1, 0.0, 0.9, 0))
    adam_segs = (lib.sod_adam_segment * 1)(lib.sod_adam_segment(0, n, 0.1, 0.0, 0.9, 0.999, 1e-8, 0))
    C_ = 64
    ws_bytes = int(L().sod_syncbn_workspace_bytes(1, C_))
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device="cuda")
    x = torch.zeros(16 * C_, device="cuda")
    y = torch.zeros_like(x)
    vec = [torch.zeros(C_, device="cuda") for _ in range(6)]
    ex = int(L().sod_syncbn_exchange_bytes(C_))
    nbt = torch.zeros(1, dtype=torch.int64, device="cuda")

    def comm(**kw):
        c = lib.sod_comm()
        C.memmove(C.byref(c), C.byref(vw.comms[0]), C.sizeof(c))
        for k, v in kw.items():
            if k == "peer1":
                c.peer[1] = v
            else:
                setattr(c, k, v)
        return C.byref(c)

    def ar(c, o=off, nn=n, algo=2):
        return L().sod_allreduce_f32(c, o, nn, 1.0, algo, 0, stream_ptr())

    def sgd(c, g=off, h=0, p=off):
        return L().sod_allreduce_sgd(c, g, h, p, mom.data_ptr(), None, n, sgd_segs, 1, None, 1.0, None, 0, stream_ptr())

    def adam(c, g=off, h=0, p=off):
        return L().sod_allreduce_adam(c, g, h, p, mom.data_ptr(), m2.data_ptr(), None, n, adam_segs, 1, None, steps.data_ptr(),
                                      1.0, None, 0, stream_ptr())

    def bnf(c, so=fb):
        return L().sod_syncbn_fwd(x.data_ptr(), None, None, y.data_ptr(), lib.SOD_F32, vec[0].data_ptr(), vec[1].data_ptr(),
                                  vec[2].data_ptr(), vec[3].data_ptr(), vec[4].data_ptr(), vec[5].data_ptr(), 16, C_, 0.1, 1e-5,
                                  0, 1, c, so, 1, None, nbt.data_ptr(), None, None, 0, ws.data_ptr(), ws_bytes, 0, stream_ptr())

    def bnb(c, so=fb):
        return L().sod_syncbn_bwd(x.data_ptr(), x.data_ptr(), None, None, y.data_ptr(), None, lib.SOD_F32, vec[0].data_ptr(),
                                  None, vec[4].data_ptr(), vec[5].data_ptr(), vec[2].data_ptr(), vec[3].data_ptr(), 16, C_, 0,
                                  c, so, 1, None, None, None, None, None, 0, ws.data_ptr(), ws_bytes, 0, stream_ptr())
    entries = (ar, sgd, adam, bnf, bnb)
    bad_comms = dict(world_9=comm(world=9), rank_eq_world=comm(rank=2), null_peer=comm(peer1=0),
                     unaligned_peer=comm(peer1=vw.arenas[1].data_ptr() + 8), null_block_seq=comm(block_seq=None))
    torch.cuda.synchronize()
    for name, c in bad_comms.items():
        for fn in entries:
            assert fn(c) == SOD_ECOMM, (name, fn.__name__)
    good = vw.ref(0)
    end = vw.nbytes
    for fn in (sgd, adam):
        for kw in (dict(g=fb - 16), dict(p=fb - 16), dict(h=fb - 16), dict(g=end - 4 * n + 16), dict(p=end - 4 * n + 16),
                   dict(h=end - 2 * n + 16)):
            assert fn(good, **kw) == SOD_ECOMM, (fn.__name__, kw)
        for kw in (dict(g=off + 8), dict(p=off + 8), dict(h=off + 8)):
            assert fn(good, **kw) == SOD_EALIGN, (fn.__name__, kw)
    for o in (fb - 16, end - 4 * n + 16):
        assert ar(good, o=o) == SOD_ECOMM
    assert ar(good, o=off + 8) == SOD_EALIGN
    for fn in (bnf, bnb):
        assert fn(good, so=fb - 16) == SOD_ECOMM and fn(good, so=end - ex + 16) == SOD_ECOMM
        assert fn(good, so=fb + 8) == SOD_EALIGN
    # one-shot above its cap: refused, whatever the arena holds
    cap = cgeo.one_shot_cap(sm_count())
    big = VirtualWorld(2, 4 * 4 * (cap + 1))
    boff = big.alloc(4 * 4 * (cap + 1))
    assert L().sod_allreduce_f32(big.ref(0), boff, 4 * (cap + 1), 1.0, 1, 0, stream_ptr()) == SOD_EUNSUPPORTED
    torch.cuda.synchronize()
    for w in (vw, big):
        assert all(int(s.abs().sum()) == 0 for s in w.seqs), "a refused call launched a kernel"
        assert all(int(e.item()) == 0 for e in w.errs)
    assert int(nbt.item()) == 0 and not bool(y.any())


# ---------------------------------------------------------------------------------------------------------------------
# (c) SyncBN at world > 1
# ---------------------------------------------------------------------------------------------------------------------
TORCH_DT = {"float32": torch.float32, "bfloat16": torch.bfloat16, "float16": torch.float16}
BN_C = (8, 64, 2048, 256, 16, 1024)


@dataclass(frozen=True)
class BnCase:
    id: str
    world: int
    kind: str
    dtype: str
    pre: bool
    res: bool
    relu: bool
    C: int
    strips: str
    xmask: bool = False
    nbias: int = 0
    n: str | None = None      # chunks per strip against the stage count (oracle/syncbn_geometry.py classify), if targeted


def _bn_cases():
    out = []
    i = 0
    for w in WORLDS:
        for dt in TORCH_DT:
            for site in bgeo.FWD_SITES:
                C_, st = BN_C[i % len(BN_C)], ("1", "few")[i % 2]
                relu = i % 2 == 0
                out.append(BnCase(f"W{w}-fwd-{dt}-pre{int(site['pre'])}res{int(site['res'])}-C{C_}-{st}", w, "fwd", dt,
                                  site["pre"], site["res"], relu, C_, st, nbias=i % 3))
                i += 1
            for fold in (False, True):
                for xmask in (False, True):
                    C_, st = BN_C[i % len(BN_C)], ("few", "1")[i % 2]
                    site = bgeo.BWD_SITES_XMASK[i % 2] if xmask else bgeo.BWD_SITES[i % 4]
                    out.append(BnCase(f"W{w}-bwd-{dt}-f{int(fold)}x{int(xmask)}-pre{int(site['pre'])}relu{int(site['relu'])}"
                                      f"res{int(site['res'])}-C{C_}-{st}", w, "bwd", dt, site["pre"], site["res"], site["relu"],
                                      C_, st, xmask=xmask, nbias=(1 + i % 2) if fold else 0))
                    i += 1
        # the ring regimes past one chunk per strip: a strip of NS+1 chunks (the ring wraps once), and of 2NS+1
        # (with few strips the traffic cap keeps row counts small, so these need wide layers)
        out.append(BnCase(f"W{w}-fwd-bfloat16-pre0res1-C2048-few-NS+1", w, "fwd", "bfloat16", False, True, True, 2048, "few",
                          nbias=1, n="NS+1"))
        out.append(BnCase(f"W{w}-bwd-float16-f1x0-pre1relu1res1-C512-few-NS+1", w, "bwd", "float16", True, True, True, 512,
                          "few", nbias=2, n="NS+1"))
        out.append(BnCase(f"W{w}-bwd-float32-f0x1-pre0relu1res0-C2048-few-2NS+1", w, "bwd", "float32", False, False, True,
                          2048, "few", xmask=True, n="2NS+1"))
    return out


BN_CASES = _bn_cases()


def bn_geoms(case, rows=None):
    """(rows, forward geometry, backward geometry or None) on this device: the target launch's strip class from the
    model's selector"""
    sm, smem = sm_count(), smem_optin()
    es = bgeo.DTYPE_BYTES[case.dtype]
    fs = bgeo.fwd_site(case.pre, case.res)
    xm = case.xmask and case.relu and not case.res
    bs = bgeo.bwd_site(case.pre, case.relu, xm)
    if rows is None:
        target = fs if case.kind == "fwd" else bs
        want = dict(strips=case.strips, C=case.C, **({"n": case.n} if case.n else {}))
        g = bgeo.select(want, es, *target, sm, smem)
        assert g is not None, f"{case.id}: {want} unreachable"
        rows = g.rows

        def same_class(r):
            return bgeo.matches(bgeo.classify(bgeo.make_geom(r, case.C, es, *target, sm, smem), sm), want)
        if case.strips == "1":
            # well inside the one strip (the smallest such geometry has a single row, so no per-rank M2): two thirds of
            # the largest row count that still gives one strip
            top = rows
            while top < 1 << 14 and same_class(top + 1):
                top += 1
            rows = max(2, 2 * top // 3)
        elif case.n is None:
            # a third strip, half filled: the last strip shorter than the others and its last chunk partial
            more = g.rows + g.chunk_rows * g.chunks_per_strip + g.chunk_rows // 2 + 1
            if same_class(more):
                rows = more
    gf = bgeo.make_geom(rows, case.C, es, *fs, sm, smem)
    gb = bgeo.make_geom(rows, case.C, es, *bs, sm, smem) if case.kind == "bwd" else None
    tgt = gf if case.kind == "fwd" else gb
    cls = bgeo.classify(tgt, sm)
    assert cls["strips"] == case.strips and (case.n is None or cls["n"] == case.n), (case.id, tgt)
    return rows, gf, gb


class BnRank:
    """one virtual rank's SyncBN state: inputs, parameters, outputs and two workspaces (forward, backward)"""

    def __init__(self, vw, r, case, rows, seed_parts):
        C_, dt = case.C, TORCH_DT[case.dtype]
        gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(seed_parts + (r,)).encode()))
        mk = lambda scale, shift=0.0: (torch.randn(rows, C_, generator=gen, device="cuda") * scale + shift).to(dt)  # noqa: E731
        dscale = 2.0 ** 16 / (rows * C_ * vw.world) if dt == torch.float16 else 1.0
        self.x = mk(1.5, 2.0 + 0.5 * r)                   # rank means apart: the merge of the per-rank moments matters
        self.pre = mk(0.5, -0.25 * r) if case.pre else None
        self.res = mk(1.0) if case.res else None
        self.dy = mk(dscale)
        bdt = torch.float32 if case.nbias == 2 else dt
        self.cbs = [(torch.linspace(-0.5, 0.5, C_, device="cuda") * (i + 1)).to(bdt) for i in range(case.nbias)]
        self.y = torch.empty(rows, C_, dtype=dt, device="cuda")
        self.dz = torch.empty_like(self.y)
        self.dres = torch.empty_like(self.y) if case.res else None
        self.ws_bytes = int(L().sod_syncbn_workspace_bytes(1, C_)) + STAMP_BYTES
        self.stamp_off = int(L().sod_syncbn_workspace_bytes(1, C_))
        self.ws = [torch.zeros(self.ws_bytes, dtype=torch.uint8, device="cuda") for _ in range(2)]
        sign = torch.where(torch.arange(C_, device="cuda") % 3 == 0, -1.0, 1.0)
        self.gamma = torch.linspace(0.5, 1.5, C_, device="cuda") * sign
        self.beta = torch.linspace(-0.3, 0.3, C_, device="cuda")
        self.reset()

    def reset(self):
        C_ = self.gamma.numel()
        self.rm = torch.linspace(-0.5, 0.5, C_, device="cuda")
        self.rv = torch.linspace(0.5, 2.0, C_, device="cuda")
        self.mean = torch.zeros(C_, device="cuda")
        self.invstd = torch.zeros(C_, device="cuda")
        self.nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
        self.dgamma = torch.zeros(C_, device="cuda")
        self.dbeta = torch.zeros(C_, device="cuda")
        self.dcbs = [torch.zeros_like(b) for b in self.cbs]
        self.y.zero_()
        self.dz.zero_()

    def cb(self, i):
        return self.cbs[i].data_ptr() if i < len(self.cbs) else None

    def dcb(self, i):
        return self.dcbs[i].data_ptr() if i < len(self.dcbs) else None


def bn_fwd_launch(vw, r, st, case, rows, gf, slot, tag, epoch=None, ws=0, out=None):
    lib = _lib()
    cbdt = lib.dtype_code(st.cbs[0].dtype) if st.cbs else 0
    mean, invstd, y = (st.mean, st.invstd, st.y) if out is None else out
    flags = lib.SOD_ALGO_NO_MULTIMEM | 4                 # SOD_DEBUG_TIMING: per-CTA start stamps
    return Launch(lambda: L().sod_syncbn_fwd(
        st.x.data_ptr(), st.pre.data_ptr() if st.pre is not None else None, st.res.data_ptr() if st.res is not None else None,
        y.data_ptr(), lib.dtype_code(st.x.dtype), st.gamma.data_ptr(), st.beta.data_ptr(), st.rm.data_ptr(), st.rv.data_ptr(),
        mean.data_ptr(), invstd.data_ptr(), rows, case.C, MOMENTUM, EPS, int(case.relu), 1, vw.ref(r), slot, tag,
        epoch.data_ptr() if epoch is not None else None, st.nbt.data_ptr(), st.cb(0), st.cb(1), cbdt,
        st.ws[ws].data_ptr(), st.ws_bytes, flags, stream_ptr()), grid=gf.strips, stamps=(st.ws[ws], st.stamp_off))


def bn_bwd_launch(vw, r, st, case, rows, gb, slot, tag, epoch=None, ws=1, inp=None, out=None):
    lib = _lib()
    cbdt = lib.dtype_code(st.cbs[0].dtype) if st.cbs else 0
    flags = lib.SOD_ALGO_NO_MULTIMEM | 4
    xm = case.xmask and case.relu and not case.res
    if xm:
        flags |= lib.SOD_BN_BWD_MASK_FROM_X
    mean, invstd, y = (st.mean, st.invstd, st.y) if inp is None else inp
    dz = st.dz if out is None else out
    return Launch(lambda: L().sod_syncbn_bwd(
        st.dy.data_ptr(), st.x.data_ptr(), st.pre.data_ptr() if st.pre is not None else None,
        y.data_ptr() if (case.relu and not xm) else None, dz.data_ptr(), st.dres.data_ptr() if st.dres is not None else None,
        lib.dtype_code(st.x.dtype), st.gamma.data_ptr(), st.beta.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
        st.dgamma.data_ptr(), st.dbeta.data_ptr(), rows, case.C, int(case.relu), vw.ref(r), slot, tag,
        epoch.data_ptr() if epoch is not None else None, st.cb(0), st.cb(1), st.dcb(0), st.dcb(1), cbdt,
        st.ws[ws].data_ptr(), st.ws_bytes, flags, stream_ptr()), grid=gb.strips, stamps=(st.ws[ws], st.stamp_off))


def _reg():
    import test_gpu_syncbn_regimes as reg           # the world-1 tolerance helpers (same directory)
    return reg


def check_bn_forward(case, sts, rows, W, y_list=None, stats=None, rm0=None, rv0=None, steps=1):
    """the W ranks' forward against oracle/syncbn.py in fp64; returns (kernel mean, invstd, global mean, var)"""
    reg = _reg()
    dt = TORCH_DT[case.dtype]
    gamma, beta = sts[0].gamma.double(), sts[0].beta.double()
    cb = sum((b.double() for b in sts[0].cbs), torch.zeros(case.C, dtype=torch.float64, device="cuda"))
    zxs = [st.x.double() + (st.pre.double() if st.pre is not None else 0.0) for st in sts]
    zall = torch.cat(zxs) + cb
    mean, var = zall.mean(0), ((zall - zall.mean(0)) ** 2).mean(0)
    std = var.sqrt()
    invstd = 1.0 / torch.sqrt(var + EPS)
    km, ki = (sts[0].mean, sts[0].invstd) if stats is None else stats[0]
    for r, st in enumerate(sts):
        m_r, i_r = (st.mean, st.invstd) if stats is None else stats[r]
        assert torch.equal(m_r, km) and torch.equal(i_r, ki), f"rank {r}: saved statistics differ from rank 0"
    reg.assert_within(km, mean, 1e-5 * (mean.abs() + std) + 1e-30, "saved mean")
    # the merge of the W per-rank (mean, M2) pairs (module docstring): 2⁻²¹·mean_q(|m_q|·|m_q − mean|) on the variance
    m_q = torch.stack([z.mean(0) for z in zxs]) + cb
    dvar = 2.0 ** -21 * (m_q.abs() * (m_q - mean).abs()).mean(0)
    reg.assert_within(ki, invstd, invstd * (1e-5 + 0.5 * dvar / (var + EPS)), "saved invstd")
    for r, st in enumerate(sts):
        z = zxs[r] + cb
        res = st.res.double() if st.res is not None else None
        y_ref = (z - mean) * (invstd * gamma) + beta
        if res is not None:
            y_ref = y_ref + res
        if case.relu:
            y_ref = y_ref.clamp_min(0.0)
        sc = (invstd * gamma).abs()
        slack = 2.0 ** -19 * (zxs[r].abs() * sc + (mean.abs() + std + cb.abs()) * sc + beta.abs() + (res.abs() if res is not None else 0.0))
        y = (st.y if y_list is None else y_list[r]).double()
        tol = reg.ulp(y_ref, dt) + slack
        reg.assert_within(y, y_ref, tol, f"rank {r}: y")
    if rm0 is not None:
        for r, st in enumerate(sts):
            assert torch.equal(st.rm, sts[0].rm) and torch.equal(st.rv, sts[0].rv), f"rank {r}: running statistics"
            assert int(st.nbt.item()) == steps, f"rank {r}: num_batches_tracked"
    return km, ki, mean, var


@pytest.mark.parametrize("case", BN_CASES, ids=[c.id for c in BN_CASES])
def test_syncbn_at_world_w(case):
    reg = _reg()
    W = case.world
    rows, gf, gb = bn_geoms(case)
    dt = TORCH_DT[case.dtype]
    ex = int(L().sod_syncbn_exchange_bytes(case.C))
    vw = VirtualWorld(W, 2 * ex + 512)
    slots = [vw.alloc(ex, 16), vw.alloc(ex, 16)]
    sts = [BnRank(vw, r, case, rows, (case.id,)) for r in range(W)]
    rm0, rv0 = sts[0].rm.clone(), sts[0].rv.clone()

    def make():
        calls = []
        t_f, t_b = vw.tag(), vw.tag()
        for r, st in enumerate(sts):
            st.reset()
            seq = [bn_fwd_launch(vw, r, st, case, rows, gf, slots[0], t_f)]
            if case.kind == "bwd":
                seq.append(bn_bwd_launch(vw, r, st, case, rows, gb, slots[1], t_b))
            calls.append(seq)
        return calls
    vw.run(make, ORDERS[zlib.crc32(case.id.encode()) % 3])
    km, ki, mean, var = check_bn_forward(case, sts, rows, W, rm0=rm0, rv0=rv0)
    n = rows * W
    rm_ref = (1 - MOMENTUM) * rm0.double() + MOMENTUM * mean
    rv_ref = (1 - MOMENTUM) * rv0.double() + MOMENTUM * var * (n / (n - 1))
    upd = 2.0 ** -22 * ((1 - MOMENTUM) * rm0.double().abs() + MOMENTUM * mean.abs())
    reg.assert_within(sts[0].rm, rm_ref, 1e-5 * (rm_ref.abs() + MOMENTUM * var.sqrt()) + upd, "running mean")
    reg.assert_within(sts[0].rv, rv_ref, 1e-5 * rv_ref.abs() + 1e-30, "running var")
    if case.kind == "fwd":
        return
    # ---- backward: fp64 over all ranks with the kernel's saved statistics and ReLU mask ------------------------------
    gamma = sts[0].gamma.double()
    cb = sum((b.double() for b in sts[0].cbs), torch.zeros(case.C, dtype=torch.float64, device="cuda"))
    kmean, kinv = km.double(), ki.double()
    zs = [st.x.double() + (st.pre.double() if st.pre is not None else 0.0) + cb for st in sts]
    dms = [st.dy.double() * (st.y.double() > 0) if case.relu else st.dy.double() for st in sts]
    mdy = torch.cat(dms).mean(0)
    mdx = torch.cat([d * (z - kmean) for d, z in zip(dms, zs)]).mean(0)
    A = gamma * kinv
    B = -A * kinv * kinv * mdx
    abs_dy = torch.cat(dms).abs().mean(0)
    abs_dx = torch.cat([(d * (z - kmean)).abs() for d, z in zip(dms, zs)]).mean(0)
    for r, st in enumerate(sts):
        z, dm = zs[r], dms[r]
        dz_ref = (dm - mdy - (z - kmean) * kinv * kinv * mdx) * kinv * gamma
        slack = (2.0 ** -19 * ((A * dm).abs() + B.abs() * (z.abs() + kmean.abs()) + (A * mdy).abs())
                 + A.abs() * 2.0 ** -18 * abs_dy + (A * kinv * kinv).abs() * (z - kmean).abs() * 2.0 ** -18 * abs_dx)
        reg.assert_within(st.dz.double(), dz_ref, reg.ulp(dz_ref, dt) + slack, f"rank {r}: dz")
        if st.dres is not None:
            assert torch.equal(st.dres.double(), dm), f"rank {r}: dres is the masked dy"
        zx = z - cb
        z_round = kinv * (2.0 ** -22 * (kmean.abs() + cb.abs()) * dm.sum(0).abs() + 2.0 ** -23 * (dm * zx).pow(2).sum(0).sqrt())
        reg.assert_sum_close(st.dgamma.double(), (dm * (z - kmean) * kinv).sum(0), dm * (z - kmean) * kinv,
                             f"rank {r}: dgamma (local)", z_round)
        reg.assert_sum_close(st.dbeta.double(), dm.sum(0), dm, f"rank {r}: dbeta (local)")
        cb_terms = (A * dm).abs() + (B * (z - kmean)).abs()
        cb_round = B.abs() * 2.0 ** -22 * (kmean.abs() + cb.abs()) * rows + A.abs() * 2.0 ** -18 * abs_dy * rows
        for i, d in enumerate(st.dcbs):
            dcb_ref = dz_ref.sum(0)
            if d.dtype == torch.float32:
                reg.assert_sum_close(d.double(), dcb_ref, cb_terms, f"rank {r}: conv bias {i} gradient (local)", cb_round)
            else:
                tol = reg.ulp(dcb_ref, d.dtype) + 1e-5 * rows ** 0.5 * cb_terms.pow(2).mean(0).sqrt() + cb_round
                reg.assert_within(d, dcb_ref, tol, f"rank {r}: conv bias {i} gradient (local)")


@pytest.mark.parametrize("tags", ["seq", "epoch"])
@pytest.mark.parametrize("world", WORLDS)
def test_syncbn_tags_never_consume_a_stale_packet(world, tags):
    """6 forward + backward launches per rank through 4 exchange slots, enqueued without syncs, new inputs every time.
    seq: host-style tags, one counter over all calls.  epoch: the tags of graph replay — 3 iterations of 2 forward +
    backward pairs, call index c = 0..3 within the iteration in slot c, the epoch bumped on every rank's stream between
    iterations.  So each slot's previous occupant is the same call index of the previous iteration, and only the epoch
    part of the tag tells its packets from the new ones.  Forward and backward use separate workspaces, so that both
    grids are read back."""
    case = BnCase("tags", world, "bwd", "bfloat16", False, False, True, 64, "few")
    rows, gf, gb = bn_geoms(case)
    ex = int(L().sod_syncbn_exchange_bytes(case.C))
    vw = VirtualWorld(world, 4 * ex + 512)
    slots = [vw.alloc(ex, 16) for _ in range(4)]
    iters, rounds = (2, 3) if tags == "epoch" else (6, 1)
    sts = [BnRank(vw, r, case, rows, ("tags", world, tags)) for r in range(world)]
    epochs = [torch.zeros(1, dtype=torch.int32, device="cuda") for _ in range(world)]
    gen = torch.Generator(device="cuda").manual_seed(world)
    total = iters * rounds
    xs = [[(torch.randn(rows, case.C, generator=gen, device="cuda") * (1 + k % 3) + k + 0.5 * r).to(torch.bfloat16)
           for r in range(world)] for k in range(total)]
    dys = [[torch.randn(rows, case.C, generator=gen, device="cuda").to(torch.bfloat16) for r in range(world)] for k in range(total)]
    outs = [[dict(mean=torch.zeros(case.C, device="cuda"), invstd=torch.zeros(case.C, device="cuda"),
                  y=torch.zeros(rows, case.C, dtype=torch.bfloat16, device="cuda"),
                  dz=torch.zeros(rows, case.C, dtype=torch.bfloat16, device="cuda"),
                  dg=torch.zeros(case.C, device="cuda"), db=torch.zeros(case.C, device="cuda")) for r in range(world)]
            for k in range(total)]
    rm0, rv0 = sts[0].rm.clone(), sts[0].rv.clone()
    made = []

    def make():
        calls = [[] for _ in range(world)]
        base = [vw.tag() for _ in range(2 * total)]
        made.append(1)
        for r, st in enumerate(sts):
            st.reset()
            epochs[r].fill_(5 + 10 * len(made))        # every run its own epochs: nothing a previous run left matches
        for k in range(total):
            rnd, i = divmod(k, iters)
            for r, st in enumerate(sts):
                o = outs[k][r]

                def stage(r=r, k=k, st=st, o=o):
                    st.x.copy_(xs[k][r])
                    st.dy.copy_(dys[k][r])
                    st.dgamma, st.dbeta = o["dg"], o["db"]
                calls[r].append(Launch(stage))
                if tags == "epoch":
                    t_f, t_b, ep = 2 * i, 2 * i + 1, epochs[r]
                else:
                    t_f, t_b, ep = base[2 * k], base[2 * k + 1], None
                calls[r].append(bn_fwd_launch(vw, r, st, case, rows, gf, slots[(2 * k) % 4], t_f, ep, ws=0,
                                              out=(o["mean"], o["invstd"], o["y"])))
                calls[r].append(bn_bwd_launch(vw, r, st, case, rows, gb, slots[(2 * k + 1) % 4], t_b, ep, ws=1,
                                              inp=(o["mean"], o["invstd"], o["y"]), out=o["dz"]))
                if tags == "epoch" and i == iters - 1:
                    calls[r].append(Launch(lambda r=r: epochs[r].add_(1)))
        return calls
    vw.run(make, "forward")
    reg = _reg()
    rm_ref, rv_ref = rm0.double(), rv0.double()
    for k in range(total):
        for r, st in enumerate(sts):
            st.x = xs[k][r]
            st.dy = dys[k][r]
        stats = [(outs[k][r]["mean"], outs[k][r]["invstd"]) for r in range(world)]
        _, _, mean, var = check_bn_forward(case, sts, rows, world, y_list=[outs[k][r]["y"] for r in range(world)], stats=stats)
        n = rows * world
        rm_ref = (1 - MOMENTUM) * rm_ref + MOMENTUM * mean
        rv_ref = (1 - MOMENTUM) * rv_ref + MOMENTUM * var * (n / (n - 1))
        km, ki = stats[0][0].double(), stats[0][1].double()
        dms = [dys[k][r].double() * (outs[k][r]["y"].double() > 0) for r in range(world)]
        zs = [xs[k][r].double() for r in range(world)]
        mdy = torch.cat(dms).mean(0)
        mdx = torch.cat([d * (z - km) for d, z in zip(dms, zs)]).mean(0)
        A = sts[0].gamma.double() * ki
        B = -A * ki * ki * mdx
        abs_dy = torch.cat(dms).abs().mean(0)
        abs_dx = torch.cat([(d * (z - km)).abs() for d, z in zip(dms, zs)]).mean(0)
        for r in range(world):
            z, dm = zs[r], dms[r]
            dz_ref = (dm - mdy - (z - km) * ki * ki * mdx) * A
            slack = (2.0 ** -19 * ((A * dm).abs() + B.abs() * (z.abs() + km.abs()) + (A * mdy).abs())
                     + A.abs() * 2.0 ** -18 * abs_dy + (A * ki * ki).abs() * (z - km).abs() * 2.0 ** -18 * abs_dx)
            reg.assert_within(outs[k][r]["dz"].double(), dz_ref, reg.ulp(dz_ref, torch.bfloat16) + slack, f"launch {k} rank {r}: dz")
            reg.assert_sum_close(outs[k][r]["db"].double(), dm.sum(0), dm, f"launch {k} rank {r}: dbeta")
    for r, st in enumerate(sts):
        assert torch.equal(st.rm, sts[0].rm) and torch.equal(st.rv, sts[0].rv)
        assert int(st.nbt.item()) == total
    # the momentum updates compound: 1e-5 of each step's statistic, summed
    reg.assert_within(sts[0].rm, rm_ref, 1e-5 * total * (rm_ref.abs() + 1.0), "running mean after the sequence")
    reg.assert_within(sts[0].rv, rv_ref, 1e-5 * total * rv_ref.abs(), "running var after the sequence")
