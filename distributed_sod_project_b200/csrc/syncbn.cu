// syncbn.cu — synchronized batch-norm forward / backward with the cross-GPU statistics exchange and
// the (pre-add → normalize/affine → residual-add → ReLU) elementwise chain in ONE kernel per direction.
//
// Reference behaviour being replaced: apex.parallel.SyncBatchNorm as installed by
// convert_syncbn_model (reference train.py:180): local Welford → 2 NCCL all_gathers → elementwise
// forward; local reduce → 2 NCCL all_reduces → elementwise backward — four kernels and two latency-
// bound collectives per layer per direction, 84 layers.  Arithmetic spec (readable in-container
// equivalent): torch/nn/modules/_functions.py:7-209.
//
// Layout: channels-last matrix [rows = N·H·W, C].  One persistent CTA per SM owns a contiguous strip
// of rows (= a contiguous byte range), every thread owns one fixed group of 8 channels.
//
//   stage   the strip is pulled through a ring of shared-memory stages (32-48 KB each) by 1-D bulk async
//           copies (TMA engine, mbarrier completion) issued by a dedicated producer warp: ≈150 KB per
//           SM in flight with no registers tied up (geometry from tools/membench.cu: a bulk-copy ring
//           delivers ∝ bytes per stage, so stages are 32-48 KB rather than 8);
//   fold    biases of the convolutions that produced x / pre_add are added here (z = x + pre + b),
//           and their gradient Σ dz comes out of the backward's own statistics;
//   phase 1 per-thread fp32 partial sums straight from shared memory → CTA total [2C];
//   hop 1   the CTA total is written as 8-byte {value, tag} packets; CTA b then owns a slice of the
//           2C entries, waits for the packets of all CTAs (spins on the tag — an 8-byte store is
//           single-copy atomic, so there is no flag, no fence, no atomic, no counter to reset), sums
//           them in CTA order and
//   hop 2   publishes the GPU-local totals as packets to EVERY rank's exchange slot: multimem.st on the
//           NVLS multicast mapping (one store, the switch replicates) or per-peer stores;
//   phase 2 every CTA of every rank sums the W per-rank packets in rank order (bit-identical
//           statistics everywhere), derives the per-channel coefficients and normalizes its strip —
//           the last ring-full of the strip is still resident in shared memory and is NOT re-read;
//           only the part of the strip that did not fit streams through the ring again (from L2).
// world == 1 uses the same packet mechanism for the intra-GPU broadcast, so there is no grid barrier.
// All CTAs must be co-resident (grid ≤ #SMs, 1 CTA/SM). Every spin is bounded; a timeout sets
// comm->error_flag and lets the kernel run to completion (outstanding bulk copies must land).
#include <cstdlib>
#include <type_traits>

#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 512;             // consumer threads (warps 0..15); every data-layout stride uses this
constexpr int kWarps = kThreads / 32;
constexpr int kBlock = kThreads + 32;     // + one producer warp that only issues bulk copies
constexpr int kMaxC = 2048;
constexpr int kMaxStages = 16;
constexpr int kMaxGrid = 160;
constexpr int kRedBytes = 49152;          // scratch of the CTA reduction: kWarps x 24 statistics x 32 lanes x 4 B
constexpr int kSmemFixed = 256 /*barriers*/ + kRedBytes + 3 * kMaxC * 4 /*coefficients*/;

struct BnGeom {
    int C, es, L;                // channels, element bytes, lanes (= C/8 packets per row)
    int chunk_bytes;             // per stream per chunk
    int chunk_rows, ppt;         // rows per chunk, packets per thread per chunk
    int nstream, nstage;
    int strips, chunks_per_strip;
    long long rows, total_chunks;
};

struct BnWork {
    uint2* partials;   // [strips][2C or 3C] packets
    uint2* ll_local;   // [2C] packets, exchange slot when world == 1
    uint2* locpk;      // [3C] packets: GPU-local totals handed from the slice owners to CTA 0 (conv-bias gradient)
    unsigned long long* stamps;  // [kMaxGrid][8] globaltimer ns when SOD_DEBUG_TIMING is set, else null
                                 // slots: 0 start, 1 phase-1 end, 2 exchange end, 3 end, 4 CTA reduced, 5 my hop-1 slice published, 6 (unused)
};

__device__ __forceinline__ void stamp(const BnWork& w, int slot) {
    if (w.stamps != nullptr && threadIdx.x == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        w.stamps[blockIdx.x * 8 + slot] = t;
    }
}

struct BnFwd {
    const void *x, *pre, *res;
    void* y;
    const float *gamma, *beta;
    float *rmean, *rvar, *smean, *sinvstd;
    long long* nbt;  // num_batches_tracked (+= 1) or null
    const void *cbias1, *cbias2;  // biases of the convolution(s) feeding this BN, folded in here (z = x + pre + b1 + b2)
    int cbias_dtype;
    float momentum, eps;
    int relu, training;
    BnGeom g;
    BnWork w;
    CommDev c;
    uint64_t stats_off;
    uint32_t tag;
    const uint32_t* epoch;
    int use_mc;
};

struct BnBwd {
    const void *dy, *x, *pre, *y;
    void *dz, *dres;
    const float *gamma, *smean, *sinvstd;
    float *dgamma, *dbeta;
    const void *cbias1, *cbias2;
    void *dcbias1, *dcbias2;      // += Σ_rows dz (gradient of a folded conv bias), dtype cbias_dtype
    int cbias_dtype;
    int relu, accumulate;
    BnGeom g;
    BnWork w;
    CommDev c;
    uint64_t stats_off;
    uint32_t tag;
    const uint32_t* epoch;
    int use_mc;
    const float* beta;            // XMASK only: the ReLU mask is recomputed from x (y is not read)
    uint64_t store_policy;        // HINT only: L2 policy of the dz / dres stores
};

// folded conv bias of the 8 channels a thread owns (fp32 master or bf16 shadow leaves)
__device__ __forceinline__ float ld_bias(const void* p, int dtype, int ch) {
    if (p == nullptr) return 0.f;
    if (dtype == SOD_F32) return static_cast<const float*>(p)[ch];
    if (dtype == SOD_BF16) return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[ch]);
    return __half2float(static_cast<const __half*>(p)[ch]);
}
__device__ __forceinline__ void acc_bias_grad(void* p, int dtype, int ch, float v) {
    if (p == nullptr) return;
    if (dtype == SOD_F32) static_cast<float*>(p)[ch] += v;
    else if (dtype == SOD_BF16) {
        __nv_bfloat16* q = static_cast<__nv_bfloat16*>(p) + ch;
        *q = __float2bfloat16_rn(__bfloat162float(*q) + v);
    } else {
        __half* q = static_cast<__half*>(p) + ch;
        *q = __float2half_rn(__half2float(*q) + v);
    }
}

// tag of this call: host counter (eager) or device epoch + call index (CUDA-graph replay)
__device__ __forceinline__ uint32_t call_tag(uint32_t seq, const uint32_t* epoch) {
    return epoch ? (0x80000000u | ((*epoch & 0x1FFFFFu) << 10) | (seq & 1023u)) : (seq & 0x7FFFFFFFu);
}

// barrier among the 512 consumer threads only (the producer warp never joins it)
__device__ __forceinline__ void cbar() { asm volatile("bar.sync 1, 512;" ::: "memory"); }

// ---- packets -------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_packet_gpu(uint2* p, float v, uint32_t tag) {
    asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(v)), "r"(tag) : "memory");
}
__device__ __forceinline__ uint2 ld_packet_gpu(const uint2* p) {
    uint2 v;
    asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float wait_packet_gpu(const uint2* p, uint32_t tag, unsigned long long timeout, int& fail) {
    uint2 v = ld_packet_gpu(p);
    if (v.y != tag) {
        const long long t0 = clock64();
        do {
            v = ld_packet_gpu(p);
            if (static_cast<unsigned long long>(clock64() - t0) > timeout) { fail = 1; return 0.f; }
        } while (v.y != tag);
    }
    return __uint_as_float(v.x);
}
__device__ __forceinline__ float wait_packet_sys(const void* p, uint32_t tag, unsigned long long timeout, int& fail) {
    uint2 v = ld_relaxed_sys_v2(p);
    if (v.y != tag) {
        const long long t0 = clock64();
        do {
            v = ld_relaxed_sys_v2(p);
            if (static_cast<unsigned long long>(clock64() - t0) > timeout) { fail = 1; return 0.f; }
        } while (v.y != tag);
    }
    return __uint_as_float(v.x);
}

// hop 2: GPU-local total of entry `entry` → every rank's exchange slot [src_rank][2C]
__device__ __forceinline__ void publish(const CommDev& c, int use_mc, uint64_t stats_off, uint2* ll_local, int C, int entry,
                                        float value, uint32_t tag) {
    if (c.world == 1) {
        st_packet_gpu(ll_local + entry, value, tag);
        return;
    }
    const uint64_t off = stats_off + (static_cast<uint64_t>(c.rank) * 2u * C + entry) * 8u;
    const uint32_t bits = __float_as_uint(value);
    if (use_mc) {
        multimem_st_b64(reinterpret_cast<void*>(c.mc + off), bits, tag);
    } else {
        for (int q = 0; q < c.world; ++q) st_relaxed_sys_v2(reinterpret_cast<void*>(c.peer[q] + off), bits, tag);
    }
}
// slot of rank q's packet for `entry` in MY copy of the exchange area
__device__ __forceinline__ const void* slot_of(const CommDev& c, uint64_t stats_off, int C, int q, int entry) {
    return reinterpret_cast<const void*>(c.peer[c.rank] + stats_off + (static_cast<uint64_t>(q) * 2u * C + entry) * 8u);
}
// The W per-rank packets of one entry are requested TOGETHER (independent loads in flight: one round trip instead of W
// serialized ones — at world 8 that was ≈5 µs per launch), and whatever has not arrived is re-requested together, round
// after round.  Values are summed by the caller in rank order, so every rank obtains bit-identical statistics.
__device__ __forceinline__ void collect_all(const CommDev& c, uint64_t stats_off, int C, int entry, uint32_t tag,
                                            unsigned long long timeout, int& fail, float (&val)[SOD_MAX_WORLD]) {
    uint2 v[SOD_MAX_WORLD];
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) v[q] = ld_relaxed_sys_v2(slot_of(c, stats_off, C, q, entry));
    const long long t0 = clock64();
    for (;;) {
        bool late = false;
#pragma unroll
        for (int q = 0; q < SOD_MAX_WORLD; ++q) late |= (q < c.world) && (v[q].y != tag);
        if (!late) break;
#pragma unroll
        for (int q = 0; q < SOD_MAX_WORLD; ++q)
            if (q < c.world && v[q].y != tag) v[q] = ld_relaxed_sys_v2(slot_of(c, stats_off, C, q, entry));
        if (static_cast<unsigned long long>(clock64() - t0) > timeout) { fail = 1; break; }
    }
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q) val[q] = (q < c.world) ? __uint_as_float(v[q].x) : 0.f;
}
// two entries at once (forward: mean and M2 of one channel): all 2W packets travel together
__device__ __forceinline__ void collect_pair(const CommDev& c, uint64_t stats_off, int C, int e0, int e1, uint32_t tag,
                                             unsigned long long timeout, int& fail, float (&v0)[SOD_MAX_WORLD],
                                             float (&v1)[SOD_MAX_WORLD]) {
    uint2 a[SOD_MAX_WORLD], b[SOD_MAX_WORLD];
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) {
            a[q] = ld_relaxed_sys_v2(slot_of(c, stats_off, C, q, e0));
            b[q] = ld_relaxed_sys_v2(slot_of(c, stats_off, C, q, e1));
        }
    const long long t0 = clock64();
    for (;;) {
        bool late = false;
#pragma unroll
        for (int q = 0; q < SOD_MAX_WORLD; ++q) late |= (q < c.world) && (a[q].y != tag || b[q].y != tag);
        if (!late) break;
#pragma unroll
        for (int q = 0; q < SOD_MAX_WORLD; ++q) {
            if (q < c.world && a[q].y != tag) a[q] = ld_relaxed_sys_v2(slot_of(c, stats_off, C, q, e0));
            if (q < c.world && b[q].y != tag) b[q] = ld_relaxed_sys_v2(slot_of(c, stats_off, C, q, e1));
        }
        if (static_cast<unsigned long long>(clock64() - t0) > timeout) { fail = 1; break; }
    }
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q) {
        v0[q] = (q < c.world) ? __uint_as_float(a[q].x) : 0.f;
        v1[q] = (q < c.world) ? __uint_as_float(b[q].x) : 0.f;
    }
}
__device__ __forceinline__ float collect(const CommDev& c, uint64_t stats_off, const uint2* ll_local, int C, int entry,
                                         uint32_t tag, unsigned long long timeout, int& fail) {
    if (c.world == 1) return wait_packet_gpu(ll_local + entry, tag, timeout, fail);
    float val[SOD_MAX_WORLD];
    collect_all(c, stats_off, C, entry, tag, timeout, fail, val);
    float acc = 0.f;
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) acc += val[q];   // rank order: identical sum on every rank
    return acc;
}

// ---- shared-memory ring ---------------------------------------------------------------------------------
struct Ring {
    uint64_t* full;
    uint64_t* empty;
    unsigned char* stages;
    int nstage, nstream, chunk_bytes;
    uint32_t full_par, empty_par;  // bit s = parity of the next completion to wait for

    __device__ __forceinline__ unsigned char* buf(int s, int k) const {
        return stages + (static_cast<size_t>(s) * nstream + k) * chunk_bytes;
    }
    __device__ __forceinline__ void wait_full(int s) {
        mbar_wait(&full[s], (full_par >> s) & 1u);
        full_par ^= 1u << s;
    }
    // called by every thread after it has finished reading stage s, when the stage is going to be refilled
    __device__ __forceinline__ void release(int s) {
        __syncwarp();
        if ((threadIdx.x & 31) == 0)
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
    }
    // producer lane only
    __device__ __forceinline__ void wait_empty(int s) {
        mbar_wait(&empty[s], (empty_par >> s) & 1u);
        empty_par ^= 1u << s;
    }
};

struct StripInfo {
    long long chunk0;   // first chunk index of this strip
    int n;              // number of chunks in this strip
};

__device__ __forceinline__ StripInfo strip_info(const BnGeom& g) {
    StripInfo s;
    s.chunk0 = static_cast<long long>(blockIdx.x) * g.chunks_per_strip;
    long long rem = g.total_chunks - s.chunk0;
    s.n = static_cast<int>(rem < g.chunks_per_strip ? rem : g.chunks_per_strip);
    return s;
}
__device__ __forceinline__ int chunk_rows_of(const BnGeom& g, long long chunk) {
    const long long r0 = chunk * g.chunk_rows;
    const long long rem = g.rows - r0;
    return static_cast<int>(rem < g.chunk_rows ? rem : g.chunk_rows);
}

// thread 0: start the bulk copies of `chunk` (all streams) into stage s
template <int NS, bool HINT = false>
__device__ __forceinline__ void issue_chunk(Ring& ring, const BnGeom& g, const void* const (&src)[NS], int s, long long chunk,
                                            uint64_t policy = 0) {
    const uint32_t bytes = static_cast<uint32_t>(chunk_rows_of(g, chunk)) * g.C * g.es;
    const size_t off = static_cast<size_t>(chunk) * g.chunk_rows * g.C * g.es;
    int active = 0;
#pragma unroll
    for (int k = 0; k < NS; ++k) active += (src[k] != nullptr);
    mbar_arrive_expect_tx(&ring.full[s], bytes * active);
#pragma unroll
    for (int k = 0; k < NS; ++k)
        if (src[k] != nullptr) {
            if (HINT) bulk_g2s_hint(ring.buf(s, k), static_cast<const char*>(src[k]) + off, bytes, &ring.full[s], policy);
            else bulk_g2s(ring.buf(s, k), static_cast<const char*>(src[k]) + off, bytes, &ring.full[s]);
        }
}

// ---- CTA-level reduction of NA (16 or 24) per-thread accumulators over the threads that share a lane ----------
// on return `red[j]`, j = k*L + l  (statistic k of channel group l), holds the CTA total
template <int NA>
__device__ __forceinline__ void cta_reduce(float (&a)[NA], int L, float* red /*[kRedBytes/4]*/) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nent = NA * L;
    if (L <= 32) {
        // threads with equal (lane % L) inside a warp share a channel group: butterfly over the row-lanes
#pragma unroll
        for (int k = 0; k < NA; ++k) {
            float v = a[k];
            for (int o = 16; o >= L; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            a[k] = v;
        }
        if (lane < L) {
#pragma unroll
            for (int k = 0; k < NA; ++k) red[warp * nent + k * L + lane] = a[k];
        }
        cbar();
        float tot[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = tid + h * kThreads;
            if (j < nent) {
#pragma unroll
                for (int w = 0; w < kWarps; ++w) tot[h] += red[w * nent + j];
            }
        }
        cbar();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = tid + h * kThreads;
            if (j < nent) red[j] = tot[h];
        }
    } else {
        // L in {64,128,256}: thread tid owns lane l = tid % L; R = kThreads / L threads share it.
        // rounds of 8 statistics; scratch [R][8][L] floats = 16 KB sits behind the NA*L results
        const int l = tid % L, r = tid / L, R = kThreads / L;
        float* scratch = red + NA * 256;
#pragma unroll
        for (int part = 0; part < NA / 8; ++part) {
            cbar();
#pragma unroll
            for (int k = 0; k < 8; ++k) scratch[(r * 8 + k) * L + l] = a[part * 8 + k];
            cbar();
            for (int j = tid; j < 8 * L; j += kThreads) {
                float tot = 0.f;
                for (int rr = 0; rr < R; ++rr) tot += scratch[rr * 8 * L + j];
                red[part * 8 * L + j] = tot;  // j = k*L + l
            }
        }
    }
    cbar();
}

// hop 1 + hop 2 (+ optional per-entry side effect through `on_total`), then collect into red[0..n16)
template <typename F>
__device__ __forceinline__ void exchange(const BnGeom& g, const BnWork& w, const CommDev& c, int use_mc, uint64_t stats_off,
                                         uint32_t tag, float* red, int* s_fail, int na, F on_total) {
    // `na` statistics per channel group enter the CTA → GPU reduction (hop 1); only the first 16 are exchanged between
    // GPUs (hop 2).  With na == 24 the GPU-local totals of statistics 0-7 and 16-23 are also left in w.locpk for CTA 0.
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nglob = 16 * g.L;
    const int n16 = na * g.L;
    const int strips = static_cast<int>(gridDim.x);
    const unsigned long long timeout = c.timeout_cycles ? c.timeout_cycles : 4000000000ull;
    int fail = 0;
    // hop 1a: my CTA total as packets
    uint2* mine = w.partials + static_cast<size_t>(blockIdx.x) * n16;
    for (int j = tid; j < n16; j += kThreads) st_packet_gpu(mine + j, red[j], tag);
    // hop 1b: my slice of entries, summed over all CTAs in CTA order (one warp per entry; the ≤5 packets a lane
    // needs are requested together so their L2 round trips overlap)
    const int per = (n16 + strips - 1) / strips;
    const int j0 = blockIdx.x * per;
    const int j1 = (j0 + per < n16) ? j0 + per : n16;
    for (int j = j0 + warp; j < j1; j += kWarps) {
        constexpr int kMaxPer = (kMaxGrid + 31) / 32;
        uint2 v[kMaxPer];
#pragma unroll
        for (int u = 0; u < kMaxPer; ++u) {
            const int t = lane + 32 * u;
            if (t < strips) v[u] = ld_packet_gpu(w.partials + static_cast<size_t>(t) * n16 + j);
        }
        // packets that have not arrived yet are re-requested TOGETHER, round after round (a lane holds up to 5 of them:
        // polling them one after the other would chain that many L2 round trips behind the slowest CTA)
        {
            const long long t0 = clock64();
            for (;;) {
                bool late = false;
#pragma unroll
                for (int u = 0; u < kMaxPer; ++u) late |= (lane + 32 * u < strips) && (v[u].y != tag);
                if (!__any_sync(0xffffffffu, late)) break;
#pragma unroll
                for (int u = 0; u < kMaxPer; ++u) {
                    const int t = lane + 32 * u;
                    if (t < strips && v[u].y != tag) v[u] = ld_packet_gpu(w.partials + static_cast<size_t>(t) * n16 + j);
                }
                if (static_cast<unsigned long long>(clock64() - t0) > timeout) { fail = 1; break; }
            }
        }
        float acc = 0.f;
#pragma unroll
        for (int u = 0; u < kMaxPer; ++u)
            if (lane + 32 * u < strips) acc += __uint_as_float(v[u].x);
        acc = warp_sum(acc);
        if (lane == 0) {
            if (j < nglob) {
                on_total(j, acc);
                publish(c, use_mc, stats_off, w.ll_local, g.C, j, acc, tag);  // hop 2
            }
            if (na > 16) st_packet_gpu(w.locpk + j, acc, tag);
        }
    }
    stamp(w, 5);
    cbar();  // everyone has finished reading red[] (hop 1a) before it is overwritten
    for (int j = tid; j < nglob; j += kThreads) red[j] = collect(c, stats_off, w.ll_local, g.C, j, tag, timeout, fail);
    if (fail) {
        *s_fail = 1;
        if (c.error_flag) atomicExch(c.error_flag, 0xDEAD0001u);
    }
    cbar();
}

// number of rows of strip t (all strips hold chunks_per_strip chunks except the last)
__device__ __forceinline__ float strip_rows(const BnGeom& g, int t) {
    const long long per = static_cast<long long>(g.chunks_per_strip) * g.chunk_rows;
    const long long r0 = per * t;
    const long long r1 = (r0 + per < g.rows) ? r0 + per : g.rows;
    return static_cast<float>(r1 - r0);
}

// Forward statistics exchange in (mean, M2) form — the parallel-variance merge apex / torch SyncBN use
// (torch/nn/modules/_functions.py: batch_norm_gather_stats_with_counts), evaluated in a fixed order.
// On entry  red[j] = Σ (r − s) and red[C + j] = Σ (r − s)² over THIS strip, j = k*L + l (C = 8L channels), s = s_raw[channel].
// On return red[j] = mean over all rows of all ranks, red[C + j] = biased variance, identical on every CTA and rank.
__device__ __forceinline__ void exchange_moments(const BnGeom& g, const BnWork& w, const CommDev& c, int use_mc, uint64_t stats_off,
                                                 uint32_t tag, float* red, const float* s_raw, int* s_fail) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int C = 8 * g.L;
    const int n16 = 2 * C;
    const int strips = static_cast<int>(gridDim.x);
    const unsigned long long timeout = c.timeout_cycles ? c.timeout_cycles : 4000000000ull;
    const float n_gpu = static_cast<float>(g.rows);
    int fail = 0;
    // hop 1a: my strip's (mean, M2) as packets — M2 = Σ(r−s)² − (Σ(r−s))²/n is well conditioned because s is a sample
    uint2* mine = w.partials + static_cast<size_t>(blockIdx.x) * n16;
    {
        const float nb = strip_rows(g, blockIdx.x);
        for (int j = tid; j < C; j += kThreads) {
            const int ch = (j % g.L) * 8 + (j / g.L);
            const float s1 = red[j], s2 = red[j + C];
            st_packet_gpu(mine + j, s_raw[ch] + s1 / nb, tag);
            st_packet_gpu(mine + C + j, fmaxf(s2 - s1 * (s1 / nb), 0.f), tag);
        }
    }
    // hop 1b: my slice of CHANNELS; one warp per channel, lane t (+32u) holds strip t's pair
    const int per = (C + strips - 1) / strips;
    const int j0 = blockIdx.x * per;
    const int j1 = (j0 + per < C) ? j0 + per : C;
    for (int j = j0 + warp; j < j1; j += kWarps) {
        constexpr int kMaxPer = (kMaxGrid + 31) / 32;
        uint2 vm[kMaxPer], vq[kMaxPer];
#pragma unroll
        for (int u = 0; u < kMaxPer; ++u) {
            const int t = lane + 32 * u;
            if (t < strips) {
                vm[u] = ld_packet_gpu(w.partials + static_cast<size_t>(t) * n16 + j);
                vq[u] = ld_packet_gpu(w.partials + static_cast<size_t>(t) * n16 + C + j);
            }
        }
        {   // late packets are re-requested together, round after round (see exchange())
            const long long t0 = clock64();
            for (;;) {
                bool late = false;
#pragma unroll
                for (int u = 0; u < kMaxPer; ++u) late |= (lane + 32 * u < strips) && (vm[u].y != tag || vq[u].y != tag);
                if (!__any_sync(0xffffffffu, late)) break;
#pragma unroll
                for (int u = 0; u < kMaxPer; ++u) {
                    const int t = lane + 32 * u;
                    if (t < strips && vm[u].y != tag) vm[u] = ld_packet_gpu(w.partials + static_cast<size_t>(t) * n16 + j);
                    if (t < strips && vq[u].y != tag) vq[u] = ld_packet_gpu(w.partials + static_cast<size_t>(t) * n16 + C + j);
                }
                if (static_cast<unsigned long long>(clock64() - t0) > timeout) { fail = 1; break; }
            }
        }
        float m[kMaxPer], q2[kMaxPer], nt[kMaxPer];
        float sm = 0.f;
#pragma unroll
        for (int u = 0; u < kMaxPer; ++u) {
            const int t = lane + 32 * u;
            m[u] = 0.f; q2[u] = 0.f; nt[u] = 0.f;
            if (t < strips) {
                m[u] = __uint_as_float(vm[u].x);
                q2[u] = __uint_as_float(vq[u].x);
                nt[u] = strip_rows(g, t);
                sm = fmaf(nt[u], m[u], sm);
            }
        }
        const float mean = warp_sum(sm) / n_gpu;
        float sq = 0.f;
#pragma unroll
        for (int u = 0; u < kMaxPer; ++u) {
            const float d = m[u] - mean;
            sq += q2[u] + nt[u] * d * d;         // nt == 0 for the lanes without a strip
        }
        sq = warp_sum(sq);
        if (lane == 0) {   // hop 2: this GPU's (mean, M2) to every rank
            publish(c, use_mc, stats_off, w.ll_local, C, j, mean, tag);
            publish(c, use_mc, stats_off, w.ll_local, C, C + j, sq, tag);
        }
    }
    stamp(w, 5);
    cbar();  // everyone has finished reading red[] (hop 1a) before it is overwritten
    for (int j = tid; j < C; j += kThreads) {
        float mean, var;
        if (c.world == 1) {
            const uint2 a = ld_packet_gpu(w.ll_local + j), b = ld_packet_gpu(w.ll_local + C + j);   // both in flight
            mean = (a.y == tag) ? __uint_as_float(a.x) : wait_packet_gpu(w.ll_local + j, tag, timeout, fail);
            var = ((b.y == tag) ? __uint_as_float(b.x) : wait_packet_gpu(w.ll_local + C + j, tag, timeout, fail)) / n_gpu;
        } else {
            float mq[SOD_MAX_WORLD], sq[SOD_MAX_WORLD];
            collect_pair(c, stats_off, C, j, C + j, tag, timeout, fail, mq, sq);
            float sm = 0.f;
#pragma unroll
            for (int q = 0; q < SOD_MAX_WORLD; ++q)
                if (q < c.world) sm += mq[q];              // every rank contributes the same number of rows
            mean = sm / static_cast<float>(c.world);
            float acc = 0.f;
#pragma unroll
            for (int q = 0; q < SOD_MAX_WORLD; ++q)
                if (q < c.world) {
                    const float d = mq[q] - mean;
                    acc += sq[q] + n_gpu * d * d;
                }
            var = acc / (n_gpu * static_cast<float>(c.world));
        }
        red[j] = mean;
        red[C + j] = var;
    }
    if (fail) {
        *s_fail = 1;
        if (c.error_flag) atomicExch(c.error_flag, 0xDEAD0001u);
    }
    cbar();
}

__device__ __forceinline__ void ring_setup(Ring& ring, unsigned char* smem, const BnGeom& g, int nstream) {
    ring.full = reinterpret_cast<uint64_t*>(smem);
    ring.empty = ring.full + kMaxStages;
    ring.stages = smem + kSmemFixed;
    ring.nstage = g.nstage;
    ring.nstream = nstream;
    ring.chunk_bytes = g.chunk_bytes;
    ring.full_par = 0;
    ring.empty_par = 0;
    if (threadIdx.x == 0) {
        for (int s = 0; s < g.nstage; ++s) {
            mbar_init(&ring.full[s], 1);
            mbar_init(&ring.empty[s], kWarps);
        }
        mbar_fence_init();
    }
    __syncthreads();  // all kBlock threads (the only block-wide barrier in the kernels)
    // programmatic dependent launch: everything above overlapped the producing kernel's tail; nothing below may read
    // global memory before that kernel has completed (a no-op for a normal launch)
    asm volatile("griddepcontrol.wait;" ::: "memory");
}

// The load sequence of one CTA (training): chunks 0..n-1 for phase 1, then the chunks that did not stay resident,
// newest first (the likeliest L2 hits), for phase 2.  Load k goes to stage k % NS.
__device__ __forceinline__ int load_chunk_of(int k, int n, int nres0) { return k < n ? k : nres0 - 1 - (k - n); }

// producer warp: lane 0 keeps the ring full
// HINT (experimental, SOD_BN_L2_HINTS): a chunk that phase 2 will have to fetch again (it does not stay resident in
// shared memory) is loaded evict-last; every last use — the chunks that stay resident, and all phase-2 re-reads — is
// loaded evict-first, so that the re-read set rather than dead data occupies L2.
template <int NSRC, bool HINT = false>
__device__ __forceinline__ void producer_loop(Ring& ring, const BnGeom& g, const void* const (&src)[NSRC], const StripInfo& sp,
                                              int total_loads, int nres0) {
    if ((threadIdx.x & 31) != 0) return;
    const int NS = g.nstage;
    for (int k = 0; k < total_loads; ++k) {
        const int s = k % NS;
        if (k >= NS) ring.wait_empty(s);
        if (HINT) {
            const bool again = k < sp.n && k < nres0;     // phase-1 load of a chunk that will not stay resident
            issue_chunk<NSRC, true>(ring, g, src, s, sp.chunk0 + load_chunk_of(k, sp.n, nres0), again ? kL2EvictLast : kL2EvictFirst);
        } else {
            issue_chunk<NSRC>(ring, g, src, s, sp.chunk0 + load_chunk_of(k, sp.n, nres0));
        }
    }
}

// =================================================================================================
// forward
// =================================================================================================
template <typename T, int PPT, bool RES>
__global__ void __launch_bounds__(kBlock, 1) syncbn_fwd_kernel(const __grid_constant__ BnFwd prm) {
    extern __shared__ __align__(128) unsigned char smem[];
    float* red = reinterpret_cast<float*>(smem + 256);
    float* s_scale = reinterpret_cast<float*>(smem + 256 + kRedBytes);
    float* s_shift = s_scale + kMaxC;
    __shared__ int s_fail;

    const BnGeom& g = prm.g;
    const int tid = threadIdx.x;
    const int L = g.L, C = g.C;
    const StripInfo sp = strip_info(g);
    const int NS = g.nstage;
    const bool has_pre = prm.pre != nullptr;
    const bool training = prm.training != 0;
    const int nres0 = training ? (sp.n > NS ? sp.n - NS : 0) : 0;   // chunks [nres0, n) stay resident after phase 1
    const int total_loads = training ? sp.n + nres0 : sp.n;
    if (tid == 0) s_fail = 0;
    stamp(prm.w, 0);

    Ring ring;
    ring_setup(ring, smem, g, has_pre ? 2 : 1);
    const void* const src[2] = {prm.x, prm.pre};
    if (tid >= kThreads) {  // ---- producer warp --------------------------------------------------------------
        producer_loop<2>(ring, g, src, sp, total_loads, nres0);
        return;
    }

    // ---- consumers -------------------------------------------------------------------------------------
    const int l = tid % L;
    float* s_raw = s_shift + kMaxC;      // per-channel shift of the statistics pass (first row of this strip)
    const T* __restrict__ gres = RES ? static_cast<const T*>(prm.res) : nullptr;
    T* __restrict__ gy = static_cast<T*>(prm.y);
    // affine / running parameters are fetched now so their DRAM latency hides behind phase 1
    for (int ch = tid; ch < C; ch += kThreads) {
        s_scale[ch] = prm.gamma[ch];
        s_shift[ch] = prm.beta[ch];
    }
    // folded conv bias of this thread's first channel (every channel when C ≤ 512), also fetched ahead of the exchange
    const float cb_first = (tid < C) ? ld_bias(prm.cbias1, prm.cbias_dtype, tid) + ld_bias(prm.cbias2, prm.cbias_dtype, tid) : 0.f;
    // The per-channel global side effects (saved statistics, running statistics) are spread over the grid: channel ch
    // belongs to CTA ch % gridDim — CTA 0 doing all C read-modify-writes after the exchange made it the last CTA to finish
    // (≈1.8 µs behind the median, tools/bn_phases.py).  The old running values of the first owned channel are fetched now.
    const int G = static_cast<int>(gridDim.x);
    const int ch_own = static_cast<int>(blockIdx.x) + tid * G;
    float rm_own = 0.f, rv_own = 0.f;
    if (training && prm.rmean != nullptr && ch_own < C) {
        rm_own = prm.rmean[ch_own];
        rv_own = prm.rvar[ch_own];
    }

    if (training) {
        // ---- phase 1: Σ(r − s), Σ(r − s)² from shared memory, r = x (+ pre) --------------------------------
        // s = the strip's first row: sums of deviations from a sample of the distribution stay well conditioned where
        // E[r²] − E[r]² loses the variance (|mean| ≫ std).  A folded conv bias is a per-channel constant: it moves the
        // mean by b and nothing else, so it does not enter this pass at all.
        float a[16], off[8];
#pragma unroll
        for (int k = 0; k < 16; ++k) a[k] = 0.f;
        for (int i = 0; i < sp.n; ++i) {
            const int s = i % NS;
            ring.wait_full(s);
            const int npk = chunk_rows_of(g, sp.chunk0 + i) * L;
            const T* xs = reinterpret_cast<const T*>(ring.buf(s, 0));
            const T* ps = reinterpret_cast<const T*>(ring.buf(s, 1));
            if (i == 0) {
                IO<T>::load8(xs + l * 8, off);
                if (has_pre) {
                    float t[8];
                    IO<T>::load8(ps + l * 8, t);
#pragma unroll
                    for (int k = 0; k < 8; ++k) off[k] += t[k];
                }
                if (tid < L) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) s_raw[l * 8 + k] = off[k];
                }
            }
            {
                const int qb = tid;
                typename IO<T>::Raw rx[PPT], rp[PPT];
#pragma unroll
                for (int j = 0; j < PPT; ++j) {
                    const int q = qb + j * kThreads;
                    if (q < npk) {
                        rx[j] = IO<T>::load_raw(xs + q * 8);
                        if (has_pre) rp[j] = IO<T>::load_raw(ps + q * 8);
                    }
                }
#pragma unroll
                for (int j = 0; j < PPT; ++j) {
                    const int q = qb + j * kThreads;
                    if (q < npk) {
                        float z[8];
                        IO<T>::unpack(rx[j], z);
                        if (has_pre) {
                            float t[8];
                            IO<T>::unpack(rp[j], t);
#pragma unroll
                            for (int k = 0; k < 8; ++k) z[k] += t[k];
                        }
#pragma unroll
                        for (int k = 0; k < 8; ++k) {
                            const float d = z[k] - off[k];
                            a[k] += d;
                            a[8 + k] = fmaf(d, d, a[8 + k]);
                        }
                    }
                }
            }
            if (i + NS < sp.n) ring.release(s);  // recycled within phase 1
        }
        stamp(prm.w, 1);
        cta_reduce<16>(a, L, red);
        stamp(prm.w, 4);
        exchange_moments(g, prm.w, prm.c, prm.use_mc, prm.stats_off, call_tag(prm.tag, prm.epoch), red, s_raw, &s_fail);
        stamp(prm.w, 2);
        // ---- per-channel coefficients --------------------------------------------------------------------
        // The shift is built from the STORED mean (which includes the folded bias) in the same operation order the
        // backward's mask-from-x variant uses (syncbn_bwd_kernel, "msc"/"msh"), so both derive the same sign for y.
        const float n = static_cast<float>(g.rows) * static_cast<float>(prm.c.world);
        for (int ch = tid; ch < C; ch += kThreads) {
            const int ll = ch >> 3, k = ch & 7;
            const float cbv = (ch == tid) ? cb_first : ld_bias(prm.cbias1, prm.cbias_dtype, ch) + ld_bias(prm.cbias2, prm.cbias_dtype, ch);
            const float mean = red[k * L + ll] + cbv;
            const float var = red[(8 + k) * L + ll];
            const float invstd = 1.0f / sqrtf(var + prm.eps);
            const float sc = invstd * s_scale[ch];
            s_scale[ch] = sc;
            s_shift[ch] = fmaf(cbv, sc, fmaf(-mean, sc, s_shift[ch]));
        }
        // side effects of the channels this CTA owns (same arithmetic as above, so every copy of a statistic is identical)
        for (int ch = ch_own; ch < C; ch += kThreads * G) {
            const int ll = ch >> 3, k = ch & 7;
            const float cbv = ld_bias(prm.cbias1, prm.cbias_dtype, ch) + ld_bias(prm.cbias2, prm.cbias_dtype, ch);
            const float mean = red[k * L + ll] + cbv;
            const float var = red[(8 + k) * L + ll];
            prm.smean[ch] = mean;
            prm.sinvstd[ch] = 1.0f / sqrtf(var + prm.eps);
            if (prm.rmean) {
                const float unbiased = var * (n / fmaxf(n - 1.f, 1.f));
                const float rm = (ch == ch_own) ? rm_own : prm.rmean[ch];
                const float rv = (ch == ch_own) ? rv_own : prm.rvar[ch];
                prm.rmean[ch] = (1.f - prm.momentum) * rm + prm.momentum * mean;
                prm.rvar[ch] = (1.f - prm.momentum) * rv + prm.momentum * unbiased;
            }
        }
        if (blockIdx.x == 0 && tid == 0 && prm.nbt) *prm.nbt += 1;
    } else {
        for (int ch = tid; ch < C; ch += kThreads) {
            const float cbv = (ch == tid) ? cb_first : ld_bias(prm.cbias1, prm.cbias_dtype, ch) + ld_bias(prm.cbias2, prm.cbias_dtype, ch);
            const float invstd = 1.0f / sqrtf(prm.rvar[ch] + prm.eps);
            const float sc = invstd * s_scale[ch];
            s_scale[ch] = sc;
            s_shift[ch] = fmaf(cbv, sc, fmaf(-prm.rmean[ch], sc, s_shift[ch]));
        }
    }
    cbar();

    // ---- phase 2: normalize; resident chunks first, then the part of the strip that did not fit ---------
    float sc[8], sh[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        sc[k] = s_scale[l * 8 + k];
        sh[k] = s_shift[l * 8 + k];                          // the folded conv bias is already inside the shift
    }
    const bool relu = prm.relu != 0;
    const int nresident = training ? sp.n - nres0 : 0;
    // use u of phase 2: u < nresident → resident chunk nres0+u (no wait); else load k = n + (u - nresident) (training)
    // or plain ring order (eval)
    constexpr int kPptMax = PPT;
    constexpr int kResBuf = RES ? PPT : 1;
    typename IO<T>::Raw rcur[kResBuf], rnext[kResBuf];
    auto chunk_of = [&](int u) -> int {
        if (!training) return u;
        return u < nresident ? nres0 + u : nres0 - 1 - (u - nresident);
    };
    // the residual is read straight from global memory, one chunk ahead, so its latency hides behind the math
    auto fetch_res = [&](int u, typename IO<T>::Raw (&dst)[kResBuf]) {
        if (!RES || u >= sp.n) return;
        const long long chunk = sp.chunk0 + chunk_of(u);
        const int npk = chunk_rows_of(g, chunk) * L;
        const size_t ebase = static_cast<size_t>(chunk) * g.chunk_rows * C;
#pragma unroll
        for (int j = 0; j < kResBuf; ++j) {
            const int q = tid + j * kThreads;
            if (q < npk) dst[j] = IO<T>::load_raw(gres + ebase + static_cast<size_t>(q) * 8);
        }
    };
    fetch_res(0, rcur);
    for (int u = 0; u < sp.n; ++u) {
        const int c = chunk_of(u);
        const bool streamed = training ? (u >= nresident) : true;
        const int kload = training ? sp.n + (u - nresident) : u;        // load index when streamed
        const int s = training ? (streamed ? kload % NS : (nres0 + u) % NS) : u % NS;
        fetch_res(u + 1, rnext);
        if (streamed) ring.wait_full(s);
        const long long chunk = sp.chunk0 + c;
        const int npk = chunk_rows_of(g, chunk) * L;
        const T* xs = reinterpret_cast<const T*>(ring.buf(s, 0));
        const T* ps = reinterpret_cast<const T*>(ring.buf(s, 1));
        const size_t ebase = static_cast<size_t>(chunk) * g.chunk_rows * C;
        typename IO<T>::Raw rx[kPptMax], rp[kPptMax];
#pragma unroll
        for (int j = 0; j < kPptMax; ++j) {
            const int q = tid + j * kThreads;
            if (q < npk) {
                rx[j] = IO<T>::load_raw(xs + q * 8);
                if (has_pre) rp[j] = IO<T>::load_raw(ps + q * 8);
            }
        }
#pragma unroll
        for (int j = 0; j < kPptMax; ++j) {
            const int q = tid + j * kThreads;
            if (q < npk) {
                float z[8];
                IO<T>::unpack(rx[j], z);
                if (has_pre) {
                    float t[8];
                    IO<T>::unpack(rp[j], t);
#pragma unroll
                    for (int k = 0; k < 8; ++k) z[k] += t[k];
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) z[k] = fmaf(z[k], sc[k], sh[k]);
                if (RES) {
                    float t[8];
                    IO<T>::unpack(rcur[RES ? j : 0], t);
#pragma unroll
                    for (int k = 0; k < 8; ++k) z[k] += t[k];
                }
                if (relu) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) z[k] = fmaxf(z[k], 0.f);
                }
                IO<T>::store8(gy + ebase + static_cast<size_t>(q) * 8, z);
            }
        }
#pragma unroll
        for (int j = 0; j < kResBuf; ++j) rcur[j] = rnext[j];
        // release the stage iff a later load targets it
        const int stage_load = training ? (streamed ? kload : nres0 + u) : u;   // index of the load that filled this stage
        if (stage_load + NS < total_loads) ring.release(s);
    }
    stamp(prm.w, 3);
}

// =================================================================================================
// backward
// =================================================================================================
// 8 values → element type → 16-byte stores carrying an L2 policy (HINT variants only)
template <typename T>
__device__ __forceinline__ void store8_hint(T* p, const float (&f)[8], uint64_t policy) {
    if constexpr (sizeof(T) == 4) {
        st16_hint(p, make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3])), policy);
        st16_hint(p + 4, make_uint4(__float_as_uint(f[4]), __float_as_uint(f[5]), __float_as_uint(f[6]), __float_as_uint(f[7])), policy);
    } else {
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if constexpr (std::is_same<T, __nv_bfloat16>::value) {
                const __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
                w[i] = *reinterpret_cast<const uint32_t*>(&h);
            } else {
                const __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
                w[i] = *reinterpret_cast<const uint32_t*>(&h);
            }
        }
        st16_hint(p, make_uint4(w[0], w[1], w[2], w[3]), policy);
    }
}

// XMASK (experimental, SOD_BN_BWD_MASK_FROM_X): a BN+ReLU layer without residual does not stream y at all — the
// mask y > 0 is re-derived from x with the forward's own arithmetic (y = fma(z, invstd*γ, fma(b, invstd*γ, β - mean*invstd*γ)),
// same operations in the same order, so the sign agrees with the stored y; for bf16 except where |y| is below the
// smallest bf16 denormal, for fp16 see stored_positive).  One stream less to read twice: compulsory bytes drop from 4
// to 3 tensors, and a third more of the strip stays resident.
//
// y > 0 as the forward STORED it: an fp16 store rounds every fp32 y in (0, 2^-25] to +0, where torch's relu (and the
// y-mask variant) pass no gradient, so the fp16 sign is taken after the same rounding.
template <typename T>
__device__ __forceinline__ bool stored_positive(float y) {
    if constexpr (std::is_same<T, __half>::value) return __half2float(__float2half_rn(y)) > 0.f;
    else return y > 0.f;
}

template <typename T, int NSTAT, bool XMASK = false, bool HINT = false>
__global__ void __launch_bounds__(kBlock, 1) syncbn_bwd_kernel(const __grid_constant__ BnBwd prm) {
    extern __shared__ __align__(128) unsigned char smem[];
    float* red = reinterpret_cast<float*>(smem + 256);
    float* s_a = reinterpret_cast<float*>(smem + 256 + kRedBytes);
    float* s_b = s_a + kMaxC;
    float* s_d = s_b + kMaxC;
    __shared__ int s_fail;

    const BnGeom& g = prm.g;
    const int tid = threadIdx.x;
    const int L = g.L, C = g.C;
    const StripInfo sp = strip_info(g);
    const int NS = g.nstage;
    const bool has_pre = prm.pre != nullptr;
    const bool relu = prm.relu != 0;
    const int nres0 = sp.n > NS ? sp.n - NS : 0;
    const int total_loads = sp.n + nres0;
    if (tid == 0) s_fail = 0;
    stamp(prm.w, 0);

    Ring ring;
    ring_setup(ring, smem, g, g.nstream);
    // stream slots: 0 dy, 1 x, then pre (if any), then y (if relu)
    const int k_pre = 2, k_y = has_pre ? 3 : 2;
    const void* src[4] = {prm.dy, prm.x, nullptr, nullptr};
    if (has_pre) src[k_pre] = prm.pre;
    if (relu && !XMASK) src[k_y] = prm.y;
    const void* const csrc[4] = {src[0], src[1], src[2], src[3]};
    if (tid >= kThreads) {  // ---- producer warp --------------------------------------------------------------
        producer_loop<4, HINT>(ring, g, csrc, sp, total_loads, nres0);
        return;
    }

    const int l = tid % L;
    T* __restrict__ gdz = static_cast<T*>(prm.dz);
    T* __restrict__ gdres = static_cast<T*>(prm.dres);
    // saved statistics / affine parameters: fetched now, used after the exchange
    for (int ch = tid; ch < C; ch += kThreads) {
        s_a[ch] = prm.gamma[ch];
        s_b[ch] = prm.sinvstd[ch];
        s_d[ch] = prm.smean[ch];
    }
    cbar();
    float mean[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) mean[k] = s_d[l * 8 + k];
    // folded conv bias: z = x + pre + b, so (z - mean) = (x + pre) - (mean - b): fold b into the per-thread mean
    constexpr bool kFold = NSTAT == 24;
    float cb[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        cb[k] = kFold ? ld_bias(prm.cbias1, prm.cbias_dtype, l * 8 + k) + ld_bias(prm.cbias2, prm.cbias_dtype, l * 8 + k) : 0.f;
        mean[k] -= cb[k];
    }
    // XMASK: the forward's scale and shift of this thread's 8 channels (csrc: syncbn_fwd_kernel, "sc" / "sh")
    float msc[XMASK ? 8 : 1], msh[XMASK ? 8 : 1];
    if (XMASK) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ch = l * 8 + k;
            const float sc = s_b[ch] * s_a[ch];                       // invstd * γ
            const float sh0 = fmaf(-s_d[ch], sc, prm.beta[ch]);       // β - mean * sc, as the forward contracts it
            msc[XMASK ? k : 0] = sc;
            msh[XMASK ? k : 0] = fmaf(cb[k], sc, sh0);
        }
    }

    // one packet of work, shared by both phases (measured: interleaving two packets per thread only added register
    // pressure here — four streams per packet already give the scheduler independent loads)
    auto load_packet = [&](int s, int q, float (&d)[8], float (&z)[8]) {
        IO<T>::load8(reinterpret_cast<const T*>(ring.buf(s, 0)) + q * 8, d);
        IO<T>::load8(reinterpret_cast<const T*>(ring.buf(s, 1)) + q * 8, z);
        if (has_pre) {
            float t[8];
            IO<T>::load8(reinterpret_cast<const T*>(ring.buf(s, k_pre)) + q * 8, t);
#pragma unroll
            for (int k = 0; k < 8; ++k) z[k] += t[k];
        }
        if (XMASK) {
#pragma unroll
            for (int k = 0; k < 8; ++k) d[k] = stored_positive<T>(fmaf(z[k], msc[XMASK ? k : 0], msh[XMASK ? k : 0])) ? d[k] : 0.f;
        } else if (relu) {
            float o[8];
            IO<T>::load8(reinterpret_cast<const T*>(ring.buf(s, k_y)) + q * 8, o);
#pragma unroll
            for (int k = 0; k < 8; ++k) d[k] = o[k] > 0.f ? d[k] : 0.f;
        }
    };

    // ---- phase 1: Σ dy_m and Σ dy_m (z - mean) -------------------------------------------------------------
    float a[NSTAT];
#pragma unroll
    for (int k = 0; k < NSTAT; ++k) a[k] = 0.f;
    for (int i = 0; i < sp.n; ++i) {
        const int s = i % NS;
        ring.wait_full(s);
        const int npk = chunk_rows_of(g, sp.chunk0 + i) * L;
        for (int q = tid; q < npk; q += kThreads) {
            float d[8], z[8];
            load_packet(s, q, d, z);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float zc = z[k] - mean[k];
                a[k] += d[k];
                a[8 + k] = fmaf(d[k], zc, a[8 + k]);
                if (kFold) a[16 + k] += zc;          // Σ (z - mean) over the LOCAL rows → gradient of the folded bias
            }
        }
        if (i + NS < sp.n) ring.release(s);
    }
    stamp(prm.w, 1);
    cta_reduce<NSTAT>(a, L, red);
    stamp(prm.w, 4);
    {
        const float* sinv = s_b;
        float* dgamma = prm.dgamma;
        float* dbeta = prm.dbeta;
        const int LL = L;
        const bool accumulate = prm.accumulate != 0;
        // GPU-local totals are also the local parameter gradients (the gradient all-reduce averages them later)
        exchange(g, prm.w, prm.c, prm.use_mc, prm.stats_off, call_tag(prm.tag, prm.epoch), red, &s_fail, NSTAT, [=](int j, float tot) {
            const int k = j / LL, ll = j % LL;
            const int ch = ll * 8 + (k & 7);
            if (accumulate) {
                if (k < 8) dbeta[ch] += tot;
                else dgamma[ch] += tot * sinv[ch];
            } else {
                if (k < 8) dbeta[ch] = tot;
                else dgamma[ch] = tot * sinv[ch];
            }
        });
    }
    stamp(prm.w, 2);
    {
        const float n = static_cast<float>(g.rows) * static_cast<float>(prm.c.world);
        for (int ch = tid; ch < C; ch += kThreads) {
            const int ll = ch >> 3, k = ch & 7;
            const float mean_dy = red[k * L + ll] / n;
            const float mean_dy_xmu = red[(8 + k) * L + ll] / n;
            const float invstd = s_b[ch];
            const float A = s_a[ch] * invstd;
            const float B = -A * invstd * invstd * mean_dy_xmu;
            float mu = s_d[ch];
            if (kFold) {
                mu -= ld_bias(prm.cbias1, prm.cbias_dtype, ch) + ld_bias(prm.cbias2, prm.cbias_dtype, ch);
                if (ch % static_cast<int>(gridDim.x) == static_cast<int>(blockIdx.x)) {
                    // (spread over the grid: channel ch belongs to CTA ch % gridDim — CTA 0 alone used to be the last to finish)
                    // Σ_local dz = A (Σ_loc dy_m - n_loc mean_dy) + B Σ_loc (z - mean): the GPU-local totals come from the
                    // slice owners as packets (same tag), so no fence or barrier is involved; both are requested together
                    int fail = 0;
                    const unsigned long long to = prm.c.timeout_cycles ? prm.c.timeout_cycles : 4000000000ull;
                    const uint32_t tg = call_tag(prm.tag, prm.epoch);
                    const uint2 p1 = ld_packet_gpu(prm.w.locpk + (k * L + ll)), p3 = ld_packet_gpu(prm.w.locpk + ((16 + k) * L + ll));
                    const float s1 = (p1.y == tg) ? __uint_as_float(p1.x) : wait_packet_gpu(prm.w.locpk + (k * L + ll), tg, to, fail);
                    const float s3 = (p3.y == tg) ? __uint_as_float(p3.x) : wait_packet_gpu(prm.w.locpk + ((16 + k) * L + ll), tg, to, fail);
                    const float db = A * (s1 - static_cast<float>(g.rows) * mean_dy) + B * s3;
                    acc_bias_grad(prm.dcbias1, prm.cbias_dtype, ch, db);
                    acc_bias_grad(prm.dcbias2, prm.cbias_dtype, ch, db);
                    if (fail && prm.c.error_flag) atomicExch(prm.c.error_flag, 0xDEAD0003u);
                }
            }
            s_a[ch] = A;
            s_b[ch] = B;
            s_d[ch] = -A * mean_dy - B * mu;
        }
    }
    cbar();

    // ---- phase 2: dz = A dy_m + B z + D ; dres = dy_m ----------------------------------------------------------
    float A[8], B[8], D[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        A[k] = s_a[l * 8 + k];
        B[k] = s_b[l * 8 + k];
        D[k] = s_d[l * 8 + k];
    }
    const int nresident = sp.n - nres0;
    for (int u = 0; u < sp.n; ++u) {
        const bool streamed = u >= nresident;
        const int c = streamed ? nres0 - 1 - (u - nresident) : nres0 + u;
        const int kload = sp.n + (u - nresident);
        const int s = streamed ? kload % NS : (nres0 + u) % NS;
        if (streamed) ring.wait_full(s);
        const long long chunk = sp.chunk0 + c;
        const int npk = chunk_rows_of(g, chunk) * L;
        const size_t ebase = static_cast<size_t>(chunk) * g.chunk_rows * C;
        for (int q = tid; q < npk; q += kThreads) {
            float d[8], z[8];
            load_packet(s, q, d, z);
            if (gdres) {
                if (HINT) store8_hint(gdres + ebase + static_cast<size_t>(q) * 8, d, prm.store_policy);
                else IO<T>::store8(gdres + ebase + static_cast<size_t>(q) * 8, d);
            }
            float o[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = fmaf(A[k], d[k], fmaf(B[k], z[k], D[k]));
            if (HINT) store8_hint(gdz + ebase + static_cast<size_t>(q) * 8, o, prm.store_policy);
            else IO<T>::store8(gdz + ebase + static_cast<size_t>(q) * 8, o);
        }
        const int stage_load = streamed ? kload : nres0 + u;
        if (stage_load + NS < total_loads) ring.release(s);
    }
    stamp(prm.w, 3);
}

// ---- host side ------------------------------------------------------------------------------------------
static int make_geom(int64_t rows, int C, int dtype, int nstream, BnGeom& g, int max_chunk = 32768) {
    // tools/membench.cu: a bulk-copy ring delivers ∝ bytes per chunk iteration (a fixed cost per iteration), so
    // small stages leave bandwidth unused.  So: the largest power-of-two chunk per stream with nstream*chunk <= 48 KB.
    int chunk_bytes = max_chunk;
    while (nstream * chunk_bytes > 49152) chunk_bytes >>= 1;
    if (rows <= 0 || C <= 0 || (C % 8) != 0 || C > kMaxC) return SOD_EUNSUPPORTED;
    g.C = C;
    g.rows = rows;
    g.es = (dtype == SOD_F32) ? 4 : 2;
    g.L = C / 8;
    if ((g.L & (g.L - 1)) || g.L > 256) return SOD_EUNSUPPORTED;  // lanes per row: power of two ≤ 256
    while (C * g.es > chunk_bytes) chunk_bytes *= 2;                // a chunk holds at least one row
    g.chunk_bytes = chunk_bytes;
    g.chunk_rows = chunk_bytes / (C * g.es);
    const int ppc = chunk_bytes / (8 * g.es);                       // packets per chunk
    g.ppt = (ppc + kThreads - 1) / kThreads;
    g.nstream = nstream;
    const DevInfo& dv = dev_info();
    const long long budget = static_cast<long long>(dv.max_smem_optin) - kSmemFixed - 1024;
    int nstage = static_cast<int>(budget / (static_cast<long long>(nstream) * chunk_bytes));
    if (nstage > kMaxStages) nstage = kMaxStages;
    if (nstage < 2) return SOD_EUNSUPPORTED;
    g.nstage = nstage;
    g.total_chunks = (rows + g.chunk_rows - 1) / g.chunk_rows;
    long long strips = g.total_chunks;
    long long cap = dv.sm_count < kMaxGrid ? dv.sm_count : kMaxGrid;
    // hop-1 packets cost strips*2C*8 bytes of traffic: keep that well below the tensor itself
    const long long tensor_bytes = rows * C * g.es;
    static const long long traffic_div = [] {          // experiment knob: SOD_BN_TRAFFIC_DIV, default 4
        const char* e = getenv("SOD_BN_TRAFFIC_DIV");
        const long long v = e ? atoll(e) : 4;
        return v >= 1 ? v : 4;
    }();
    long long by_traffic = tensor_bytes / (traffic_div * 2 * C * 8);
    if (by_traffic < 1) by_traffic = 1;
    if (cap > by_traffic) cap = by_traffic;
    if (strips > cap) strips = cap;
    g.chunks_per_strip = static_cast<int>((g.total_chunks + strips - 1) / strips);
    g.strips = static_cast<int>((g.total_chunks + g.chunks_per_strip - 1) / g.chunks_per_strip);
    return SOD_OK;
}

static size_t bn_ws_layout(int C, BnWork* w, void* base) {
    size_t off = 0;
    if (w) w->ll_local = reinterpret_cast<uint2*>(static_cast<char*>(base) + off);
    off += static_cast<size_t>(2) * kMaxC * sizeof(uint2);
    if (w) w->locpk = reinterpret_cast<uint2*>(static_cast<char*>(base) + off);
    off += static_cast<size_t>(3) * kMaxC * sizeof(uint2);
    if (w) w->partials = reinterpret_cast<uint2*>(static_cast<char*>(base) + off);
    off += static_cast<size_t>(kMaxGrid) * 3 * C * sizeof(uint2);
    if (w) w->stamps = nullptr;
    return off;
}

// Every CTA spins on packets written by the other CTAs of the grid, so the whole grid has to be resident at once.
// Geometry guarantees grid ≤ #SMs at one CTA per SM; what it cannot guarantee is that nothing else holds an SM.
//   SOD_BN_LAUNCH_COOP : cooperative launch — the driver itself guarantees co-residency (or fails the launch) even
//                        next to a concurrent kernel on another stream / under MPS / under a profiler replay;
//   SOD_BN_LAUNCH_PDL  : programmatic dependent launch — the grid may be scheduled while the producing kernel drains;
//                        the kernels execute griddepcontrol.wait before their first global read.
// Independent of the mode, the launch is refused (SOD_EUNSUPPORTED) when the occupancy calculator says the kernel
// cannot have one CTA per SM with the requested shared memory.
template <typename K>
static int launch_bn(K kern, const void* prm, const BnGeom& g, int nstream, int flags, cudaStream_t stream) {
    const size_t smem = kSmemFixed + static_cast<size_t>(g.nstage) * nstream * g.chunk_bytes;
    static thread_local const void* configured[64] = {nullptr};   // per kernel instantiation, once per thread
    cudaError_t e;
    bool done = false;
    for (const void* c : configured) done |= (c == reinterpret_cast<const void*>(kern));
    if (!done) {
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dev_info().max_smem_optin - 1024);
        if (e != cudaSuccess) return static_cast<int>(e);
        int per_sm = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kBlock, dev_info().max_smem_optin - 1024);
        if (e != cudaSuccess) return static_cast<int>(e);
        if (per_sm < 1) return SOD_EUNSUPPORTED;
        for (auto& c : configured)
            if (c == nullptr) { c = reinterpret_cast<const void*>(kern); break; }
    }
    if (g.strips > dev_info().sm_count) return SOD_EUNSUPPORTED;
    void* args[] = {const_cast<void*>(prm)};
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(g.strips);
    cfg.blockDim = dim3(kBlock);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    unsigned na = 0;
    if (flags & SOD_BN_LAUNCH_COOP) {
        attr[na].id = cudaLaunchAttributeCooperative;
        attr[na].val.cooperative = 1;
        ++na;
    } else if (flags & SOD_BN_LAUNCH_PDL) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    e = cudaLaunchKernelExC(&cfg, reinterpret_cast<const void*>(kern), args);
    return static_cast<int>(e);
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_syncbn_workspace_bytes(int64_t rows, int channels) {
    (void)rows;
    return sod::bn_ws_layout(channels > 0 ? channels : sod::kMaxC, nullptr, nullptr);
}

extern "C" size_t sod_syncbn_exchange_bytes(int channels) {
    return static_cast<size_t>(SOD_MAX_WORLD) * 2u * channels * 8u;
}

extern "C" int sod_syncbn_fwd(const void* x, const void* pre_add, const void* residual, void* y, int dtype,
                              const float* gamma, const float* beta, float* running_mean, float* running_var,
                              float* save_mean, float* save_invstd, int64_t rows, int channels, float momentum,
                              float eps, int relu, int training, const sod_comm* comm, uint64_t stats_off,
                              uint32_t seq, const uint32_t* epoch, int64_t* num_batches_tracked, const void* conv_bias1,
                              const void* conv_bias2, int conv_bias_dtype, void* workspace, size_t workspace_bytes,
                              int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && y && gamma && beta && workspace, SOD_EINVAL);
    SOD_CHECK_ARG(training ? (save_mean && save_invstd) : (running_mean && running_var), SOD_EINVAL);
    SOD_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr), SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(x) && aligned16(y) && aligned16(workspace) && (!pre_add || aligned16(pre_add)) &&
                      (!residual || aligned16(residual)), SOD_EALIGN);
    if (dev_info().cc_major != 9) return SOD_EUNSUPPORTED;
    BnFwd p{};
    int rc = make_comm_dev(training ? comm : nullptr, p.c);
    if (rc != SOD_OK) return rc;
    if (p.c.world > 1) {
        SOD_CHECK_ARG((stats_off & 15) == 0, SOD_EALIGN);
        SOD_CHECK_ARG(stats_off >= sod_comm_flag_bytes() &&
                          stats_off + sod_syncbn_exchange_bytes(channels) <= comm->arena_bytes, SOD_ECOMM);
    }
    const int nstream = pre_add ? 2 : 1;
    // with a residual operand the kernel prefetches it through registers: keep that to 2 packets per thread
    rc = make_geom(rows, channels, dtype, nstream, p.g, residual ? 16384 : 32768);
    if (rc != SOD_OK) return rc;
    if (bn_ws_layout(channels, &p.w, workspace) > workspace_bytes) return SOD_EWORKSPACE;
    p.x = x; p.pre = pre_add; p.res = residual; p.y = y;
    p.gamma = gamma; p.beta = beta; p.rmean = running_mean; p.rvar = running_var;
    p.smean = save_mean; p.sinvstd = save_invstd;
    p.nbt = training ? reinterpret_cast<long long*>(num_batches_tracked) : nullptr;
    p.cbias1 = conv_bias1; p.cbias2 = conv_bias2; p.cbias_dtype = conv_bias_dtype;
    p.momentum = momentum; p.eps = eps; p.relu = relu; p.training = training;
    p.stats_off = stats_off; p.tag = seq; p.epoch = epoch;
    p.use_mc = (p.c.mc != 0) && !(flags & SOD_ALGO_NO_MULTIMEM);
    if ((flags & SOD_DEBUG_TIMING) && workspace_bytes >= bn_ws_layout(channels, nullptr, nullptr) + kMaxGrid * 64)
        p.w.stamps = reinterpret_cast<unsigned long long*>(static_cast<char*>(workspace) + bn_ws_layout(channels, nullptr, nullptr));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        const bool r = residual != nullptr;
        switch (p.g.ppt) {
            case 1: return r ? launch_bn(syncbn_fwd_kernel<T, 1, true>, &p, p.g, nstream, flags, s) : launch_bn(syncbn_fwd_kernel<T, 1, false>, &p, p.g, nstream, flags, s);
            case 2: return r ? launch_bn(syncbn_fwd_kernel<T, 2, true>, &p, p.g, nstream, flags, s) : launch_bn(syncbn_fwd_kernel<T, 2, false>, &p, p.g, nstream, flags, s);
            case 4: return r ? static_cast<int>(SOD_EUNSUPPORTED) : launch_bn(syncbn_fwd_kernel<T, 4, false>, &p, p.g, nstream, flags, s);
            default: return static_cast<int>(SOD_EUNSUPPORTED);
        }
    });
}

extern "C" int sod_syncbn_bwd(const void* dy, const void* x, const void* pre_add, const void* y, void* dz, void* dres,
                              int dtype, const float* gamma, const float* beta, const float* save_mean,
                              const float* save_invstd, float* dgamma, float* dbeta, int64_t rows, int channels, int relu,
                              const sod_comm* comm,
                              uint64_t stats_off, uint32_t seq, const uint32_t* epoch, const void* conv_bias1,
                              const void* conv_bias2, void* dconv_bias1, void* dconv_bias2, int conv_bias_dtype,
                              void* workspace, size_t workspace_bytes, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && x && dz && gamma && save_mean && save_invstd && dgamma && dbeta && workspace, SOD_EINVAL);
    // experimental: ReLU mask from x instead of y — only for BN+ReLU without a residual operand
    const bool xmask = (flags & SOD_BN_BWD_MASK_FROM_X) != 0;
    SOD_CHECK_ARG(!xmask || (relu && !dres && beta), SOD_EINVAL);
    SOD_CHECK_ARG(!relu || y || xmask, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(dy) && aligned16(x) && aligned16(dz) && aligned16(workspace) &&
                      (!pre_add || aligned16(pre_add)) && (!y || aligned16(y)) && (!dres || aligned16(dres)), SOD_EALIGN);
    if (dev_info().cc_major != 9) return SOD_EUNSUPPORTED;
    BnBwd p{};
    int rc = make_comm_dev(comm, p.c);
    if (rc != SOD_OK) return rc;
    if (p.c.world > 1) {
        SOD_CHECK_ARG((stats_off & 15) == 0, SOD_EALIGN);
        SOD_CHECK_ARG(stats_off >= sod_comm_flag_bytes() &&
                          stats_off + sod_syncbn_exchange_bytes(channels) <= comm->arena_bytes, SOD_ECOMM);
    }
    const int nstream = 2 + (pre_add ? 1 : 0) + ((relu && !xmask) ? 1 : 0);
    rc = make_geom(rows, channels, dtype, nstream, p.g);
    if (rc != SOD_OK) return rc;
    if (bn_ws_layout(channels, &p.w, workspace) > workspace_bytes) return SOD_EWORKSPACE;
    p.dy = dy; p.x = x; p.pre = pre_add; p.y = (relu && !xmask) ? y : nullptr; p.dz = dz; p.dres = dres;
    p.beta = beta;
    {   // HINT: a layer whose operands cannot all sit in L2 anyway writes its outputs evict-first, so that the part of the
        // strip phase 2 still has to fetch is not pushed out by them; a small layer keeps its outputs for the consumer
        const long long footprint = static_cast<long long>(rows) * channels * (dtype == SOD_F32 ? 4 : 2) * (nstream + 1 + (dres ? 1 : 0));
        p.store_policy = footprint > static_cast<long long>(dev_info().l2_bytes) * 3 / 4 ? kL2EvictFirst : kL2EvictNormal;
    }
    p.gamma = gamma; p.smean = save_mean; p.sinvstd = save_invstd; p.dgamma = dgamma; p.dbeta = dbeta;
    p.relu = relu; p.stats_off = stats_off; p.tag = seq; p.epoch = epoch;
    p.accumulate = (flags & SOD_BN_ACCUMULATE_PARAM_GRADS) ? 1 : 0;
    p.cbias1 = conv_bias1; p.cbias2 = conv_bias2; p.dcbias1 = dconv_bias1; p.dcbias2 = dconv_bias2; p.cbias_dtype = conv_bias_dtype;
    const bool fold = conv_bias1 != nullptr || conv_bias2 != nullptr;
    p.use_mc = (p.c.mc != 0) && !(flags & SOD_ALGO_NO_MULTIMEM);
    if ((flags & SOD_DEBUG_TIMING) && workspace_bytes >= bn_ws_layout(channels, nullptr, nullptr) + kMaxGrid * 64)
        p.w.stamps = reinterpret_cast<unsigned long long*>(static_cast<char*>(workspace) + bn_ws_layout(channels, nullptr, nullptr));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        if (flags & SOD_BN_L2_HINTS) {
            if (xmask)
                return fold ? launch_bn(syncbn_bwd_kernel<T, 24, true, true>, &p, p.g, nstream, flags, s)
                            : launch_bn(syncbn_bwd_kernel<T, 16, true, true>, &p, p.g, nstream, flags, s);
            return fold ? launch_bn(syncbn_bwd_kernel<T, 24, false, true>, &p, p.g, nstream, flags, s)
                        : launch_bn(syncbn_bwd_kernel<T, 16, false, true>, &p, p.g, nstream, flags, s);
        }
        if (xmask)
            return fold ? launch_bn(syncbn_bwd_kernel<T, 24, true>, &p, p.g, nstream, flags, s)
                        : launch_bn(syncbn_bwd_kernel<T, 16, true>, &p, p.g, nstream, flags, s);
        return fold ? launch_bn(syncbn_bwd_kernel<T, 24>, &p, p.g, nstream, flags, s) : launch_bn(syncbn_bwd_kernel<T, 16>, &p, p.g, nstream, flags, s);
    });
}
