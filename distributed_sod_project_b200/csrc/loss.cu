// loss.cu — BCE-with-logits + CEL, forward and backward in ONE persistent kernel.
//
// Reference arithmetic: torch.nn.BCEWithLogitsLoss (reference train.py:203) + CEL.forward
// (reference loss/CEL.py:15-20) summed by get_total_loss (reference utils/pipeline_ops.py:37-42).
//
// The CEL gradient of every pixel needs three sums over the WHOLE tensor (Σp, Σt, Σd), so a plain
// elementwise kernel cannot emit gradients in the pass that reads the logits.  Design:
//   * one CTA per SM (cooperative launch), each owning a contiguous slice of the tensor;
//   * the slice is pulled into shared memory with 1-D bulk async copies (TMA engine, mbarrier
//     completion) in 4096-element chunks so compute on chunk 0 overlaps the arrival of chunk k;
//   * phase 1 reduces (Σbce, Σp, Σt, Σd) from shared memory (d: see Sums) → per-CTA partial → grid barrier →
//     every CTA re-reduces the per-CTA partials (one per SM) in the same fixed order (deterministic, no atomics);
//   * phase 2 re-reads the slice FROM SHARED MEMORY and writes the gradient: logits and mask cross
//     HBM exactly once (8 B/elem algorithmic with bf16 logits + fp32 mask + bf16 grad).
// Slices larger than the shared-memory window (≈36 K elements per CTA, 4.8 M per launch on 132 SMs) take loss_stream_kernel
// below: the slice flows through a shared-memory ring fed by a producer warp, and phase 2 re-streams what did not stay
// resident (newest first, L2 eviction hints).
#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 512;
constexpr int kChunk = 4096;      // elements per staged chunk = kThreads * 8
constexpr int kMaxResident = 12;  // mbarriers reserved
constexpr int kMaxGrid = 1024;    // partial slots in the workspace

struct LossParams {
    const void* x;
    const void* m;
    void* g;
    float* scalars;
    float4* partials;
    long long n;
    long long per_cta;  // multiple of 8
    int resident;       // chunks held in shared memory per CTA
    int reduction_sum;
    float w_bce, w_cel, grad_scale, eps;
};

// d = p(1-t) + t(1-p) = |p - t| for a binary t: CEL's numerator term.  It is summed as such, never formed as
// Σp + Σt - 2Σpt, which cancels when the predictions are confident and p ≈ t (late in training).
struct Sums {
    float bce, p, t, d;
};

// p = sigmoid(x) and q = 1 - p, each from e = exp(-|x|) without a subtraction (1 - p loses q when q < ulp(1)); returns e
__device__ __forceinline__ float sigmoid_pq(float x, float& p, float& q) {
    const float e = __expf(-fabsf(x));
    const float r = __fdividef(1.0f, 1.0f + e);
    p = x >= 0.0f ? r : e * r;
    q = x >= 0.0f ? e * r : r;
    return e;
}

__device__ __forceinline__ void loss_terms(float x, float t, Sums& s) {
    float p, q;
    const float e = sigmoid_pq(x, p, q);
    // log1pf, not __logf(1 + e): that is off by up to 2^-21.4 absolute, 1 % of the whole term at |x| = 10
    s.bce += fmaxf(x, 0.0f) - x * t + log1pf(e);
    s.p += p;
    s.t += t;
    s.d += fmaf(p, 1.0f - t, t * q);
}

__device__ __forceinline__ float loss_grad(float x, float t, float kb, float alpha, float beta) {
    float p, q;
    sigmoid_pq(x, p, q);
    // kb*(p - t) + p(1-p) * ((1-2t)*alpha + beta); alpha/beta already carry w_cel*grad_scale.  p - t and 1 - p are
    // subtractions, as in the reference's autograd (sigmoid(x) - t): one fp32 ulp of 1 absolute.  Forming them from q
    // instead rounds every gradient differently, and a training run drifts away from the reference's trajectory.
    return kb * (p - t) + p * (1.0f - p) * fmaf(1.0f - 2.0f * t, alpha, beta);
}

template <typename TX, typename TM>
__global__ void __launch_bounds__(kThreads, 1) loss_bce_cel_kernel(const LossParams prm) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);  // kMaxResident barriers (128 B reserved)
    TX* sx = reinterpret_cast<TX*>(smem_raw + 128);
    TM* sm = reinterpret_cast<TM*>(smem_raw + 128 + static_cast<size_t>(prm.resident) * kChunk * sizeof(TX));
    __shared__ float s_red[kThreads / 32][4];
    __shared__ double s_tot[4];

    const TX* __restrict__ gx = static_cast<const TX*>(prm.x);
    const TM* __restrict__ gm = static_cast<const TM*>(prm.m);
    TX* __restrict__ gg = static_cast<TX*>(prm.g);

    const int tid = threadIdx.x;
    const long long n = prm.n;
    const long long nvec = n & ~7ll;  // the 16-byte-packet part; [nvec, n) is a scalar tail on CTA 0
    long long e0 = static_cast<long long>(blockIdx.x) * prm.per_cta;
    long long e1 = e0 + prm.per_cta;
    if (e0 > nvec) e0 = nvec;
    if (e1 > nvec) e1 = nvec;
    const int nchunks = static_cast<int>((e1 - e0 + kChunk - 1) / kChunk);
    const int nres = nchunks < prm.resident ? nchunks : prm.resident;

    // ---- stage: kick off every resident chunk's bulk copy up front --------------------------------
    if (tid == 0) {
        for (int c = 0; c < nres; ++c) mbar_init(&bars[c], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        for (int c = 0; c < nres; ++c) {
            const long long base = e0 + static_cast<long long>(c) * kChunk;
            const uint32_t cnt = static_cast<uint32_t>((e1 - base) < kChunk ? (e1 - base) : kChunk);
            mbar_arrive_expect_tx(&bars[c], cnt * static_cast<uint32_t>(sizeof(TX) + sizeof(TM)));
            bulk_g2s(sx + static_cast<size_t>(c) * kChunk, gx + base, cnt * static_cast<uint32_t>(sizeof(TX)), &bars[c]);
            bulk_g2s(sm + static_cast<size_t>(c) * kChunk, gm + base, cnt * static_cast<uint32_t>(sizeof(TM)), &bars[c]);
        }
    }

    // ---- phase 1: partial sums -----------------------------------------------------------------------
    Sums acc{0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < nchunks; ++c) {
        const long long base = e0 + static_cast<long long>(c) * kChunk;
        const int cnt = static_cast<int>((e1 - base) < kChunk ? (e1 - base) : kChunk);
        const TX* xs;
        const TM* ms;
        if (c < nres) {
            mbar_wait(&bars[c], 0);
            xs = sx + static_cast<size_t>(c) * kChunk;
            ms = sm + static_cast<size_t>(c) * kChunk;
        } else {
            xs = gx + base;
            ms = gm + base;
        }
        const int i = tid * 8;
        if (i < cnt) {
            float xv[8], tv[8];
            IO<TX>::load8(xs + i, xv);
            IO<TM>::load8(ms + i, tv);
#pragma unroll
            for (int k = 0; k < 8; ++k) loss_terms(xv[k], tv[k], acc);
        }
    }
    const int ntail = static_cast<int>(n - nvec);
    if (blockIdx.x == 0 && tid < ntail)
        loss_terms(IO<TX>::load1(gx + nvec + tid), IO<TM>::load1(gm + nvec + tid), acc);

    // block reduce (fixed order) → one partial per CTA
    {
        const float a = warp_sum(acc.bce), b = warp_sum(acc.p), c2 = warp_sum(acc.t), d = warp_sum(acc.d);
        if ((tid & 31) == 0) {
            s_red[tid >> 5][0] = a; s_red[tid >> 5][1] = b; s_red[tid >> 5][2] = c2; s_red[tid >> 5][3] = d;
        }
        __syncthreads();
        if (tid == 0) {
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int w = 0; w < kThreads / 32; ++w) {
                o.x += s_red[w][0]; o.y += s_red[w][1]; o.z += s_red[w][2]; o.w += s_red[w][3];
            }
            prm.partials[blockIdx.x] = o;
        }
    }
    cg::this_grid().sync();

    // ---- every CTA reduces all partials in the same order (double) ---------------------------------
    if (tid < 32) {
        double a = 0, b = 0, c2 = 0, d = 0;
        for (int i = tid; i < static_cast<int>(gridDim.x); i += 32) {
            const float4 v = prm.partials[i];
            a += v.x; b += v.y; c2 += v.z; d += v.w;
        }
        a = warp_sum(a); b = warp_sum(b); c2 = warp_sum(c2); d = warp_sum(d);
        if (tid == 0) { s_tot[0] = a; s_tot[1] = b; s_tot[2] = c2; s_tot[3] = d; }
    }
    __syncthreads();
    const double bce_sum = s_tot[0], sp = s_tot[1], st = s_tot[2], num = s_tot[3];
    const double spt = 0.5 * (sp + st - num);   // reported only: Σp·t = (Σp + Σt - Σd) / 2
    const double den = sp + st + static_cast<double>(prm.eps);
    const double cel = num / den;
    const double bce = prm.reduction_sum ? bce_sum : bce_sum / static_cast<double>(n);
    if (blockIdx.x == 0 && tid == 0) {
        float* o = prm.scalars;
        o[0] = static_cast<float>(bce);
        o[1] = static_cast<float>(cel);
        o[2] = static_cast<float>(prm.w_bce * bce + prm.w_cel * cel);
        o[3] = static_cast<float>(sp);
        o[4] = static_cast<float>(st);
        o[5] = static_cast<float>(spt);
        o[6] = static_cast<float>(bce_sum);
        o[7] = static_cast<float>(n);
    }
    // d total/dx = kb (p-t) + w_cel gs p(1-p) [ (1-2t)/den - num/den^2 ]
    const float kb = prm.grad_scale * prm.w_bce * (prm.reduction_sum ? 1.0f : static_cast<float>(1.0 / static_cast<double>(n)));
    const float alpha = static_cast<float>(static_cast<double>(prm.grad_scale) * prm.w_cel / den);
    const float beta = static_cast<float>(-static_cast<double>(prm.grad_scale) * prm.w_cel * num / (den * den));

    // ---- phase 2: gradients, re-reading the slice from shared memory --------------------------------
    for (int c = 0; c < nchunks; ++c) {
        const long long base = e0 + static_cast<long long>(c) * kChunk;
        const int cnt = static_cast<int>((e1 - base) < kChunk ? (e1 - base) : kChunk);
        const TX* xs = (c < nres) ? sx + static_cast<size_t>(c) * kChunk : gx + base;
        const TM* ms = (c < nres) ? sm + static_cast<size_t>(c) * kChunk : gm + base;
        const int i = tid * 8;
        if (i < cnt) {
            float xv[8], tv[8], gv[8];
            IO<TX>::load8(xs + i, xv);
            IO<TM>::load8(ms + i, tv);
#pragma unroll
            for (int k = 0; k < 8; ++k) gv[k] = loss_grad(xv[k], tv[k], kb, alpha, beta);
            IO<TX>::store8(gg + base + i, gv);
        }
    }
    if (blockIdx.x == 0 && tid < ntail) {
        const float x = IO<TX>::load1(gx + nvec + tid), t = IO<TM>::load1(gm + nvec + tid);
        IO<TX>::store1(gg + nvec + tid, loss_grad(x, t, kb, alpha, beta));
    }
}

// ------------------------------------------------------------------------------------------------
// streaming variant for tensors larger than the resident window (SURVEY §8d's scaled shape [64,1,1024,1024]):
// the slice flows through a shared-memory ring fed by a dedicated producer warp (same scheme as csrc/syncbn.cu):
// phase 1 consumes every chunk once, the last `nstage` chunks stay resident; after the grid barrier phase 2 takes the
// resident chunks first and re-streams the rest newest-first (the likeliest L2 hits), with L2 eviction hints:
// evict-last for chunks that will be fetched again, evict-first for every last use.
// ------------------------------------------------------------------------------------------------
constexpr int kStreamBlock = kThreads + 32;
constexpr int kMaxStreamStages = 12;

struct StreamRing {
    uint64_t* full;
    uint64_t* empty;
    uint32_t full_par, empty_par;
    __device__ __forceinline__ void wait_full(int s) { mbar_wait(&full[s], (full_par >> s) & 1u); full_par ^= 1u << s; }
    __device__ __forceinline__ void wait_empty(int s) { mbar_wait(&empty[s], (empty_par >> s) & 1u); empty_par ^= 1u << s; }
    __device__ __forceinline__ void release(int s) {
        __syncwarp();
        if ((threadIdx.x & 31) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(&empty[s])) : "memory");
    }
};

template <typename TX, typename TM>
__global__ void __launch_bounds__(kStreamBlock, 1) loss_stream_kernel(const LossParams prm) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);          // full[12] | empty[12] (256 B reserved)
    const int NS = prm.resident;                                     // stages of the ring
    constexpr size_t kStage = static_cast<size_t>(kChunk) * (sizeof(TX) + sizeof(TM));
    unsigned char* stages = smem_raw + 256;
    __shared__ float s_red[kThreads / 32][4];
    __shared__ double s_tot[4];

    const TX* __restrict__ gx = static_cast<const TX*>(prm.x);
    const TM* __restrict__ gm = static_cast<const TM*>(prm.m);
    TX* __restrict__ gg = static_cast<TX*>(prm.g);
    const int tid = threadIdx.x;
    const long long n = prm.n;
    const long long nvec = n & ~7ll;
    long long e0 = static_cast<long long>(blockIdx.x) * prm.per_cta;
    long long e1 = e0 + prm.per_cta;
    if (e0 > nvec) e0 = nvec;
    if (e1 > nvec) e1 = nvec;
    const int nchunks = static_cast<int>((e1 - e0 + kChunk - 1) / kChunk);
    const int nres0 = nchunks > NS ? nchunks - NS : 0;               // chunks [nres0, nchunks) stay resident after phase 1
    const int total_loads = nchunks + nres0;

    StreamRing ring{bars, bars + kMaxStreamStages, 0u, 0u};
    if (tid == 0) {
        for (int s = 0; s < NS; ++s) { mbar_init(&ring.full[s], 1); mbar_init(&ring.empty[s], kThreads / 32); }
        mbar_fence_init();
    }
    __syncthreads();
    auto sx_of = [&](int s) { return reinterpret_cast<TX*>(stages + static_cast<size_t>(s) * kStage); };
    auto sm_of = [&](int s) { return reinterpret_cast<TM*>(stages + static_cast<size_t>(s) * kStage + static_cast<size_t>(kChunk) * sizeof(TX)); };
    auto cnt_of = [&](int c) -> int {
        const long long base = e0 + static_cast<long long>(c) * kChunk;
        return static_cast<int>((e1 - base) < kChunk ? (e1 - base) : kChunk);
    };

    if (tid >= kThreads) {   // ---- producer warp --------------------------------------------------------------------
        if ((tid & 31) == 0) {
            for (int k = 0; k < total_loads; ++k) {
                if (k == nchunks) cg::this_grid().sync();            // phase-1 loads are all issued: join the grid barrier
                const int s = k % NS;
                if (k >= NS) ring.wait_empty(s);
                const int c = k < nchunks ? k : nres0 - 1 - (k - nchunks);
                const long long base = e0 + static_cast<long long>(c) * kChunk;
                const uint32_t cnt = static_cast<uint32_t>(cnt_of(c));
                const uint64_t policy = (k < nchunks && k < nres0) ? kL2EvictLast : kL2EvictFirst;
                mbar_arrive_expect_tx(&ring.full[s], cnt * static_cast<uint32_t>(sizeof(TX) + sizeof(TM)));
                bulk_g2s_hint(sx_of(s), gx + base, cnt * static_cast<uint32_t>(sizeof(TX)), &ring.full[s], policy);
                bulk_g2s_hint(sm_of(s), gm + base, cnt * static_cast<uint32_t>(sizeof(TM)), &ring.full[s], policy);
            }
            if (total_loads <= nchunks) cg::this_grid().sync();      // nothing to re-stream: the barrier was not met inside the loop
        } else {
            cg::this_grid().sync();
        }
        return;
    }

    // ---- phase 1 ---------------------------------------------------------------------------------------------------
    Sums acc{0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < nchunks; ++i) {
        const int s = i % NS;
        ring.wait_full(s);
        const int cnt = cnt_of(i);
        const int e = tid * 8;
        if (e < cnt) {
            float xv[8], tv[8];
            IO<TX>::load8(sx_of(s) + e, xv);
            IO<TM>::load8(sm_of(s) + e, tv);
#pragma unroll
            for (int k = 0; k < 8; ++k) loss_terms(xv[k], tv[k], acc);
        }
        if (i + NS < nchunks) ring.release(s);
    }
    const int ntail = static_cast<int>(n - nvec);
    if (blockIdx.x == 0 && tid < ntail)
        loss_terms(IO<TX>::load1(gx + nvec + tid), IO<TM>::load1(gm + nvec + tid), acc);
    {
        const float a = warp_sum(acc.bce), b = warp_sum(acc.p), c2 = warp_sum(acc.t), d = warp_sum(acc.d);
        if ((tid & 31) == 0) { s_red[tid >> 5][0] = a; s_red[tid >> 5][1] = b; s_red[tid >> 5][2] = c2; s_red[tid >> 5][3] = d; }
        asm volatile("bar.sync 1, 512;" ::: "memory");
        if (tid == 0) {
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int w = 0; w < kThreads / 32; ++w) { o.x += s_red[w][0]; o.y += s_red[w][1]; o.z += s_red[w][2]; o.w += s_red[w][3]; }
            prm.partials[blockIdx.x] = o;
        }
    }
    cg::this_grid().sync();
    if (tid < 32) {
        double a = 0, b = 0, c2 = 0, d = 0;
        for (int i = tid; i < static_cast<int>(gridDim.x); i += 32) {
            const float4 v = prm.partials[i];
            a += v.x; b += v.y; c2 += v.z; d += v.w;
        }
        a = warp_sum(a); b = warp_sum(b); c2 = warp_sum(c2); d = warp_sum(d);
        if (tid == 0) { s_tot[0] = a; s_tot[1] = b; s_tot[2] = c2; s_tot[3] = d; }
    }
    asm volatile("bar.sync 1, 512;" ::: "memory");
    const double bce_sum = s_tot[0], sp = s_tot[1], st = s_tot[2], num = s_tot[3];
    const double spt = 0.5 * (sp + st - num);   // reported only: Σp·t = (Σp + Σt - Σd) / 2
    const double den = sp + st + static_cast<double>(prm.eps);
    const double cel = num / den;
    const double bce = prm.reduction_sum ? bce_sum : bce_sum / static_cast<double>(n);
    if (blockIdx.x == 0 && tid == 0) {
        float* o = prm.scalars;
        o[0] = static_cast<float>(bce); o[1] = static_cast<float>(cel);
        o[2] = static_cast<float>(prm.w_bce * bce + prm.w_cel * cel);
        o[3] = static_cast<float>(sp); o[4] = static_cast<float>(st); o[5] = static_cast<float>(spt);
        o[6] = static_cast<float>(bce_sum); o[7] = static_cast<float>(n);
    }
    const float kb = prm.grad_scale * prm.w_bce * (prm.reduction_sum ? 1.0f : static_cast<float>(1.0 / static_cast<double>(n)));
    const float alpha = static_cast<float>(static_cast<double>(prm.grad_scale) * prm.w_cel / den);
    const float beta = static_cast<float>(-static_cast<double>(prm.grad_scale) * prm.w_cel * num / (den * den));

    // ---- phase 2: resident chunks first, then the re-streamed ones (newest first) ----------------------------------
    const int nresident = nchunks - nres0;
    for (int u = 0; u < nchunks; ++u) {
        const bool streamed = u >= nresident;
        const int c = streamed ? nres0 - 1 - (u - nresident) : nres0 + u;
        const int kload = nchunks + (u - nresident);
        const int s = streamed ? kload % NS : (nres0 + u) % NS;
        if (streamed) ring.wait_full(s);
        const long long base = e0 + static_cast<long long>(c) * kChunk;
        const int cnt = cnt_of(c);
        const int e = tid * 8;
        if (e < cnt) {
            float xv[8], tv[8], gv[8];
            IO<TX>::load8(sx_of(s) + e, xv);
            IO<TM>::load8(sm_of(s) + e, tv);
#pragma unroll
            for (int k = 0; k < 8; ++k) gv[k] = loss_grad(xv[k], tv[k], kb, alpha, beta);
            IO<TX>::store8(gg + base + e, gv);
        }
        const int stage_load = streamed ? kload : nres0 + u;
        if (stage_load + NS < total_loads) ring.release(s);
    }
    if (blockIdx.x == 0 && tid < ntail) {
        const float x = IO<TX>::load1(gx + nvec + tid), t = IO<TM>::load1(gm + nvec + tid);
        IO<TX>::store1(gg + nvec + tid, loss_grad(x, t, kb, alpha, beta));
    }
}

template <typename T>
__global__ void scale_by_scalar_kernel(T* g, long long n, const float* s) {
    const float sc = *s;
    const long long nv = n >> 3;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nv;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        float v[8];
        IO<T>::load8(g + i * 8, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] *= sc;
        IO<T>::store8(g + i * 8, v);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 7)) {
        T* p = g + (n & ~7ll) + threadIdx.x;
        IO<T>::store1(p, IO<T>::load1(p) * sc);
    }
}

template <typename TX, typename TM>
int launch_loss(LossParams& prm, int mode, cudaStream_t stream) {
    const DevInfo& dv = dev_info();
    auto kern = loss_bce_cel_kernel<TX, TM>;
    const size_t per_chunk = static_cast<size_t>(kChunk) * (sizeof(TX) + sizeof(TM));
    const size_t budget = static_cast<size_t>(dv.max_smem_optin) - 128 - 1024;  // barriers + static smem
    int resident = static_cast<int>(budget / per_chunk);
    if (resident > kMaxResident) resident = kMaxResident;
    if (mode == 2) resident = 0;

    long long grid = (prm.n + kChunk - 1) / kChunk;
    if (grid < 1) grid = 1;
    if (grid > dv.sm_count) grid = dv.sm_count;
    long long per_cta = (prm.n + grid - 1) / grid;
    per_cta = (per_cta + 7) & ~7ll;
    const int need = static_cast<int>((per_cta + kChunk - 1) / kChunk);
    if (resident > need) resident = need;
    if (mode == 1 && need > resident) return SOD_EUNSUPPORTED;  // caller demanded the single-read path

    prm.per_cta = per_cta;
    if (need > resident) {
        // larger than the resident window: the ring-streamed kernel (mode 2 = "streaming" selects it as well)
        auto skern = loss_stream_kernel<TX, TM>;
        int stages = static_cast<int>((static_cast<size_t>(dv.max_smem_optin) - 256 - 1024) / per_chunk);
        if (stages > kMaxStreamStages) stages = kMaxStreamStages;
        if (stages < 2) return SOD_EUNSUPPORTED;
        prm.resident = stages;
        const size_t ssmem = 256 + static_cast<size_t>(stages) * per_chunk;
        cudaError_t e = cudaFuncSetAttribute(skern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ssmem));
        if (e != cudaSuccess) return static_cast<int>(e);
        void* sargs[] = {&prm};
        e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(skern), dim3(static_cast<unsigned>(grid)), dim3(kStreamBlock), sargs,
                                        ssmem, stream);
        return static_cast<int>(e);
    }
    prm.resident = resident;
    const size_t smem = 128 + static_cast<size_t>(resident) * per_chunk;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return static_cast<int>(e);
    void* args[] = {&prm};
    e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kern), dim3(static_cast<unsigned>(grid)), dim3(kThreads), args,
                                    smem, stream);
    return static_cast<int>(e);
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_loss_workspace_bytes(void) { return sizeof(float4) * sod::kMaxGrid; }

extern "C" int sod_loss_bce_cel_fwd_bwd(const void* logits, int logits_dtype, const void* mask, int mask_dtype,
                                        void* grad_logits, int grad_dtype, float* scalars_out, int64_t n,
                                        int reduction_sum, float w_bce, float w_cel, float grad_scale, float eps,
                                        int mode, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(logits && mask && grad_logits && scalars_out && workspace, SOD_EINVAL);
    SOD_CHECK_ARG(n > 0 && mode >= 0 && mode <= 2, SOD_EINVAL);
    SOD_CHECK_ARG(grad_dtype == logits_dtype, SOD_EUNSUPPORTED);
    SOD_CHECK_ARG(mask_dtype == SOD_F32 || mask_dtype == logits_dtype, SOD_EUNSUPPORTED);
    SOD_CHECK_ARG(aligned16(logits) && aligned16(mask) && aligned16(grad_logits) && aligned16(workspace), SOD_EALIGN);
    SOD_CHECK_ARG(workspace_bytes >= sod_loss_workspace_bytes(), SOD_EWORKSPACE);
    if (dev_info().cc_major != 9) return SOD_EUNSUPPORTED;

    LossParams prm{};
    prm.x = logits; prm.m = mask; prm.g = grad_logits; prm.scalars = scalars_out;
    prm.partials = static_cast<float4*>(workspace);
    prm.n = n; prm.reduction_sum = reduction_sum ? 1 : 0;
    prm.w_bce = w_bce; prm.w_cel = w_cel; prm.grad_scale = grad_scale; prm.eps = eps;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (logits_dtype) {
        case SOD_F32: return launch_loss<float, float>(prm, mode, s);
        case SOD_BF16:
            return mask_dtype == SOD_F32 ? launch_loss<__nv_bfloat16, float>(prm, mode, s)
                                         : launch_loss<__nv_bfloat16, __nv_bfloat16>(prm, mode, s);
        case SOD_F16:
            return mask_dtype == SOD_F32 ? launch_loss<__half, float>(prm, mode, s)
                                         : launch_loss<__half, __half>(prm, mode, s);
        default: return SOD_EINVAL;
    }
}

extern "C" int sod_scale_by_device_scalar(void* grad, int dtype, int64_t n, const float* scale_dev, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(grad && scale_dev && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(grad), SOD_EALIGN);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    long long blocks = ((n >> 3) + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > 4 * dev_info().sm_count) blocks = 4 * dev_info().sm_count;
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        scale_by_scalar_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, s>>>(static_cast<T*>(grad), n, scale_dev);
        return static_cast<int>(cudaGetLastError());
    });
}
