// sgd.cu — gradient all-reduce ⊕ unscale ⊕ SGD-momentum over flat fp32 buffers, plus the plain
// peer-memory all-reduce used by the bandwidth sweep.
//
// Reference arithmetic being replaced (paths relative to the reference repo):
//   apex DDP(delay_allreduce=True): flat SUM all-reduce then ×1/W            train.py:185
//   apex amp unscale ×1/S with overflow skip                                  train.py:299
//   torch.optim.SGD.step (momentum, wd folded into g, no nesterov/dampening)  train.py:303,
//       groups from make_optimizer("f3_trick")                                utils/pipeline_ops.py:295-313
//   optimizer.zero_grad                                                       train.py:297
//
// world == 1 : one streaming pass, 20 B/elem (read g,p,v; write p,v) [+4 B/elem to zero g].
// world  > 1 : two-shot over NVSwitch peer memory. Rank r owns shard r of the flat index space:
//     start barrier → reduce shard r across ranks (multimem.ld_reduce in the switch, or peer loads
//     summed in rank order) → unscale/÷W → SGD on (p,v) shard in registers → write the UPDATED
//     PARAMETERS to every rank (multimem.st / peer stores) → end barrier [→ zero local grads].
//   So what crosses NVLink is reduce-scatter(grads) + all-gather(params): the same bus bytes as an
//   all-reduce, but no separate NCCL call, no ÷W pass, no optimizer kernel, and momentum is only ever
//   touched on the owning rank (1/W of the optimizer-state traffic).
//   Owner-computes + broadcast also makes parameters bit-identical on all ranks by construction.
#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 512;
constexpr int kUnroll = 4;

struct SegTable {
    int n;
    long long begin[SOD_MAX_SEGMENTS], end[SOD_MAX_SEGMENTS];  // in float4 units
    float lr[SOD_MAX_SEGMENTS], wd[SOD_MAX_SEGMENTS], mu[SOD_MAX_SEGMENTS];
    int flags[SOD_MAX_SEGMENTS];
};

static int make_seg_table(const sod_sgd_segment* segs, int nseg, int64_t n, SegTable& t) {
    if (nseg < 0 || nseg > SOD_MAX_SEGMENTS || (nseg > 0 && segs == nullptr)) return SOD_EINVAL;
    t.n = nseg;
    long long prev = 0;
    for (int i = 0; i < nseg; ++i) {
        const sod_sgd_segment& s = segs[i];
        if (s.begin < prev || s.end < s.begin || s.end > n) return SOD_EINVAL;  // sorted, disjoint, in range
        if ((s.begin & 3) || (s.end & 3)) return SOD_EALIGN;
        t.begin[i] = s.begin >> 2; t.end[i] = s.end >> 2;
        t.lr[i] = s.lr; t.wd[i] = s.weight_decay; t.mu[i] = s.momentum; t.flags[i] = s.flags;
        prev = s.end;
    }
    return SOD_OK;
}

// segment cursor: indices visited by one thread only ever increase
// learning rate of segment s: from device memory when the host passed a table (a captured CUDA graph then follows
// the scheduler without being re-captured: reference utils/pipeline_ops.py:225-229 rewrites param_groups[i]["lr"]
// every epoch or every iteration), else the by-value copy
__device__ __forceinline__ float seg_lr(const SegTable& t, const float* lr_dev, int s) {
    return lr_dev != nullptr ? __ldg(lr_dev + s) : t.lr[s];
}

struct SegCursor {
    int s = 0;
    // segment containing `vec` (any kind), or false when it lies in a gap / behind the last segment
    __device__ __forceinline__ bool locate(const SegTable& t, long long vec) {
        while (s < t.n && vec >= t.end[s]) ++s;
        return s < t.n && vec >= t.begin[s];
    }
    __device__ __forceinline__ bool find(const SegTable& t, long long vec) {
        return locate(t, vec) && !(t.flags[s] & SOD_SEG_FROZEN);
    }
};

__device__ __forceinline__ void sgd_update(float4& p, float4& v, const float4& g, float lr, float wd, float mu) {
    // g' = g + wd*p ; v = mu*v + g' ; p = p - lr*v   (operation order of torch/optim/sgd.py:343-380)
    float gx = fmaf(wd, p.x, g.x), gy = fmaf(wd, p.y, g.y), gz = fmaf(wd, p.z, g.z), gw = fmaf(wd, p.w, g.w);
    v.x = fmaf(mu, v.x, gx); v.y = fmaf(mu, v.y, gy); v.z = fmaf(mu, v.z, gz); v.w = fmaf(mu, v.w, gw);
    p.x = fmaf(-lr, v.x, p.x); p.y = fmaf(-lr, v.y, p.y); p.z = fmaf(-lr, v.z, p.z); p.w = fmaf(-lr, v.w, p.w);
}

// ------------------------------------------------------------------------------------------------
// world == 1
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 bf16x4_to_f32(uint2 u) {
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
    const float2 a = __bfloat1622float2(h[0]), b = __bfloat1622float2(h[1]);
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ uint2 f32x4_to_bf16(const float4& f) {
    uint2 u;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
    h[0] = __floats2bfloat162_rn(f.x, f.y);
    h[1] = __floats2bfloat162_rn(f.z, f.w);
    return u;
}

__global__ void __launch_bounds__(kThreads) sgd_local_kernel(float4* __restrict__ p, float4* __restrict__ v,
                                                             float4* __restrict__ g, uint2* __restrict__ g16,
                                                             uint2* __restrict__ shadow, long long nvec,
                                                             const __grid_constant__ SegTable segs, float inv_scale,
                                                             const uint32_t* found_inf, int zero_grad,
                                                             const float* __restrict__ lr_dev) {
    const bool skip = (found_inf != nullptr && *found_inf != 0);  // amp overflow: no update, but still clear g
    SegCursor cur;
    const long long stride = static_cast<long long>(gridDim.x) * kThreads;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i0 = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i0 < nvec; i0 += stride * kUnroll) {
        float4 gv[kUnroll], pv[kUnroll], vv[kUnroll];
        int sidx[kUnroll];
        bool only16[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long i = i0 + u * stride;
            sidx[u] = -1;
            only16[u] = false;
            if (i < nvec) {
                const bool in_seg = cur.locate(segs, i);
                // SOD_SEG_GRAD16: the gradient of this range exists in bf16 only — the fp32 buffer is neither read nor cleared
                only16[u] = in_seg && g16 != nullptr && (segs.flags[cur.s] & SOD_SEG_GRAD16);
                if (only16[u]) {
                    gv[u] = bf16x4_to_f32(g16[i]);
                } else {
                    gv[u] = g[i];
                    if (g16 != nullptr) {   // gradients autograd left in bf16: fold them in here (the "cast" of amp O1)
                        const float4 h = bf16x4_to_f32(g16[i]);
                        gv[u].x += h.x; gv[u].y += h.y; gv[u].z += h.z; gv[u].w += h.w;
                    }
                }
                if (!skip && in_seg && !(segs.flags[cur.s] & SOD_SEG_FROZEN)) {
                    sidx[u] = cur.s;
                    pv[u] = p[i];
                    vv[u] = v[i];
                }
            }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long i = i0 + u * stride;
            if (i < nvec) {
                if (sidx[u] >= 0) {
                    const int s = sidx[u];
                    const float4 gs = make_float4(gv[u].x * inv_scale, gv[u].y * inv_scale, gv[u].z * inv_scale, gv[u].w * inv_scale);
                    sgd_update(pv[u], vv[u], gs, seg_lr(segs, lr_dev, s), segs.wd[s], segs.mu[s]);
                    p[i] = pv[u];
                    v[i] = vv[u];
                    if (shadow != nullptr) shadow[i] = f32x4_to_bf16(pv[u]);
                }
                if (zero_grad) {
                    if (!only16[u]) g[i] = zero;
                    if (g16 != nullptr) g16[i] = make_uint2(0u, 0u);
                }
            }
        }
    }
}

__global__ void grad_merge_bf16_kernel(float4* __restrict__ g, uint2* __restrict__ g16, long long nvec) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const uint2 raw = g16[i];
        if ((raw.x | raw.y) != 0u) {   // most of the flat buffer (BN parameters, padding) never sees a bf16 gradient
            float4 a = g[i];
            const float4 h = bf16x4_to_f32(raw);
            a.x += h.x; a.y += h.y; a.z += h.z; a.w += h.w;
            g[i] = a;
            g16[i] = make_uint2(0u, 0u);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// multi-tensor gather: the bf16 weight gradients autograd produced (one freshly allocated tensor per
// parameter) → the flat bf16 gradient buffer, ONE launch instead of one accumulate kernel per tensor
// ------------------------------------------------------------------------------------------------
constexpr int kGatherMax = SOD_GATHER_MAX_ITEMS;
constexpr int kGatherChunk = 8192;          // elements per work unit
struct GatherTable {
    int n;
    const void* src[kGatherMax];
    unsigned dst_off8[kGatherMax];          // destination offset in units of 8 elements
    unsigned numel[kGatherMax];
    unsigned chunk0[kGatherMax + 1];        // prefix sum of ceil(numel / kGatherChunk)
};

__global__ void __launch_bounds__(256) grad_gather16_kernel(const __grid_constant__ GatherTable t, uint4* __restrict__ dst) {
    const unsigned total = t.chunk0[t.n];
    for (unsigned c = blockIdx.x; c < total; c += gridDim.x) {
        int lo = 0, hi = t.n - 1;           // item with chunk0[item] <= c < chunk0[item+1]
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (t.chunk0[mid] <= c) lo = mid; else hi = mid - 1;
        }
        const unsigned first = (c - t.chunk0[lo]) * kGatherChunk;
        const unsigned left = t.numel[lo] - first;
        const unsigned cnt = left < kGatherChunk ? left : kGatherChunk;
        const unsigned short* src = static_cast<const unsigned short*>(t.src[lo]) + first;
        unsigned short* out = reinterpret_cast<unsigned short*>(dst + t.dst_off8[lo]) + first;
        if ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) {
            const uint4* s4 = reinterpret_cast<const uint4*>(src);
            uint4* d4 = reinterpret_cast<uint4*>(out);                 // dst offsets and chunk starts are multiples of 8
            const unsigned nv = cnt >> 3;
            for (unsigned i = threadIdx.x; i < nv; i += 256) d4[i] = __ldcs(s4 + i);
            for (unsigned i = (nv << 3) + threadIdx.x; i < cnt; i += 256) out[i] = src[i];
        } else {
            for (unsigned i = threadIdx.x; i < cnt; i += 256) out[i] = src[i];
        }
    }
}

__global__ void grad_nonfinite_kernel(const float4* __restrict__ g, long long nvec, uint32_t* found) {
    bool bad = false;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const float4 v = g[i];
        bad |= !(isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w));
    }
    if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(found, 1u);
}

// ------------------------------------------------------------------------------------------------
// world > 1 : fused reduce-scatter + SGD + parameter all-gather over peer memory
// ------------------------------------------------------------------------------------------------
template <bool kMulticast>
__device__ __forceinline__ float4 reduce_vec(const CommDev& c, uint64_t byte_off) {
    if constexpr (kMulticast) {
        return multimem_ld_reduce_add_f32x4(reinterpret_cast<const void*>(c.mc + byte_off));
    } else {
        float4 acc = ld_peer_f32x4(reinterpret_cast<const void*>(c.peer[0] + byte_off));
        for (int q = 1; q < c.world; ++q) {  // fixed rank order: every owner sums identically
            const float4 t = ld_peer_f32x4(reinterpret_cast<const void*>(c.peer[q] + byte_off));
            acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
        }
        return acc;
    }
}
template <bool kMulticast>
__device__ __forceinline__ void broadcast_vec(const CommDev& c, uint64_t byte_off, const float4& v) {
    if constexpr (kMulticast) {
        multimem_st_f32x4(reinterpret_cast<void*>(c.mc + byte_off), v);
    } else {
        for (int q = 0; q < c.world; ++q) st_peer_f32x4(reinterpret_cast<void*>(c.peer[q] + byte_off), v);
    }
}

// bf16 gradients on the wire: 4 elements = 8 bytes per rank, summed in fp32 in rank order (exact: no rounding of the sum,
// unlike a bf16 multimem reduction), so every owner obtains the same value it would from an fp32 exchange of the same data
__device__ __forceinline__ float4 reduce_vec16(const CommDev& c, uint64_t byte_off) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    uint2 raw[SOD_MAX_WORLD];
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) raw[q] = ld_relaxed_sys_v2(reinterpret_cast<const void*>(c.peer[q] + byte_off));
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) {
            const float4 t = bf16x4_to_f32(raw[q]);
            acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
        }
    return acc;
}

template <bool kMulticast>
__global__ void __launch_bounds__(kThreads) allreduce_sgd_kernel(const __grid_constant__ CommDev c, uint64_t grad_off,
                                                                 uint64_t param_off, float4* __restrict__ mom,
                                                                 long long nvec, const __grid_constant__ SegTable segs,
                                                                 float scale, const uint32_t* found_inf,
                                                                 int zero_grad, uint2* __restrict__ shadow,
                                                                 const float* __restrict__ lr_dev, uint64_t grad16_off,
                                                                 int has_grad16) {
    const bool skip = (found_inf != nullptr && *found_inf != 0);  // caller guarantees identical on all ranks
    // every rank's backward has finished writing its gradients
    if (!comm_block_barrier(c, 0, blockIdx.x)) return;

    const long long shard = (nvec + c.world - 1) / c.world;
    const long long stride = static_cast<long long>(gridDim.x) * kThreads;
    const long long lo = shard * c.rank;
    const long long hi = (lo + shard < nvec) ? lo + shard : nvec;
    float4* p_local = reinterpret_cast<float4*>(c.peer[c.rank] + param_off);

    if (!skip) {
        SegCursor cur;
        for (long long i0 = lo + static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i0 < hi; i0 += stride * kUnroll) {
            float4 gv[kUnroll];
            int sidx[kUnroll];
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const long long i = i0 + u * stride;
                sidx[u] = -1;
                if (i < hi && cur.find(segs, i)) {        // frozen ranges and gaps are never consumed: not even reduced
                    sidx[u] = cur.s;
                    if (has_grad16 && (segs.flags[cur.s] & SOD_SEG_GRAD16))
                        gv[u] = reduce_vec16(c, grad16_off + static_cast<uint64_t>(i) * 8u);
                    else
                        gv[u] = reduce_vec<kMulticast>(c, grad_off + static_cast<uint64_t>(i) * 16u);
                }
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const long long i = i0 + u * stride;
                if (sidx[u] >= 0) {
                    const int s = sidx[u];
                    float4 pv = p_local[i], vv = mom[i];
                    const float4 gs = make_float4(gv[u].x * scale, gv[u].y * scale, gv[u].z * scale, gv[u].w * scale);
                    sgd_update(pv, vv, gs, seg_lr(segs, lr_dev, s), segs.wd[s], segs.mu[s]);
                    mom[i] = vv;
                    broadcast_vec<kMulticast>(c, param_off + static_cast<uint64_t>(i) * 16u, pv);
                }
            }
        }
    }
    // every rank's parameter shard has landed everywhere (and every peer is done reading my gradients)
    if (!comm_block_barrier(c, 0, blockIdx.x)) return;

    if (zero_grad || shadow != nullptr) {
        // this block's peers read / wrote exactly the vectors {q*shard + blockIdx*kThreads + t + k*stride}: after the
        // barrier it is safe to clear those gradients, and the parameters that landed there are final — refresh the
        // local bf16 shadow from them
        float4* g_local = reinterpret_cast<float4*>(c.peer[c.rank] + grad_off);
        uint2* g16_local = has_grad16 ? reinterpret_cast<uint2*>(c.peer[c.rank] + grad16_off) : nullptr;
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int q = 0; q < c.world; ++q) {
            const long long qlo = shard * q;
            const long long qhi = (qlo + shard < nvec) ? qlo + shard : nvec;
            SegCursor cur;                                   // indices restart for every shard
            for (long long i = qlo + static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i < qhi; i += stride) {
                const bool in_seg = cur.locate(segs, i);
                const bool only16 = in_seg && has_grad16 && (segs.flags[cur.s] & SOD_SEG_GRAD16);
                if (zero_grad) {
                    if (!only16) g_local[i] = zero;
                    if (g16_local != nullptr) g16_local[i] = make_uint2(0u, 0u);
                }
                if (shadow != nullptr && !skip) shadow[i] = f32x4_to_bf16(p_local[i]);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// plain all-reduce (bandwidth sweep; scalar loss mean)
// ------------------------------------------------------------------------------------------------
template <bool kMulticast>
__global__ void __launch_bounds__(kThreads) allreduce_two_shot_kernel(const __grid_constant__ CommDev c, uint64_t off,
                                                                      long long nvec, float scale) {
    if (!comm_block_barrier(c, 3, blockIdx.x)) return;
    const long long shard = (nvec + c.world - 1) / c.world;
    const long long stride = static_cast<long long>(gridDim.x) * kThreads;
    const long long lo = shard * c.rank;
    const long long hi = (lo + shard < nvec) ? lo + shard : nvec;
    for (long long i0 = lo + static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i0 < hi; i0 += stride * kUnroll) {
        float4 v[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long i = i0 + u * stride;
            if (i < hi) v[u] = reduce_vec<kMulticast>(c, off + static_cast<uint64_t>(i) * 16u);
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const long long i = i0 + u * stride;
            if (i < hi) {
                v[u].x *= scale; v[u].y *= scale; v[u].z *= scale; v[u].w *= scale;
                broadcast_vec<kMulticast>(c, off + static_cast<uint64_t>(i) * 16u, v[u]);
            }
        }
    }
    comm_block_barrier(c, 3, blockIdx.x);
}

// one-shot: every rank reads every peer's whole buffer and keeps the sum locally (latency-optimal for
// small messages). In place is safe because results are written only after the mid barrier.
__global__ void __launch_bounds__(kThreads) allreduce_one_shot_kernel(const __grid_constant__ CommDev c, uint64_t off,
                                                                      long long nvec, float scale) {
    if (!comm_block_barrier(c, 3, blockIdx.x)) return;
    const long long stride = static_cast<long long>(gridDim.x) * kThreads;
    const long long first = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
    // the host sizes the grid so that each thread owns at most kUnroll vectors → results stay in registers
    float4 acc[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
        const long long i = first + u * stride;
        if (i < nvec) {
            acc[u] = reduce_vec<false>(c, off + static_cast<uint64_t>(i) * 16u);
            acc[u].x *= scale; acc[u].y *= scale; acc[u].z *= scale; acc[u].w *= scale;
        }
    }
    if (!comm_block_barrier(c, 3, blockIdx.x)) return;  // everyone has finished reading
    float4* local = reinterpret_cast<float4*>(c.peer[c.rank] + off);
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
        const long long i = first + u * stride;
        if (i < nvec) local[i] = acc[u];
    }
}

static unsigned comm_grid(long long vecs_per_rank) {
    long long blocks = (vecs_per_rank + static_cast<long long>(kThreads) * kUnroll - 1) / (static_cast<long long>(kThreads) * kUnroll);
    const long long cap = dev_info().sm_count < SOD_COMM_MAX_BLOCKS ? dev_info().sm_count : SOD_COMM_MAX_BLOCKS;
    if (blocks < 1) blocks = 1;
    if (blocks > cap) blocks = cap;
    return static_cast<unsigned>(blocks);
}

}  // namespace
}  // namespace sod

extern "C" int sod_sgd_momentum(float* param, float* mom, float* grad, void* grad16, void* shadow16, int64_t n,
                                const sod_sgd_segment* segs, int nseg, const float* lr_dev, float inv_scale,
                                const uint32_t* found_inf, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(param && mom && grad && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && aligned16(param) && aligned16(mom) && aligned16(grad), SOD_EALIGN);
    SOD_CHECK_ARG((!grad16 || aligned16(grad16)) && (!shadow16 || aligned16(shadow16)), SOD_EALIGN);
    SegTable t;
    int rc = make_seg_table(segs, nseg, n, t);
    if (rc != SOD_OK) return rc;
    const long long nvec = n >> 2;
    long long blocks = (nvec + static_cast<long long>(kThreads) * kUnroll - 1) / (static_cast<long long>(kThreads) * kUnroll);
    const long long cap = 2ll * dev_info().sm_count;
    if (blocks > cap) blocks = cap;
    sgd_local_kernel<<<static_cast<unsigned>(blocks), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<float4*>(param), reinterpret_cast<float4*>(mom), reinterpret_cast<float4*>(grad),
        reinterpret_cast<uint2*>(grad16), reinterpret_cast<uint2*>(shadow16), nvec, t, inv_scale, found_inf,
        (flags & SOD_SGD_ZERO_GRAD) ? 1 : 0, lr_dev);
    return static_cast<int>(cudaGetLastError());
}

extern "C" int sod_grad_gather16(const sod_gather_item* items, int nitems, void* dst16, int64_t dst_elems, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(nitems >= 0 && (nitems == 0 || items) && dst16 && dst_elems > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(dst16), SOD_EALIGN);
    for (int base = 0; base < nitems; base += kGatherMax) {
        GatherTable t;
        t.n = (nitems - base < kGatherMax) ? nitems - base : kGatherMax;
        unsigned chunks = 0;
        for (int i = 0; i < t.n; ++i) {
            const sod_gather_item& it = items[base + i];
            if (it.src == nullptr || it.numel <= 0 || it.dst_offset < 0 || it.dst_offset + it.numel > dst_elems ||
                it.numel > 0x7fffffffll)
                return SOD_EINVAL;
            if (it.dst_offset & 7) return SOD_EALIGN;
            t.src[i] = it.src;
            t.dst_off8[i] = static_cast<unsigned>(it.dst_offset >> 3);
            t.numel[i] = static_cast<unsigned>(it.numel);
            t.chunk0[i] = chunks;
            chunks += static_cast<unsigned>((it.numel + kGatherChunk - 1) / kGatherChunk);
        }
        t.chunk0[t.n] = chunks;
        if (chunks == 0) continue;
        unsigned grid = chunks;
        const unsigned cap = 8u * static_cast<unsigned>(dev_info().sm_count);
        if (grid > cap) grid = cap;
        grad_gather16_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(t, reinterpret_cast<uint4*>(dst16));
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return static_cast<int>(e);
    }
    return SOD_OK;
}

extern "C" int sod_grad_nonfinite(const float* grad, int64_t n, uint32_t* found_inf, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(grad && found_inf && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && aligned16(grad), SOD_EALIGN);
    const long long nvec = n >> 2;
    long long blocks = (nvec + 1023) / 1024;
    if (blocks > 4ll * dev_info().sm_count) blocks = 4ll * dev_info().sm_count;
    grad_nonfinite_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const float4*>(grad), nvec, found_inf);
    return static_cast<int>(cudaGetLastError());
}

extern "C" int sod_grad_merge_bf16(float* grad, void* grad16, int64_t n, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(grad && grad16 && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && aligned16(grad) && aligned16(grad16), SOD_EALIGN);
    const long long nvec = n >> 2;
    long long blocks = (nvec + 1023) / 1024;
    if (blocks > 8ll * dev_info().sm_count) blocks = 8ll * dev_info().sm_count;
    grad_merge_bf16_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<float4*>(grad), reinterpret_cast<uint2*>(grad16), nvec);
    return static_cast<int>(cudaGetLastError());
}

extern "C" int sod_allreduce_sgd(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off, float* mom,
                                 void* shadow16, int64_t n, const sod_sgd_segment* segs, int nseg, const float* lr_dev,
                                 float inv_scale, const uint32_t* found_inf, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(comm && mom && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && aligned16(mom) && (grad_off & 15) == 0 && (param_off & 15) == 0, SOD_EALIGN);
    CommDev c;
    int rc = make_comm_dev(comm, c);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(grad_off >= sod_comm_flag_bytes() && param_off >= sod_comm_flag_bytes(), SOD_ECOMM);
    SOD_CHECK_ARG(grad_off + static_cast<uint64_t>(n) * 4 <= comm->arena_bytes &&
                      param_off + static_cast<uint64_t>(n) * 4 <= comm->arena_bytes, SOD_ECOMM);
    const int has16 = grad16_off != 0 ? 1 : 0;
    if (has16) {
        SOD_CHECK_ARG((grad16_off & 15) == 0, SOD_EALIGN);
        SOD_CHECK_ARG(grad16_off >= sod_comm_flag_bytes() && grad16_off + static_cast<uint64_t>(n) * 2 <= comm->arena_bytes, SOD_ECOMM);
    }
    SegTable t;
    rc = make_seg_table(segs, nseg, n, t);
    if (rc != SOD_OK) return rc;
    const long long nvec = n >> 2;
    const unsigned grid = comm_grid((nvec + c.world - 1) / c.world);
    const float scale = inv_scale / static_cast<float>(c.world);
    const int zg = (flags & SOD_SGD_ZERO_GRAD) ? 1 : 0;
    // with two ranks plain peer loads move the gradient bucket faster than the in-switch reduction; from four ranks up
    // NVLS wins (an all-reduce sweep, `bench.py --sweep`, decides this per system)
    const bool mc = (c.mc != 0) && !(flags & SOD_ALGO_NO_MULTIMEM) && (c.world > 2 || (flags & SOD_ALGO_FORCE_MULTIMEM));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (mc)
        allreduce_sgd_kernel<true><<<grid, kThreads, 0, s>>>(c, grad_off, param_off, reinterpret_cast<float4*>(mom), nvec, t,
                                                             scale, found_inf, zg, reinterpret_cast<uint2*>(shadow16), lr_dev, grad16_off, has16);
    else
        allreduce_sgd_kernel<false><<<grid, kThreads, 0, s>>>(c, grad_off, param_off, reinterpret_cast<float4*>(mom), nvec, t,
                                                              scale, found_inf, zg, reinterpret_cast<uint2*>(shadow16), lr_dev, grad16_off, has16);
    return static_cast<int>(cudaGetLastError());
}

extern "C" int sod_allreduce_f32(const sod_comm* comm, uint64_t off, int64_t n, float scale, int algo, int flags,
                                 void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(comm && n > 0 && algo >= 0 && algo <= 2, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && (off & 15) == 0, SOD_EALIGN);
    CommDev c;
    int rc = make_comm_dev(comm, c);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(off >= sod_comm_flag_bytes() && off + static_cast<uint64_t>(n) * 4 <= comm->arena_bytes, SOD_ECOMM);
    const long long nvec = n >> 2;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long one_shot_cap = static_cast<long long>(kThreads) * kUnroll *
                                   (dev_info().sm_count < SOD_COMM_MAX_BLOCKS ? dev_info().sm_count : SOD_COMM_MAX_BLOCKS);
    // the two-shot kernel over the NVLS mapping beats the one-shot kernel at every size once a multicast mapping exists
    // (`bench.py --sweep`); one-shot (every rank reads every peer) is only kept for fabrics without multicast
    const bool has_mc = (c.mc != 0) && !(flags & SOD_ALGO_NO_MULTIMEM);
    if (algo == 0) algo = (!has_mc && n * 4 <= (256 << 10)) ? 1 : 2;
    if (algo == 1 && nvec > one_shot_cap) return SOD_EUNSUPPORTED;
    if (algo == 1) {
        const unsigned grid = comm_grid(nvec);
        allreduce_one_shot_kernel<<<grid, kThreads, 0, s>>>(c, off, nvec, scale);
    } else {
        const unsigned grid = comm_grid((nvec + c.world - 1) / c.world);
        // in-switch reduction: always from four ranks up; with two ranks peer loads win above ≈2 MB
        const bool mc = has_mc && (c.world > 2 || n * 4 <= (2 << 20) || (flags & SOD_ALGO_FORCE_MULTIMEM));
        if (mc) allreduce_two_shot_kernel<true><<<grid, kThreads, 0, s>>>(c, off, nvec, scale);
        else allreduce_two_shot_kernel<false><<<grid, kThreads, 0, s>>>(c, off, nvec, scale);
    }
    return static_cast<int>(cudaGetLastError());
}
