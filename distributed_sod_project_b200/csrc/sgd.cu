// sgd.cu — gradient all-reduce ⊕ unscale ⊕ optimizer step (SGD-momentum, optionally Nesterov, or Adam) over flat fp32
// buffers, plus the plain peer-memory all-reduce used by the bandwidth sweep.
//
// Reference arithmetic being replaced (paths relative to the reference repo):
//   apex DDP(delay_allreduce=True): flat SUM all-reduce then ×1/W            train.py:185
//   apex amp unscale ×1/S with overflow skip                                  train.py:299
//   torch.optim.SGD.step (momentum, wd folded into g, no dampening, nesterov  train.py:303,
//       per segment) with groups from make_optimizer("f3_trick"/"sgd_trick")  utils/pipeline_ops.py:235-313
//   torch.optim.Adam.step (L2 weight decay, no amsgrad) of make_optimizer("adam") utils/pipeline_ops.py:287-294
//   optimizer.zero_grad                                                       train.py:297
//
// world == 1 : one streaming pass, 20 B/elem (read g,p,v; write p,v) [+4 B/elem to zero g]; Adam 28 B/elem (+ m).
// world  > 1 : two-shot over NVSwitch peer memory. Rank r owns shard r of the flat index space:
//     start barrier → reduce shard r across ranks (multimem.ld_reduce in the switch, or peer loads
//     summed in rank order) → unscale/÷W → SGD on (p,v) shard in registers → write the UPDATED
//     PARAMETERS to every rank (multimem.st / peer stores) → end barrier [→ zero local grads].
//   So what crosses NVLink is reduce-scatter(grads) + all-gather(params): the same bus bytes as an
//   all-reduce, but no separate NCCL call, no ÷W pass, no optimizer kernel, and momentum is only ever
//   touched on the owning rank (1/W of the optimizer-state traffic; the same holds for Adam's m and v).
// Both kernels are templates on the update rule (SgdRule / AdamRule below): the segment walk, the bf16-gradient
// handling, the exchange and the zero-grad / shadow tail exist once.  Two more template parameters: the 16-bit format of
// grad16 / shadow16 (Bf16x4, or F16x4 for amp fp16) and whether skip and 1/scale come from the device-resident loss
// scaler, which the kernel then advances (apex amp O1's dynamic loss scale, no host round trip).
//   Owner-computes + broadcast also makes parameters bit-identical on all ranks by construction.
#include "common.cuh"

#include <cstdio>
#include <cstdlib>
#include <type_traits>

namespace sod {
namespace {

constexpr int kThreads = 512;
constexpr int kUnroll = 4;

struct SegTable {
    int n;
    long long begin[SOD_MAX_SEGMENTS], end[SOD_MAX_SEGMENTS];  // in float4 units
    float lr[SOD_MAX_SEGMENTS], wd[SOD_MAX_SEGMENTS];
    float mu[SOD_MAX_SEGMENTS];                              // SGD momentum
    // Adam: β1, β2 as the decimals the caller wrote (see adam_beta), 1-β1 and 1-β2 rounded to fp32 as torch rounds the
    // Python scalars, β2 and eps in fp32
    double beta1d[SOD_MAX_SEGMENTS], beta2d[SOD_MAX_SEGMENTS];
    float w1[SOD_MAX_SEGMENTS], c2[SOD_MAX_SEGMENTS], beta2[SOD_MAX_SEGMENTS], eps[SOD_MAX_SEGMENTS];
    int flags[SOD_MAX_SEGMENTS];
};

// the range and flag fields shared by both segment kinds
template <class Seg>
static int make_seg_ranges(const Seg* segs, int nseg, int64_t n, SegTable& t) {
    if (nseg < 0 || nseg > SOD_MAX_SEGMENTS || (nseg > 0 && segs == nullptr)) return SOD_EINVAL;
    t.n = nseg;
    long long prev = 0;
    for (int i = 0; i < nseg; ++i) {
        const Seg& s = segs[i];
        if (s.begin < prev || s.end < s.begin || s.end > n) return SOD_EINVAL;  // sorted, disjoint, in range
        if ((s.begin & 3) || (s.end & 3)) return SOD_EALIGN;
        t.begin[i] = s.begin >> 2; t.end[i] = s.end >> 2;
        t.lr[i] = s.lr; t.wd[i] = s.weight_decay; t.flags[i] = s.flags;
        t.mu[i] = 0.f; t.beta1d[i] = t.beta2d[i] = 0.0; t.w1[i] = t.c2[i] = t.beta2[i] = t.eps[i] = 0.f;
        prev = s.end;
    }
    return SOD_OK;
}

static int make_seg_table(const sod_sgd_segment* segs, int nseg, int64_t n, SegTable& t) {
    const int rc = make_seg_ranges(segs, nseg, n, t);
    if (rc != SOD_OK) return rc;
    for (int i = 0; i < nseg; ++i) t.mu[i] = segs[i].momentum;
    return SOD_OK;
}

// The segment carries β as fp32, torch.optim.Adam as a Python float: 0.999f is 0.99900001287…, and 1 - 0.999f differs from
// fp32(1 - 0.999) by 1.3e-5 relative.  Recover the decimal the caller wrote — the shortest one that rounds to the same
// fp32 value, which is what an fp32 of a literal like 0.9 or 0.999 came from — so that 1-β and the bias corrections are
// formed from the same double torch uses.
static double adam_beta(float b) {
    char buf[32];
    for (int digits = 1; digits <= 9; ++digits) {
        snprintf(buf, sizeof(buf), "%.*g", digits, static_cast<double>(b));
        const double d = strtod(buf, nullptr);
        if (static_cast<float>(d) == b) return d;
    }
    return static_cast<double>(b);
}

static int make_seg_table(const sod_adam_segment* segs, int nseg, int64_t n, SegTable& t) {
    const int rc = make_seg_ranges(segs, nseg, n, t);
    if (rc != SOD_OK) return rc;
    for (int i = 0; i < nseg; ++i) {
        const sod_adam_segment& s = segs[i];
        if (!(s.beta1 >= 0.f && s.beta1 < 1.f && s.beta2 >= 0.f && s.beta2 < 1.f && s.eps >= 0.f)) return SOD_EINVAL;
        if (s.flags & SOD_SEG_NESTEROV) return SOD_EINVAL;
        t.beta1d[i] = adam_beta(s.beta1); t.beta2d[i] = adam_beta(s.beta2);
        t.w1[i] = static_cast<float>(1.0 - t.beta1d[i]); t.c2[i] = static_cast<float>(1.0 - t.beta2d[i]);
        t.beta2[i] = s.beta2; t.eps[i] = s.eps;
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

__device__ __forceinline__ void sgd_update(float4& p, float4& v, const float4& g, float lr, float wd, float mu, bool nesterov) {
    // g' = g + wd*p ; v = mu*v + g' ; p = p - lr*v   (operation order of torch/optim/sgd.py:343-380)
    // nesterov:                       p = p - lr*(g' + mu*v)
    float gx = fmaf(wd, p.x, g.x), gy = fmaf(wd, p.y, g.y), gz = fmaf(wd, p.z, g.z), gw = fmaf(wd, p.w, g.w);
    v.x = fmaf(mu, v.x, gx); v.y = fmaf(mu, v.y, gy); v.z = fmaf(mu, v.z, gz); v.w = fmaf(mu, v.w, gw);
    if (nesterov) {
        gx = fmaf(mu, v.x, gx); gy = fmaf(mu, v.y, gy); gz = fmaf(mu, v.z, gz); gw = fmaf(mu, v.w, gw);
    } else {
        gx = v.x; gy = v.y; gz = v.z; gw = v.w;
    }
    p.x = fmaf(-lr, gx, p.x); p.y = fmaf(-lr, gy, p.y); p.z = fmaf(-lr, gz, p.z); p.w = fmaf(-lr, gw, p.w);
}

// An update rule is what the two step kernels below are templated on:
//   State                per-vector optimizer state held in registers between load and store
//   Cta                  per-CTA constants, computed once into shared memory by prologue()
//   load / store         the state of flat vector i
//   update               one float4 of parameters, given the unscaled-and-averaged gradient and its segment
//   epilogue             after the last access of the CTA (Adam: the last CTA advances the step counters)
// kNesterov: some segment carries SOD_SEG_NESTEROV (the plain instantiation is the kernel without that select)
template <bool kNesterov>
struct SgdRule {
    static constexpr bool kHasCta = false;
    float4* __restrict__ v;
    struct State { float4 v; };
    struct Cta {};
    __device__ __forceinline__ void prologue(Cta&, const SegTable&, const float*) const {}
    __device__ __forceinline__ void load(State& st, long long i) const { st.v = v[i]; }
    __device__ __forceinline__ void store(const State& st, long long i) const { v[i] = st.v; }
    __device__ __forceinline__ void update(float4& p, State& st, const float4& g, const SegTable& segs, const float* lr_dev,
                                           const Cta&, int s) const {
        sgd_update(p, st.v, g, seg_lr(segs, lr_dev, s), segs.wd[s], segs.mu[s], kNesterov && (segs.flags[s] & SOD_SEG_NESTEROV));
    }
    __device__ __forceinline__ void epilogue(const SegTable&, bool) const {}
};

__device__ __forceinline__ void adam_update1(float& p, float& m, float& v, float g, float wd, float w1, float b2, float c2,
                                             float step_size, float bc2_sqrt, float eps) {
    // torch/optim/adam.py _single_tensor_adam (amsgrad=False, maximize=False, L2 weight decay):
    //   g' = g + wd*p ; m.lerp_(g', 1-β1) ; v.mul_(β2).addcmul_(g', g', 1-β2) ;
    //   p.addcdiv_(m, sqrt(v)/bc2_sqrt + eps, -step_size)          IEEE sqrt and division (no fast-math in this build)
    const float gg = fmaf(wd, p, g);
    m = fmaf(w1, gg - m, m);
    v = fmaf(c2 * gg, gg, v * b2);
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p = fmaf(-step_size, m / denom, p);
}

struct AdamRule {
    static constexpr bool kHasCta = true;
    float4* __restrict__ m;
    float4* __restrict__ v;
    int32_t* step;          // [SOD_MAX_SEGMENTS] step counts, then the CTA ticket (sod_adam in include/sod_b200.h)
    struct State { float4 m, v; };
    struct Cta { float step_size[SOD_MAX_SEGMENTS], bc2_sqrt[SOD_MAX_SEGMENTS]; };
    // bias corrections of step t = step+1, in fp64 once per CTA and segment, rounded as torch rounds the Python scalars
    __device__ __forceinline__ void prologue(Cta& cta, const SegTable& segs, const float* lr_dev) const {
        const int s = threadIdx.x;
        if (s < segs.n) {
            const double t = static_cast<double>(step[s]) + 1.0;
            const double bc1 = 1.0 - pow(segs.beta1d[s], t);
            const double bc2 = 1.0 - pow(segs.beta2d[s], t);
            cta.step_size[s] = static_cast<float>(static_cast<double>(seg_lr(segs, lr_dev, s)) / bc1);
            cta.bc2_sqrt[s] = static_cast<float>(sqrt(bc2));
        }
    }
    __device__ __forceinline__ void load(State& st, long long i) const { st.m = m[i]; st.v = v[i]; }
    __device__ __forceinline__ void store(const State& st, long long i) const { m[i] = st.m; v[i] = st.v; }
    __device__ __forceinline__ void update(float4& p, State& st, const float4& g, const SegTable& segs, const float*,
                                           const Cta& cta, int s) const {
        const float wd = segs.wd[s], b2 = segs.beta2[s], eps = segs.eps[s], w1 = segs.w1[s], c2 = segs.c2[s];
        const float ss = cta.step_size[s], bs = cta.bc2_sqrt[s];
        adam_update1(p.x, st.m.x, st.v.x, g.x, wd, w1, b2, c2, ss, bs, eps);
        adam_update1(p.y, st.m.y, st.v.y, g.y, wd, w1, b2, c2, ss, bs, eps);
        adam_update1(p.z, st.m.z, st.v.z, g.z, wd, w1, b2, c2, ss, bs, eps);
        adam_update1(p.w, st.m.w, st.v.w, g.w, wd, w1, b2, c2, ss, bs, eps);
    }
    // every CTA read the counters in its prologue; the last one to get here (ticket, as in resample.cu's colsum) advances
    // them — unless the step was skipped for an amp overflow — and re-arms the ticket for the next launch
    __device__ __forceinline__ void epilogue(const SegTable& segs, bool skip) const {
        __shared__ bool s_last;
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            s_last = atomicAdd(reinterpret_cast<unsigned*>(step + SOD_MAX_SEGMENTS), 1u) == gridDim.x - 1;
        }
        __syncthreads();
        if (s_last && threadIdx.x == 0) {
            __threadfence();
            if (!skip)
                for (int s = 0; s < segs.n; ++s)
                    if (!(segs.flags[s] & SOD_SEG_FROZEN)) step[s] += 1;
            step[SOD_MAX_SEGMENTS] = 0;
        }
    }
};

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

// The 16-bit format of `grad16` / `shadow16`, four elements per uint2, and the exponent field that marks inf / NaN:
// bf16 (amp bf16, the default) or fp16 (SOD_GRAD16_F16, amp fp16).  Both convert with round-to-nearest-even.
struct Bf16x4 {
    static constexpr uint32_t kExp = 0x7f80u;
    __device__ __forceinline__ static float4 to_f32(uint2 u) { return bf16x4_to_f32(u); }
    __device__ __forceinline__ static uint2 from_f32(const float4& f) { return f32x4_to_bf16(f); }
};
struct F16x4 {
    static constexpr uint32_t kExp = 0x7c00u;
    __device__ __forceinline__ static float4 to_f32(uint2 u) {
        const __half2* h = reinterpret_cast<const __half2*>(&u);
        const float2 a = __half22float2(h[0]), b = __half22float2(h[1]);
        return make_float4(a.x, a.y, b.x, b.y);
    }
    __device__ __forceinline__ static uint2 from_f32(const float4& f) {
        uint2 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
        h[0] = __floats2half2_rn(f.x, f.y);
        h[1] = __floats2half2_rn(f.z, f.w);
        return u;
    }
};

// both 16-bit halves of w: is either inf or NaN (exponent field all ones) in the format whose exponent mask is kExp
template <uint32_t kExp>
__device__ __forceinline__ bool nonfinite16x2(uint32_t w) {
    return (w & kExp) == kExp || ((w >> 16) & kExp) == kExp;
}

// The dynamic loss scale's rules (apex amp O1, include/sod_b200.h sod_loss_scaler), applied once per step by the last CTA
// to get here (a ticket, as AdamRule::epilogue does), which then re-arms the ticket.  found_inf is left at the verdict.
__device__ __forceinline__ void scaler_epilogue(sod_loss_scaler* sc, bool skip) {
    __shared__ bool s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = atomicAdd(&sc->ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0) {
        __threadfence();
        if (skip) {
            sc->scale = fmaxf(sc->scale * 0.5f, 1.0f);
            sc->unskipped = 0;
        } else {
            sc->unskipped += 1;
            if (sc->growth_interval > 0 && sc->unskipped % sc->growth_interval == 0) sc->scale *= 2.0f;
        }
        sc->found_inf = skip ? 1u : 0u;
        sc->ticket = 0u;
    }
}

// kScaler: skip and 1/scale come from the device-resident loss scaler (read at execution time), which the kernel then
// advances; otherwise from the (inv_scale, found_inf) arguments
template <class Rule, class H, bool kScaler>
__global__ void __launch_bounds__(kThreads) local_step_kernel(float4* __restrict__ p, const Rule rule,
                                                              float4* __restrict__ g, uint2* __restrict__ g16,
                                                              uint2* __restrict__ shadow, long long nvec,
                                                              const __grid_constant__ SegTable segs, float inv_scale_arg,
                                                              const uint32_t* found_inf, int zero_grad,
                                                              const float* __restrict__ lr_dev, sod_loss_scaler* scaler) {
    bool skip;                                                     // amp overflow: no update, but still clear g
    float inv_scale = inv_scale_arg;
    if constexpr (kScaler) {
        skip = scaler->found_inf != 0u;
        inv_scale = 1.0f / scaler->scale;
    } else {
        skip = (found_inf != nullptr && *found_inf != 0);
    }
    __shared__ typename Rule::Cta cta;
    rule.prologue(cta, segs, lr_dev);
    if constexpr (Rule::kHasCta) __syncthreads();
    SegCursor cur;
    const long long stride = static_cast<long long>(gridDim.x) * kThreads;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long i0 = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; i0 < nvec; i0 += stride * kUnroll) {
        float4 gv[kUnroll], pv[kUnroll];
        typename Rule::State st[kUnroll];
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
                    gv[u] = H::to_f32(g16[i]);
                } else {
                    gv[u] = g[i];
                    if (g16 != nullptr) {   // gradients autograd left in bf16: fold them in here (the "cast" of amp O1)
                        const float4 h = H::to_f32(g16[i]);
                        gv[u].x += h.x; gv[u].y += h.y; gv[u].z += h.z; gv[u].w += h.w;
                    }
                }
                if (!skip && in_seg && !(segs.flags[cur.s] & SOD_SEG_FROZEN)) {
                    sidx[u] = cur.s;
                    pv[u] = p[i];
                    rule.load(st[u], i);
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
                    rule.update(pv[u], st[u], gs, segs, lr_dev, cta, s);
                    p[i] = pv[u];
                    rule.store(st[u], i);
                    if (shadow != nullptr) shadow[i] = H::from_f32(pv[u]);
                }
                if (zero_grad) {
                    if (!only16[u]) g[i] = zero;
                    if (g16 != nullptr) g16[i] = make_uint2(0u, 0u);
                }
            }
        }
    }
    rule.epilogue(segs, skip);
    if constexpr (kScaler) scaler_epilogue(scaler, skip);
}

template <class H>
__global__ void grad_merge16_kernel(float4* __restrict__ g, uint2* __restrict__ g16, long long nvec) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < nvec;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const uint2 raw = g16[i];
        if ((raw.x | raw.y) != 0u) {   // most of the flat buffer (BN parameters, padding) never sees a bf16 gradient
            float4 a = g[i];
            const float4 h = H::to_f32(raw);
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

// kExp != 0 (sod_grad_gather16_checked): also OR into *found whether anything copied is inf / NaN in the format of kExp
template <uint32_t kExp>
__global__ void __launch_bounds__(256) grad_gather16_kernel(const __grid_constant__ GatherTable t, uint4* __restrict__ dst,
                                                            uint32_t* found) {
    bool bad = false;
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
            for (unsigned i = threadIdx.x; i < nv; i += 256) {
                const uint4 v = __ldcs(s4 + i);
                d4[i] = v;
                if constexpr (kExp != 0u)
                    bad |= nonfinite16x2<kExp>(v.x) | nonfinite16x2<kExp>(v.y) | nonfinite16x2<kExp>(v.z) |
                           nonfinite16x2<kExp>(v.w);
            }
            for (unsigned i = (nv << 3) + threadIdx.x; i < cnt; i += 256) {
                const unsigned short v = src[i];
                out[i] = v;
                if constexpr (kExp != 0u) bad |= (v & kExp) == kExp;
            }
        } else {
            for (unsigned i = threadIdx.x; i < cnt; i += 256) {
                const unsigned short v = src[i];
                out[i] = v;
                if constexpr (kExp != 0u) bad |= (v & kExp) == kExp;
            }
        }
    }
    if constexpr (kExp != 0u)
        if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(found, 1u);
}

// ------------------------------------------------------------------------------------------------
// amp overflow check of the gradients the checked gather does not copy: listed ranges of the fp32 buffer (BN γ/β and
// other parameters without a 16-bit gradient) and of the 16-bit one (folded convolution-bias gradients the SyncBN backward
// accumulates in place).  Same chunked work split as the gather.
// ------------------------------------------------------------------------------------------------
constexpr int kCheckMax = SOD_CHECK_MAX_RANGES;
constexpr int kCheckChunk = 4096;
struct CheckTable {
    int n;
    long long begin[kCheckMax];
    unsigned numel[kCheckMax];
    unsigned chunk0[kCheckMax + 1];
    unsigned char in16[kCheckMax];
};

template <uint32_t kExp>
__global__ void __launch_bounds__(256) grad_check_ranges_kernel(const __grid_constant__ CheckTable t, const float* __restrict__ g,
                                                                const unsigned short* __restrict__ g16, uint32_t* found) {
    bool bad = false;
    const unsigned total = t.chunk0[t.n];
    for (unsigned c = blockIdx.x; c < total; c += gridDim.x) {
        int lo = 0, hi = t.n - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (t.chunk0[mid] <= c) lo = mid; else hi = mid - 1;
        }
        const unsigned first = (c - t.chunk0[lo]) * kCheckChunk;
        const unsigned left = t.numel[lo] - first;
        const unsigned cnt = left < kCheckChunk ? left : kCheckChunk;
        const long long b = t.begin[lo] + first;
        if (t.in16[lo]) {
            for (unsigned i = threadIdx.x; i < cnt; i += 256) bad |= (g16[b + i] & kExp) == kExp;
        } else {
            for (unsigned i = threadIdx.x; i < cnt; i += 256) bad |= !isfinite(g[b + i]);
        }
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(found, 1u);
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
// unlike a bf16 multimem reduction), so every owner obtains the same value it would from an fp32 exchange of the same data.
// H = F16x4: the same for fp16 gradients (exact as well: every fp16 value is an fp32 value)
template <class H>
__device__ __forceinline__ float4 reduce_vec16(const CommDev& c, uint64_t byte_off) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    uint2 raw[SOD_MAX_WORLD];
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) raw[q] = ld_relaxed_sys_v2(reinterpret_cast<const void*>(c.peer[q] + byte_off));
#pragma unroll
    for (int q = 0; q < SOD_MAX_WORLD; ++q)
        if (q < c.world) {
            const float4 t = H::to_f32(raw[q]);
            acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
        }
    return acc;
}

// kScaler: the loss scaler sits at arena offset scaler_off on every rank; the verdict is the OR of all ranks' found_inf
// words, read after the start barrier (each rank cleared its own before its checks, after its previous step), and the
// scale is the local scaler's (bit-identical on all ranks, since every rank applies the same verdict)
template <class Rule, bool kMulticast, class H, bool kScaler>
__global__ void __launch_bounds__(kThreads) allreduce_step_kernel(const __grid_constant__ CommDev c, uint64_t grad_off,
                                                                  uint64_t param_off, const Rule rule,
                                                                  long long nvec, const __grid_constant__ SegTable segs,
                                                                  float scale_arg, const uint32_t* found_inf,
                                                                  int zero_grad, uint2* __restrict__ shadow,
                                                                  const float* __restrict__ lr_dev, uint64_t grad16_off,
                                                                  int has_grad16, uint64_t scaler_off) {
    bool skip = !kScaler && (found_inf != nullptr && *found_inf != 0);  // caller guarantees identical on all ranks
    float scale = scale_arg;
    __shared__ typename Rule::Cta cta;
    rule.prologue(cta, segs, lr_dev);                             // (the barrier below orders it for the whole CTA)
    // every rank's backward has finished writing its gradients
    if (!comm_block_barrier(c, 0, blockIdx.x)) return;
    sod_loss_scaler* scaler = nullptr;
    if constexpr (kScaler) {
        __shared__ bool s_skip;
        scaler = reinterpret_cast<sod_loss_scaler*>(c.peer[c.rank] + scaler_off);
        if (threadIdx.x == 0) {
            uint32_t any = 0u;
            for (int q = 0; q < c.world; ++q)
                any |= ld_acquire_sys(reinterpret_cast<const uint32_t*>(c.peer[q] + scaler_off));  // found_inf is word 0
            s_skip = any != 0u;
        }
        __syncthreads();
        skip = s_skip;
        scale = (1.0f / scaler->scale) / static_cast<float>(c.world);
    }

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
                        gv[u] = reduce_vec16<H>(c, grad16_off + static_cast<uint64_t>(i) * 8u);
                    else
                        gv[u] = reduce_vec<kMulticast>(c, grad_off + static_cast<uint64_t>(i) * 16u);
                }
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const long long i = i0 + u * stride;
                if (sidx[u] >= 0) {
                    const int s = sidx[u];
                    float4 pv = p_local[i];
                    typename Rule::State st;
                    rule.load(st, i);
                    const float4 gs = make_float4(gv[u].x * scale, gv[u].y * scale, gv[u].z * scale, gv[u].w * scale);
                    rule.update(pv, st, gs, segs, lr_dev, cta, s);
                    rule.store(st, i);
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
                if (shadow != nullptr && !skip) shadow[i] = H::from_f32(p_local[i]);
            }
        }
    }
    rule.epilogue(segs, skip);
    // every CTA of this rank has passed the end barrier, so every peer has read this rank's found_inf: the last CTA may
    // overwrite it with the verdict
    if constexpr (kScaler) scaler_epilogue(scaler, skip);
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

namespace sod {
namespace {

static bool any_nesterov(const sod_sgd_segment* segs, int nseg) {
    for (int i = 0; segs != nullptr && i < nseg && i < SOD_MAX_SEGMENTS; ++i)
        if (segs[i].flags & SOD_SEG_NESTEROV) return true;
    return false;
}

// world 1: validation shared by sod_sgd_momentum and sod_adam, then one streaming launch of local_step_kernel<Rule>
// world 1: validation shared by sod_sgd_momentum, sod_adam and their *_scaler forms, then one streaming launch of
// local_step_kernel<Rule, 16-bit format, scaler?>
template <class Rule, class Seg>
int launch_local_step(float* param, const Rule& rule, float* grad, void* grad16, void* shadow16, int64_t n, const Seg* segs,
                      int nseg, const float* lr_dev, float inv_scale, const uint32_t* found_inf, sod_loss_scaler* scaler,
                      int flags, void* stream) {
    SOD_CHECK_ARG(param && grad && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && aligned16(param) && aligned16(grad), SOD_EALIGN);
    SOD_CHECK_ARG((!grad16 || aligned16(grad16)) && (!shadow16 || aligned16(shadow16)), SOD_EALIGN);
    SegTable t;
    int rc = make_seg_table(segs, nseg, n, t);
    if (rc != SOD_OK) return rc;
    const long long nvec = n >> 2;
    long long blocks = (nvec + static_cast<long long>(kThreads) * kUnroll - 1) / (static_cast<long long>(kThreads) * kUnroll);
    const long long cap = 2ll * dev_info().sm_count;
    if (blocks > cap) blocks = cap;
    auto go = [&](auto kernel) {
        kernel<<<static_cast<unsigned>(blocks), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
            reinterpret_cast<float4*>(param), rule, reinterpret_cast<float4*>(grad),
            reinterpret_cast<uint2*>(grad16), reinterpret_cast<uint2*>(shadow16), nvec, t, inv_scale, found_inf,
            (flags & SOD_SGD_ZERO_GRAD) ? 1 : 0, lr_dev, scaler);
        return static_cast<int>(cudaGetLastError());
    };
    if (flags & SOD_GRAD16_F16)
        return scaler ? go(local_step_kernel<Rule, F16x4, true>) : go(local_step_kernel<Rule, F16x4, false>);
    return scaler ? go(local_step_kernel<Rule, Bf16x4, true>) : go(local_step_kernel<Rule, Bf16x4, false>);
}

// world > 1: validation shared by sod_allreduce_sgd, sod_allreduce_adam and their *_scaler forms, then
// allreduce_step_kernel<Rule, multicast?, 16-bit format, scaler?>
template <class Rule, class Seg>
int launch_allreduce_step(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off, const Rule& rule,
                          void* shadow16, int64_t n, const Seg* segs, int nseg, const float* lr_dev, float inv_scale,
                          const uint32_t* found_inf, sod_loss_scaler* scaler, int flags, void* stream) {
    SOD_CHECK_ARG(comm && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && (grad_off & 15) == 0 && (param_off & 15) == 0, SOD_EALIGN);
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
    uint64_t scaler_off = 0;
    if (scaler != nullptr) {   // the local scaler must be the arena's: its offset addresses every rank's copy
        const uint64_t a = reinterpret_cast<uint64_t>(scaler), base = comm->peer[comm->rank];
        SOD_CHECK_ARG((a & 15) == 0, SOD_EALIGN);
        SOD_CHECK_ARG(a >= base + sod_comm_flag_bytes() && a + sizeof(sod_loss_scaler) <= base + comm->arena_bytes, SOD_ECOMM);
        scaler_off = a - base;
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
    auto go = [&](auto kernel) {
        kernel<<<grid, kThreads, 0, s>>>(c, grad_off, param_off, rule, nvec, t, scale, found_inf, zg,
                                         reinterpret_cast<uint2*>(shadow16), lr_dev, grad16_off, has16, scaler_off);
        return static_cast<int>(cudaGetLastError());
    };
    auto pick = [&](auto h, auto sc) {
        using H = decltype(h);
        constexpr bool kSc = decltype(sc)::value;
        return mc ? go(allreduce_step_kernel<Rule, true, H, kSc>) : go(allreduce_step_kernel<Rule, false, H, kSc>);
    };
    if (flags & SOD_GRAD16_F16)
        return scaler ? pick(F16x4{}, std::true_type{}) : pick(F16x4{}, std::false_type{});
    return scaler ? pick(Bf16x4{}, std::true_type{}) : pick(Bf16x4{}, std::false_type{});
}

}  // namespace
}  // namespace sod

extern "C" int sod_sgd_momentum(float* param, float* mom, float* grad, void* grad16, void* shadow16, int64_t n,
                                const sod_sgd_segment* segs, int nseg, const float* lr_dev, float inv_scale,
                                const uint32_t* found_inf, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(param && mom && grad && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(mom), SOD_EALIGN);
    if (any_nesterov(segs, nseg))
        return launch_local_step(param, SgdRule<true>{reinterpret_cast<float4*>(mom)}, grad, grad16, shadow16, n, segs, nseg,
                                 lr_dev, inv_scale, found_inf, nullptr, flags, stream);
    return launch_local_step(param, SgdRule<false>{reinterpret_cast<float4*>(mom)}, grad, grad16, shadow16, n, segs, nseg,
                             lr_dev, inv_scale, found_inf, nullptr, flags, stream);
}

extern "C" int sod_adam(float* param, float* exp_avg, float* exp_avg_sq, float* grad, void* grad16, void* shadow16, int64_t n,
                        const sod_adam_segment* segs, int nseg, const float* lr_dev, int32_t* step_dev, float inv_scale,
                        const uint32_t* found_inf, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(param && exp_avg && exp_avg_sq && step_dev && grad && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(exp_avg) && aligned16(exp_avg_sq), SOD_EALIGN);
    const AdamRule rule{reinterpret_cast<float4*>(exp_avg), reinterpret_cast<float4*>(exp_avg_sq), step_dev};
    return launch_local_step(param, rule, grad, grad16, shadow16, n, segs, nseg, lr_dev, inv_scale, found_inf, nullptr, flags, stream);
}

namespace sod {
namespace {

template <uint32_t kExp>
int gather16(const sod_gather_item* items, int nitems, void* dst16, int64_t dst_elems, uint32_t* found, void* stream) {
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
        grad_gather16_kernel<kExp><<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(t, reinterpret_cast<uint4*>(dst16), found);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return static_cast<int>(e);
    }
    return SOD_OK;
}

template <class H>
int merge16(float* grad, void* grad16, int64_t n, void* stream) {
    SOD_CHECK_ARG(grad && grad16 && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG((n & 3) == 0 && aligned16(grad) && aligned16(grad16), SOD_EALIGN);
    const long long nvec = n >> 2;
    long long blocks = (nvec + 1023) / 1024;
    if (blocks > 8ll * dev_info().sm_count) blocks = 8ll * dev_info().sm_count;
    grad_merge16_kernel<H><<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<float4*>(grad), reinterpret_cast<uint2*>(grad16), nvec);
    return static_cast<int>(cudaGetLastError());
}

}  // namespace
}  // namespace sod

extern "C" int sod_grad_gather16(const sod_gather_item* items, int nitems, void* dst16, int64_t dst_elems, void* stream) {
    return sod::gather16<0u>(items, nitems, dst16, dst_elems, nullptr, stream);
}

extern "C" int sod_grad_gather16_checked(const sod_gather_item* items, int nitems, void* dst16, int64_t dst_elems, int dtype,
                                         uint32_t* found_inf, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(found_inf && (dtype == SOD_BF16 || dtype == SOD_F16), SOD_EINVAL);
    return dtype == SOD_F16 ? gather16<F16x4::kExp>(items, nitems, dst16, dst_elems, found_inf, stream)
                            : gather16<Bf16x4::kExp>(items, nitems, dst16, dst_elems, found_inf, stream);
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

extern "C" int sod_grad_check_ranges(const float* grad, const void* grad16, int64_t n, const sod_check_range* ranges,
                                     int nranges, int flags, uint32_t* found_inf, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(found_inf && n > 0 && nranges >= 0 && (nranges == 0 || ranges), SOD_EINVAL);
    for (int base = 0; base < nranges; base += kCheckMax) {
        CheckTable t;
        t.n = 0;
        unsigned chunks = 0;
        for (int i = base; i < nranges && i < base + kCheckMax; ++i) {
            const sod_check_range& r = ranges[i];
            const bool in16 = (r.flags & SOD_SEG_GRAD16) != 0;
            if (r.begin < 0 || r.end < r.begin || r.end > n || r.end - r.begin > 0x7fffffffll) return SOD_EINVAL;
            if (in16 ? grad16 == nullptr : grad == nullptr) return SOD_EINVAL;
            if (r.end == r.begin) continue;
            t.begin[t.n] = r.begin;
            t.numel[t.n] = static_cast<unsigned>(r.end - r.begin);
            t.in16[t.n] = in16 ? 1 : 0;
            t.chunk0[t.n] = chunks;
            chunks += static_cast<unsigned>((r.end - r.begin + kCheckChunk - 1) / kCheckChunk);
            ++t.n;
        }
        t.chunk0[t.n] = chunks;
        if (chunks == 0) continue;
        unsigned grid = chunks;
        const unsigned cap = 4u * static_cast<unsigned>(dev_info().sm_count);
        if (grid > cap) grid = cap;
        cudaStream_t s = static_cast<cudaStream_t>(stream);
        const unsigned short* g16 = static_cast<const unsigned short*>(grad16);
        if (flags & SOD_GRAD16_F16)
            grad_check_ranges_kernel<F16x4::kExp><<<grid, 256, 0, s>>>(t, grad, g16, found_inf);
        else
            grad_check_ranges_kernel<Bf16x4::kExp><<<grid, 256, 0, s>>>(t, grad, g16, found_inf);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return static_cast<int>(e);
    }
    return SOD_OK;
}

extern "C" int sod_grad_merge_bf16(float* grad, void* grad16, int64_t n, void* stream) {
    return sod::merge16<sod::Bf16x4>(grad, grad16, n, stream);
}

extern "C" int sod_grad_merge16(float* grad, void* grad16, int64_t n, int flags, void* stream) {
    return (flags & SOD_GRAD16_F16) ? sod::merge16<sod::F16x4>(grad, grad16, n, stream)
                                    : sod::merge16<sod::Bf16x4>(grad, grad16, n, stream);
}

extern "C" int sod_allreduce_sgd(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off, float* mom,
                                 void* shadow16, int64_t n, const sod_sgd_segment* segs, int nseg, const float* lr_dev,
                                 float inv_scale, const uint32_t* found_inf, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(comm && mom && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(mom), SOD_EALIGN);
    if (any_nesterov(segs, nseg))
        return launch_allreduce_step(comm, grad_off, grad16_off, param_off, SgdRule<true>{reinterpret_cast<float4*>(mom)},
                                     shadow16, n, segs, nseg, lr_dev, inv_scale, found_inf, nullptr, flags, stream);
    return launch_allreduce_step(comm, grad_off, grad16_off, param_off, SgdRule<false>{reinterpret_cast<float4*>(mom)},
                                 shadow16, n, segs, nseg, lr_dev, inv_scale, found_inf, nullptr, flags, stream);
}

extern "C" int sod_allreduce_adam(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off,
                                  float* exp_avg, float* exp_avg_sq, void* shadow16, int64_t n, const sod_adam_segment* segs,
                                  int nseg, const float* lr_dev, int32_t* step_dev, float inv_scale,
                                  const uint32_t* found_inf, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(comm && exp_avg && exp_avg_sq && step_dev && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(exp_avg) && aligned16(exp_avg_sq), SOD_EALIGN);
    const AdamRule rule{reinterpret_cast<float4*>(exp_avg), reinterpret_cast<float4*>(exp_avg_sq), step_dev};
    return launch_allreduce_step(comm, grad_off, grad16_off, param_off, rule, shadow16, n, segs, nseg, lr_dev, inv_scale,
                                 found_inf, nullptr, flags, stream);
}

extern "C" int sod_sgd_momentum_scaler(float* param, float* mom, float* grad, void* grad16, void* shadow16, int64_t n,
                                       const sod_sgd_segment* segs, int nseg, const float* lr_dev, sod_loss_scaler* scaler,
                                       int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(param && mom && grad && scaler && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(mom), SOD_EALIGN);
    if (any_nesterov(segs, nseg))
        return launch_local_step(param, SgdRule<true>{reinterpret_cast<float4*>(mom)}, grad, grad16, shadow16, n, segs, nseg,
                                 lr_dev, 1.0f, nullptr, scaler, flags, stream);
    return launch_local_step(param, SgdRule<false>{reinterpret_cast<float4*>(mom)}, grad, grad16, shadow16, n, segs, nseg,
                             lr_dev, 1.0f, nullptr, scaler, flags, stream);
}

extern "C" int sod_adam_scaler(float* param, float* exp_avg, float* exp_avg_sq, float* grad, void* grad16, void* shadow16,
                               int64_t n, const sod_adam_segment* segs, int nseg, const float* lr_dev, int32_t* step_dev,
                               sod_loss_scaler* scaler, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(param && exp_avg && exp_avg_sq && step_dev && grad && scaler && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(exp_avg) && aligned16(exp_avg_sq), SOD_EALIGN);
    const AdamRule rule{reinterpret_cast<float4*>(exp_avg), reinterpret_cast<float4*>(exp_avg_sq), step_dev};
    return launch_local_step(param, rule, grad, grad16, shadow16, n, segs, nseg, lr_dev, 1.0f, nullptr, scaler, flags, stream);
}

extern "C" int sod_allreduce_sgd_scaler(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off,
                                        float* mom, void* shadow16, int64_t n, const sod_sgd_segment* segs, int nseg,
                                        const float* lr_dev, sod_loss_scaler* scaler, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(comm && mom && scaler && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(mom), SOD_EALIGN);
    if (any_nesterov(segs, nseg))
        return launch_allreduce_step(comm, grad_off, grad16_off, param_off, SgdRule<true>{reinterpret_cast<float4*>(mom)},
                                     shadow16, n, segs, nseg, lr_dev, 1.0f, nullptr, scaler, flags, stream);
    return launch_allreduce_step(comm, grad_off, grad16_off, param_off, SgdRule<false>{reinterpret_cast<float4*>(mom)},
                                 shadow16, n, segs, nseg, lr_dev, 1.0f, nullptr, scaler, flags, stream);
}

extern "C" int sod_allreduce_adam_scaler(const sod_comm* comm, uint64_t grad_off, uint64_t grad16_off, uint64_t param_off,
                                         float* exp_avg, float* exp_avg_sq, void* shadow16, int64_t n,
                                         const sod_adam_segment* segs, int nseg, const float* lr_dev, int32_t* step_dev,
                                         sod_loss_scaler* scaler, int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(comm && exp_avg && exp_avg_sq && step_dev && scaler && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(exp_avg) && aligned16(exp_avg_sq), SOD_EALIGN);
    const AdamRule rule{reinterpret_cast<float4*>(exp_avg), reinterpret_cast<float4*>(exp_avg_sq), step_dev};
    return launch_allreduce_step(comm, grad_off, grad16_off, param_off, rule, shadow16, n, segs, nseg, lr_dev, 1.0f, nullptr,
                                 scaler, flags, stream);
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
