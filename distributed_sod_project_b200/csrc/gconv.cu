// gconv.cu — the 32-group 3×3 convolutions of the weight-standardised GroupNorm ResNeXt-50 32×4d backbone
// (`wsgn_resnext50`, `cp_wsgn_resnext50`): `conv2` of every bottleneck, channels per group (cpg) 4, 8, 16 or 32,
// C_in = C_out = 32·cpg, padding 1, stride 1 or 2, no bias.
//
// Activations are channels-last [N, H, W, C]; Ŵ and dŴ are [C_out][3][3][cpg], the memory order of a channels-last
// master weight.  Per group the convolution is an implicit GEMM with K = 9·cpg, k = tap·cpg + c, tap = 3·kh + kw:
//   fwd    y[p, g·cpg + n]  = Σ_k x[src(p, tap), g·cpg + c] · Ŵ[g·cpg + n][tap][c]
//   dgrad  dx[p, g·cpg + n] = Σ_k dy[dst(p, tap), g·cpg + c] · Ŵ[g·cpg + c][tap][n]
//          (the transposed scatter as a gather: dst(p, tap) = ((h + 1 − kh) / s, (w + 1 − kw) / s) where both divide)
//   wgrad  dŴ[g·cpg + n][tap][c] = Σ_p dy[p, g·cpg + n] · x[src(p, tap), g·cpg + c]
// 16-bit activations run on tensor cores (mma.sync m16n8k16, fp32 accumulation); fp32 activations run in true fp32 on
// FFMA (no TF32).  Every output element is a sum in a fixed order that depends on the shape only, never on the SM
// count: fwd and dgrad accumulate one output per thread (fp32) or per mma lane (16-bit) in k order; wgrad splits the
// N·Ho·Wo pixels into S fixed chunks (gconv_wgrad_geometry, restated by oracle/gconv_geometry.py), writes one fp32
// partial per chunk and adds the S partials in chunk order in a second launch.  No atomics; bit-identical reruns.
#include "common.cuh"

namespace sod {
namespace {

constexpr int kGcThreads = 128;
constexpr int kGcWarps = kGcThreads / 32;
constexpr int kGcTilesPerWarp = 8;       // 16-pixel m-tiles per warp and n-tile (fwd / dgrad, 16-bit)
constexpr int kWgPixels = 32;            // pixels per wgrad staging step
constexpr int kWgMinChunk = 512;         // wgrad: at least this many pixels per chunk …
constexpr int kWgMaxSplit = 32;          // … and at most this many chunks

struct Shape {
    int n, h, w, ho, wo, stride;
    long long P;   // pixels of the convolution's output, n·ho·wo
};

Shape make_shape(int n, int h, int w, int stride) {
    Shape s;
    s.n = n; s.h = h; s.w = w; s.stride = stride;
    s.ho = (h - 1) / stride + 1;
    s.wo = (w - 1) / stride + 1;
    s.P = static_cast<long long>(n) * s.ho * s.wo;
    return s;
}

struct WgGeom {
    int S;          // chunks
    long long pc;   // pixels per chunk (a multiple of kWgPixels; the last chunk may have fewer)
};

// restated by oracle/gconv_geometry.py
WgGeom gconv_wgrad_geometry(long long P) {
    long long s = (P + kWgMinChunk - 1) / kWgMinChunk;
    if (s > kWgMaxSplit) s = kWgMaxSplit;
    if (s < 1) s = 1;
    const long long per = (P + s - 1) / s;
    WgGeom g;
    g.pc = (per + kWgPixels - 1) / kWgPixels * kWgPixels;
    g.S = static_cast<int>((P + g.pc - 1) / g.pc);
    return g;
}

// the input pixel a tap reads for output pixel (b, oh, ow): the forward's window (DGRAD = false) or the transposed
// convolution's gather (DGRAD = true); −1 where the tap falls into the padding or between stride-2 samples
template <bool DGRAD>
__device__ __forceinline__ long long src_pixel(int b, int oh, int ow, int tap, int hi, int wi, int stride) {
    const int kh = tap / 3, kw = tap - 3 * (tap / 3);
    int ih, iw;
    if (DGRAD) {
        const int th = oh + 1 - kh, tw = ow + 1 - kw;
        if (th < 0 || tw < 0) return -1;
        if (stride == 2 && ((th | tw) & 1)) return -1;
        ih = stride == 2 ? th >> 1 : th;
        iw = stride == 2 ? tw >> 1 : tw;
    } else {
        ih = oh * stride - 1 + kh;
        iw = ow * stride - 1 + kw;
        if (ih < 0 || iw < 0) return -1;
    }
    if (ih >= hi || iw >= wi) return -1;
    return (static_cast<long long>(b) * hi + ih) * wi + iw;
}

// ---- fp32: one thread per output pixel and group, cpg accumulators, the group's filters in shared memory ----------
template <int CPG, bool DGRAD>
__global__ void __launch_bounds__(kGcThreads) gconv_simt_kernel(const float* __restrict__ in,
                                                                 const float* __restrict__ wt, float* __restrict__ out,
                                                                 int hi, int wi, int ho, int wo, int stride,
                                                                 long long P) {
    constexpr int C = 32 * CPG;
    __shared__ float sw[9 * CPG * CPG];                  // [tap][c][n]
    const int g = blockIdx.y;
    for (int i = threadIdx.x; i < 9 * CPG * CPG; i += kGcThreads) {
        const int n = i % CPG, c = (i / CPG) % CPG, tap = i / (CPG * CPG);
        sw[i] = DGRAD ? wt[(static_cast<size_t>(g * CPG + c) * 9 + tap) * CPG + n]
                      : wt[(static_cast<size_t>(g * CPG + n) * 9 + tap) * CPG + c];
    }
    __syncthreads();
    const long long p = static_cast<long long>(blockIdx.x) * kGcThreads + threadIdx.x;
    if (p >= P) return;
    const int ow = static_cast<int>(p % wo);
    const long long q = p / wo;
    const int oh = static_cast<int>(q % ho), b = static_cast<int>(q / ho);
    float acc[CPG];
#pragma unroll
    for (int n = 0; n < CPG; ++n) acc[n] = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
        const long long sp = src_pixel<DGRAD>(b, oh, ow, tap, hi, wi, stride);
        if (sp < 0) continue;
        const float* src = in + sp * C + g * CPG;
#pragma unroll
        for (int c0 = 0; c0 < CPG; c0 += 4) {
            const float4 v4 = __ldg(reinterpret_cast<const float4*>(src + c0));
            const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float* wr = sw + (tap * CPG + c0 + k) * CPG;
#pragma unroll
                for (int n = 0; n < CPG; ++n) acc[n] = fmaf(v[k], wr[n], acc[n]);
            }
        }
    }
    float* dst = out + p * C + g * CPG;
#pragma unroll
    for (int n = 0; n < CPG; n += 4)
        *reinterpret_cast<float4*>(dst + n) = make_float4(acc[n], acc[n + 1], acc[n + 2], acc[n + 3]);
}

// ---- 16-bit: tensor cores ------------------------------------------------------------------------------------
template <typename T>
struct Mma;

template <>
struct Mma<__nv_bfloat16> {
    __device__ __forceinline__ static void run(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    __device__ __forceinline__ static uint32_t pack(float lo, float hi) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<const uint32_t*>(&h);
    }
};

template <>
struct Mma<__half> {
    __device__ __forceinline__ static void run(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                     "{%0,%1,%2,%3};\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
    __device__ __forceinline__ static uint32_t pack(float lo, float hi) {
        const __half2 h = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<const uint32_t*>(&h);
    }
};

template <typename T>
__device__ __forceinline__ uint32_t raw16(T v) {
    return static_cast<uint32_t>(*reinterpret_cast<const unsigned short*>(&v));
}

// fwd / dgrad on tensor cores.  A CTA owns one group and kGcWarps·kGcTilesPerWarp / NT m-tiles of 16 output pixels;
// a warp owns one n-tile (8 output channels) of the group, holds its B fragments (the K × 8 slice of Ŵ, K padded to
// a multiple of 16 with zeros) in registers for the whole CTA, and walks its m-tiles.  A fragments are 32-bit loads of
// channel pairs straight from the activation (pairs never straddle a tap: cpg is even); taps in the padding, between
// stride-2 samples or beyond K load zeros.
template <typename T, int CPG, bool DGRAD>
__global__ void __launch_bounds__(kGcThreads) gconv_mma_kernel(const T* __restrict__ in, const T* __restrict__ wt,
                                                                T* __restrict__ out, int hi, int wi, int ho, int wo,
                                                                int stride, long long P) {
    constexpr int C = 32 * CPG, KT = 9 * CPG, KS = (KT + 15) / 16, NT = CPG >= 8 ? CPG / 8 : 1;
    constexpr int MB = kGcWarps * kGcTilesPerWarp / NT;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gid = lane >> 2, t4 = lane & 3;
    const int g = blockIdx.y, j = warp % NT;
    uint32_t bf[KS][2];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int k0 = ks * 16 + 2 * t4 + 8 * hh, n = j * 8 + gid;
            uint32_t v = 0;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int k = k0 + e, tap = k / CPG, c = k % CPG;
                if (k < KT && n < CPG) {
                    const T w = DGRAD ? wt[(static_cast<size_t>(g * CPG + c) * 9 + tap) * CPG + n]
                                      : wt[(static_cast<size_t>(g * CPG + n) * 9 + tap) * CPG + c];
                    v |= raw16(w) << (16 * e);
                }
            }
            bf[ks][hh] = v;
        }
    }
    const long long mt0 = static_cast<long long>(blockIdx.x) * MB;
    for (int i = warp / NT; i < MB; i += kGcWarps / NT) {
        const long long pbase = (mt0 + i) * 16;
        if (pbase >= P) break;
        int rb[2], roh[2], row_[2];
        bool ok[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const long long p = pbase + gid + 8 * r;
            ok[r] = p < P;
            const long long pp = ok[r] ? p : 0;
            row_[r] = static_cast<int>(pp % wo);
            const long long q = pp / wo;
            roh[r] = static_cast<int>(q % ho);
            rb[r] = static_cast<int>(q / ho);
        }
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            uint32_t a[4];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int k = ks * 16 + 2 * t4 + 8 * hh, tap = k / CPG, c = k % CPG;
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    uint32_t v = 0;
                    if (k < KT && ok[r]) {
                        const long long sp = src_pixel<DGRAD>(rb[r], roh[r], row_[r], tap, hi, wi, stride);
                        if (sp >= 0) v = __ldg(reinterpret_cast<const unsigned int*>(in + sp * C + g * CPG + c));
                    }
                    a[2 * hh + r] = v;
                }
            }
            Mma<T>::run(acc, a, bf[ks]);
        }
        const int n = j * 8 + 2 * t4;
        if (n < CPG) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if (!ok[r]) continue;
                const long long p = pbase + gid + 8 * r;
                *reinterpret_cast<uint32_t*>(out + p * C + g * CPG + n) = Mma<T>::pack(acc[2 * r], acc[2 * r + 1]);
            }
        }
    }
}

// ---- wgrad: per (chunk, group) CTA, pixels staged transposed in shared memory --------------------------------------
// xs[m][p] = x[src(p, tap), g·cpg + c] with m = tap·cpg + c, dys[n][p] = dy[p, g·cpg + n], kWgPixels pixels per step.
// 16-bit: dŴᵀ-tile GEMM on tensor cores, M = m (padded to 16), N = n (padded to 8), K = pixels; the warps split the
// (m-tile, n-tile) pairs.  fp32: one thread per (n, m) element, pixel order.
template <typename T>
struct WgSmem {
    using S = T;
    static constexpr int LD = kWgPixels + 8;    // 80-byte rows: the 8 rows of a fragment load hit distinct banks
};
template <>
struct WgSmem<float> {
    using S = float;
    static constexpr int LD = kWgPixels + 1;
};

template <typename T, int CPG>
__global__ void __launch_bounds__(kGcThreads) gconv_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy,
                                                                  float* __restrict__ part, int hi, int wi, int ho,
                                                                  int wo, int stride, long long P, long long pc) {
    constexpr bool kF32 = sizeof(T) == 4;
    constexpr int C = 32 * CPG, KT = 9 * CPG, MR = (KT + 15) / 16 * 16, NR = CPG >= 8 ? CPG : 8;
    constexpr int LD = WgSmem<T>::LD;
    constexpr int VE = CPG * static_cast<int>(sizeof(T)) >= 16 ? 16 / static_cast<int>(sizeof(T)) : CPG;
    using S = typename WgSmem<T>::S;
    __shared__ __align__(16) S xs[MR * LD];
    __shared__ __align__(16) S dys[NR * LD];
    const int g = blockIdx.y, s = blockIdx.x, tid = threadIdx.x;
    const long long pb = static_cast<long long>(s) * pc;
    const long long pe = pb + pc < P ? pb + pc : P;
    for (int i = tid; i < (MR - KT) * LD; i += kGcThreads) xs[KT * LD + i] = S(0.f);
    for (int i = tid; i < (NR - CPG) * LD; i += kGcThreads) dys[CPG * LD + i] = S(0.f);

    constexpr int MT = MR / 16, NTN = NR / 8, TASKS = MT * NTN, TPW = (TASKS + kGcWarps - 1) / kGcWarps;
    constexpr int EPT = (KT * CPG + kGcThreads - 1) / kGcThreads;
    constexpr int NACC = kF32 ? EPT : TPW * 4;
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    const int lane = tid & 31, warp = tid >> 5, gid = lane >> 2, t4 = lane & 3;

    for (long long p0 = pb; p0 < pe; p0 += kWgPixels) {
        __syncthreads();                                   // the previous step's reads are done
        for (int item = tid; item < kWgPixels * 10; item += kGcThreads) {
            const int pp = item % kWgPixels, tap = item / kWgPixels;      // tap 9: the dy row
            const long long p = p0 + pp;
            const T* src = nullptr;
            if (p < pe) {
                const int ow = static_cast<int>(p % wo);
                const long long q = p / wo;
                const int oh = static_cast<int>(q % ho), b = static_cast<int>(q / ho);
                if (tap == 9) {
                    src = dy + p * C + g * CPG;
                } else {
                    const long long sp = src_pixel<false>(b, oh, ow, tap, hi, wi, stride);
                    if (sp >= 0) src = x + sp * C + g * CPG;
                }
            }
            S* dst = tap == 9 ? dys + pp : xs + tap * CPG * LD + pp;
#pragma unroll
            for (int c0 = 0; c0 < CPG; c0 += VE) {
                __align__(16) T v[VE];
                if (src != nullptr) {
                    if constexpr (VE * sizeof(T) == 16) *reinterpret_cast<uint4*>(v) = __ldg(reinterpret_cast<const uint4*>(src + c0));
                    else *reinterpret_cast<uint2*>(v) = __ldg(reinterpret_cast<const uint2*>(src + c0));
                } else {
#pragma unroll
                    for (int e = 0; e < VE; ++e) v[e] = T(0.f);
                }
#pragma unroll
                for (int e = 0; e < VE; ++e) dst[(c0 + e) * LD] = v[e];
            }
        }
        __syncthreads();
        if constexpr (kF32) {
#pragma unroll
            for (int i = 0; i < EPT; ++i) {
                const int e = tid + i * kGcThreads;
                if (e < KT * CPG) {
                    const int n = e / KT, m = e - n * KT;
                    float a = acc[i];
                    for (int pp = 0; pp < kWgPixels; ++pp) a = fmaf(dys[n * LD + pp], xs[m * LD + pp], a);
                    acc[i] = a;
                }
            }
        } else {
#pragma unroll
            for (int ks = 0; ks < kWgPixels / 16; ++ks) {
#pragma unroll
                for (int ti = 0; ti < TPW; ++ti) {
                    const int task = warp + ti * kGcWarps;
                    if (task < TASKS) {
                        const int mt = task / NTN, nt = task % NTN;
                        const S* xa = xs + (mt * 16 + gid) * LD + ks * 16 + 2 * t4;
                        const S* db = dys + (nt * 8 + gid) * LD + ks * 16 + 2 * t4;
                        uint32_t a[4], bb[2];
                        a[0] = *reinterpret_cast<const uint32_t*>(xa);
                        a[1] = *reinterpret_cast<const uint32_t*>(xa + 8 * LD);
                        a[2] = *reinterpret_cast<const uint32_t*>(xa + 8);
                        a[3] = *reinterpret_cast<const uint32_t*>(xa + 8 * LD + 8);
                        bb[0] = *reinterpret_cast<const uint32_t*>(db);
                        bb[1] = *reinterpret_cast<const uint32_t*>(db + 8);
                        float* d = acc + 4 * ti;
                        float d4[4] = {d[0], d[1], d[2], d[3]};
                        Mma<T>::run(d4, a, bb);
                        d[0] = d4[0]; d[1] = d4[1]; d[2] = d4[2]; d[3] = d4[3];
                    }
                }
            }
        }
    }
    // partial of chunk s: [C][KT] fp32, the dŴ order
    float* mine = part + static_cast<size_t>(s) * C * KT + static_cast<size_t>(g) * CPG * KT;
    if constexpr (kF32) {
#pragma unroll
        for (int i = 0; i < EPT; ++i) {
            const int e = tid + i * kGcThreads;
            if (e < KT * CPG) mine[e] = acc[i];           // e = n·KT + m
        }
    } else {
#pragma unroll
        for (int ti = 0; ti < TPW; ++ti) {
            const int task = warp + ti * kGcWarps;
            if (task >= TASKS) continue;
            const int mt = task / NTN, nt = task % NTN;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int m = mt * 16 + gid + 8 * (r >> 1), n = nt * 8 + 2 * t4 + (r & 1);
                if (m < KT && n < CPG) mine[n * KT + m] = acc[4 * ti + r];
            }
        }
    }
}

__global__ void __launch_bounds__(256) gconv_wgrad_merge_kernel(const float* __restrict__ part, float* __restrict__ dw,
                                                                  long long len, int S) {
    for (long long i = blockIdx.x * 256ll + threadIdx.x; i < len; i += static_cast<long long>(gridDim.x) * 256) {
        float t = part[i];
        for (int s = 1; s < S; ++s) t += part[static_cast<size_t>(s) * len + i];
        dw[i] = t;
    }
}

int gc_check(int n, int h, int w, int c, int groups, int stride, int dtype) {
    SOD_CHECK_ARG(n > 0 && h > 0 && w > 0 && c > 0 && groups > 0, SOD_EINVAL);
    SOD_CHECK_ARG(dtype == SOD_F32 || dtype == SOD_BF16 || dtype == SOD_F16, SOD_EINVAL);
    SOD_CHECK_ARG(c % groups == 0, SOD_EINVAL);
    SOD_CHECK_ARG(groups == SOD_GCONV_GROUPS, SOD_EUNSUPPORTED);
    const int cpg = c / groups;
    SOD_CHECK_ARG(cpg == 4 || cpg == 8 || cpg == 16 || cpg == 32, SOD_EUNSUPPORTED);
    SOD_CHECK_ARG(stride == 1 || stride == 2, SOD_EUNSUPPORTED);
    // pixel indices are 64-bit; the grid's x dimension and the spatial indices are not
    SOD_CHECK_ARG(static_cast<long long>(n) * h * w <= (1ll << 31) - 1, SOD_EUNSUPPORTED);
    return SOD_OK;
}

// fwd (DGRAD = false: in = x, out = y) or dgrad (in = dy, out = dx); (h, w) is always the size of x
template <bool DGRAD>
int gc_launch(const void* in, const void* wt, void* out, int dtype, const Shape& sh, int cpg, cudaStream_t st) {
    const int hi = DGRAD ? sh.ho : sh.h, wi = DGRAD ? sh.wo : sh.w;
    const int ho = DGRAD ? sh.h : sh.ho, wo = DGRAD ? sh.w : sh.wo;
    const long long P = static_cast<long long>(sh.n) * ho * wo;
    auto simt = [&](auto cpg_tag) -> int {
        constexpr int CPG = decltype(cpg_tag)::value;
        const dim3 grid(static_cast<unsigned>((P + kGcThreads - 1) / kGcThreads), SOD_GCONV_GROUPS);
        gconv_simt_kernel<CPG, DGRAD><<<grid, kGcThreads, 0, st>>>(static_cast<const float*>(in),
                                                                   static_cast<const float*>(wt),
                                                                   static_cast<float*>(out), hi, wi, ho, wo, sh.stride, P);
        return static_cast<int>(cudaGetLastError());
    };
    auto mma = [&](auto t_tag, auto cpg_tag) -> int {
        using T = decltype(t_tag);
        constexpr int CPG = decltype(cpg_tag)::value;
        constexpr int NT = CPG >= 8 ? CPG / 8 : 1;
        const long long pixels_per_cta = 16ll * kGcWarps * kGcTilesPerWarp / NT;
        const dim3 grid(static_cast<unsigned>((P + pixels_per_cta - 1) / pixels_per_cta), SOD_GCONV_GROUPS);
        gconv_mma_kernel<T, CPG, DGRAD><<<grid, kGcThreads, 0, st>>>(
            static_cast<const T*>(in), static_cast<const T*>(wt), static_cast<T*>(out), hi, wi, ho, wo, sh.stride, P);
        return static_cast<int>(cudaGetLastError());
    };
    auto by_cpg = [&](auto fn, auto... t) -> int {
        switch (cpg) {
            case 4: return fn(t..., std::integral_constant<int, 4>{});
            case 8: return fn(t..., std::integral_constant<int, 8>{});
            case 16: return fn(t..., std::integral_constant<int, 16>{});
            default: return fn(t..., std::integral_constant<int, 32>{});
        }
    };
    if (dtype == SOD_F32) return by_cpg(simt);
    if (dtype == SOD_BF16) return by_cpg(mma, __nv_bfloat16{});
    return by_cpg(mma, __half{});
}

}  // namespace
}  // namespace sod

extern "C" int sod_gconv3x3_fwd(const void* x, const void* w_hat, void* y, int dtype, int n, int h, int w, int c,
                                int groups, int stride, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && w_hat && y, SOD_EINVAL);
    const int rc = gc_check(n, h, w, c, groups, stride, dtype);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(aligned16(x) && aligned16(w_hat) && aligned16(y), SOD_EALIGN);
    return gc_launch<false>(x, w_hat, y, dtype, make_shape(n, h, w, stride), c / groups,
                            static_cast<cudaStream_t>(stream));
}

extern "C" int sod_gconv3x3_dgrad(const void* dy, const void* w_hat, void* dx, int dtype, int n, int h, int w, int c,
                                  int groups, int stride, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && w_hat && dx, SOD_EINVAL);
    const int rc = gc_check(n, h, w, c, groups, stride, dtype);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(aligned16(dy) && aligned16(w_hat) && aligned16(dx), SOD_EALIGN);
    return gc_launch<true>(dy, w_hat, dx, dtype, make_shape(n, h, w, stride), c / groups,
                           static_cast<cudaStream_t>(stream));
}

extern "C" int sod_gconv3x3_wgrad_splits(int n, int h, int w, int c, int groups, int stride) {
    using namespace sod;
    if (gc_check(n, h, w, c, groups, stride, SOD_F32) != SOD_OK) return 0;
    return gconv_wgrad_geometry(make_shape(n, h, w, stride).P).S;
}

extern "C" size_t sod_gconv3x3_wgrad_workspace_bytes(int n, int h, int w, int c, int groups, int stride) {
    using namespace sod;
    if (gc_check(n, h, w, c, groups, stride, SOD_F32) != SOD_OK) return 0;
    const WgGeom g = gconv_wgrad_geometry(make_shape(n, h, w, stride).P);
    return static_cast<size_t>(g.S) * c * 9 * (c / groups) * sizeof(float);
}

extern "C" int sod_gconv3x3_wgrad(const void* x, const void* dy, float* dw_hat, int dtype, int n, int h, int w, int c,
                                  int groups, int stride, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && dy && dw_hat && workspace, SOD_EINVAL);
    const int rc = gc_check(n, h, w, c, groups, stride, dtype);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(aligned16(x) && aligned16(dy) && aligned16(dw_hat) && aligned16(workspace), SOD_EALIGN);
    const Shape sh = make_shape(n, h, w, stride);
    const WgGeom g = gconv_wgrad_geometry(sh.P);
    const int cpg = c / groups;
    const long long len = static_cast<long long>(c) * 9 * cpg;
    SOD_CHECK_ARG(workspace_bytes >= static_cast<size_t>(g.S) * len * sizeof(float), SOD_EWORKSPACE);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* part = static_cast<float*>(workspace);
    auto run = [&](auto t_tag, auto cpg_tag) -> int {
        using T = decltype(t_tag);
        constexpr int CPG = decltype(cpg_tag)::value;
        gconv_wgrad_kernel<T, CPG><<<dim3(g.S, SOD_GCONV_GROUPS), kGcThreads, 0, st>>>(
            static_cast<const T*>(x), static_cast<const T*>(dy), part, sh.h, sh.w, sh.ho, sh.wo, sh.stride, sh.P, g.pc);
        return static_cast<int>(cudaGetLastError());
    };
    auto by_cpg = [&](auto t) -> int {
        switch (cpg) {
            case 4: return run(t, std::integral_constant<int, 4>{});
            case 8: return run(t, std::integral_constant<int, 8>{});
            case 16: return run(t, std::integral_constant<int, 16>{});
            default: return run(t, std::integral_constant<int, 32>{});
        }
    };
    int e = dtype == SOD_F32 ? by_cpg(float{}) : dtype == SOD_BF16 ? by_cpg(__nv_bfloat16{}) : by_cpg(__half{});
    if (e != 0) return e;
    long long blocks = (len + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    gconv_wgrad_merge_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(part, dw_hat, len, g.S);
    return static_cast<int>(cudaGetLastError());
}
