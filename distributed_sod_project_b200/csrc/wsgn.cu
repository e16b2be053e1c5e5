// wsgn.cu — GroupNorm(32) with the bottleneck's residual-add / ReLU epilogue, and weight standardisation, for the
// weight-standardised GroupNorm ResNet-50 backbone (`wsgn_res50`, `cp_wsgn_res50`).
//
// GroupNorm works on channels-last [N·HW, C] matrices.  Statistics are per (sample, group), so no rank exchange is
// involved at any world size.  A sample is split over S CTAs (gn_geometry); each CTA reduces its row chunk, writes a
// per-CTA partial, and the last CTA of the sample to finish (integer ticket, as in resample.cu's colsum) merges the S
// partials in CTA order.  No floating-point atomics and no grid-wide wait: every result is a fixed-order sum, so a
// launch is bit-identical from run to run.  Two launches per direction: reduce (+ ticket merge), then the elementwise
// pass that reads the merged values.
//
// Statistics: every thread sums (x − s) and (x − s)² of its 8 channels with s the channel's value in the sample's
// first row, the CTA turns them into per-channel (mean, M2) and merges the group's channels and then the S CTA partials
// by Chan's pairwise rule — the (mean, M2) merge of syncbn.cu's exchange_moments, never Σx and Σx².  The shift takes
// the mean out of the sums, so a large mean costs nothing; what remains is the cancellation in Σd² − (Σd)²/n, a
// relative error of about u·((s − μ)/σ)² in the variance.  s is one sample of the data, so that factor is small unless
// row 0 is an outlier far beyond the spread of its group (tests/test_gpu_wsgn_kernels.py covers 10σ).
#include "common.cuh"

namespace sod {
namespace {

constexpr int kGnThreads = 256;
constexpr int kGnMaxC = 2048;
constexpr int kGnMaxSplit = 1024;

struct GnGeom {
    int L, R, S;       // lanes of 8 channels, rows per pass, CTAs per sample
    long long rc;      // rows per CTA (the last CTA of a sample may have fewer)
};

// restated by oracle/wsgn_geometry.py: ≥ 8 row passes per thread, about two CTAs per SM over the whole batch, no
// empty CTA
GnGeom gn_geometry(int n, long long hw, int c, int sm_count) {
    GnGeom g;
    g.L = c / 8;
    g.R = kGnThreads / g.L;
    const long long want = (2ll * sm_count + n - 1) / n;
    const long long min_rows = 8ll * g.R;
    const long long most = (hw + min_rows - 1) / min_rows;
    long long s = want < most ? want : most;
    if (s > kGnMaxSplit) s = kGnMaxSplit;
    if (s < 1) s = 1;
    g.rc = (hw + s - 1) / s;
    g.S = static_cast<int>((hw + g.rc - 1) / g.rc);
    return g;
}

size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

struct GnWork {
    unsigned* ticket;   // [n + 1]: per sample, and one for the whole launch (backward's dγ/dβ)
    float2* part;       // forward: [n·S·G] (mean, M2); backward: [n·S·C] (Σdz, Σdz·x̂)
    float2* dsum;       // backward: [n·C] (Σdz, Σdz·x̂) per sample
    float2* coef;       // backward: [n·G] (Σγ·dz / M, Σγ·dz·x̂ / M)
};

size_t gn_work_bytes(int n, const GnGeom& g, int c, int groups) {
    const size_t part = static_cast<size_t>(n) * g.S * (c > groups ? c : groups) * sizeof(float2);
    return align256(sizeof(unsigned) * (n + 1)) + align256(part) + align256(sizeof(float2) * n * c) +
           align256(sizeof(float2) * n * groups);
}

GnWork gn_work(void* ws, int n, const GnGeom& g, int c, int groups) {
    char* p = static_cast<char*>(ws);
    GnWork w;
    w.ticket = reinterpret_cast<unsigned*>(p);
    p += align256(sizeof(unsigned) * (n + 1));
    w.part = reinterpret_cast<float2*>(p);
    p += align256(static_cast<size_t>(n) * g.S * (c > groups ? c : groups) * sizeof(float2));
    w.dsum = reinterpret_cast<float2*>(p);
    p += align256(sizeof(float2) * n * c);
    w.coef = reinterpret_cast<float2*>(p);
    return w;
}

// Chan's merge of (count na, mean ma, M2 qa) with (nb, mb, qb)
__device__ __forceinline__ void chan_merge(float& na, float& ma, float& qa, float nb, float mb, float qb) {
    const float n = na + nb;
    const float d = mb - ma;
    const float f = nb / n;
    ma = ma + d * f;
    qa = qa + qb + d * d * na * f;
    na = n;
}

// ---- forward, launch 1: statistics --------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(const T* __restrict__ x, float2* __restrict__ stats,
                                                                long long hw, int L, int S, long long rc, int groups,
                                                                float eps, GnWork w) {
    __shared__ float s_acc[2][kGnThreads * 8];
    __shared__ float s_mean[kGnMaxC], s_m2[kGnMaxC];
    __shared__ bool s_last;
    const int tid = threadIdx.x, n = blockIdx.y, s = blockIdx.x;
    const int R = kGnThreads / L, C = 8 * L, l = tid % L, r0 = tid / L;
    const int cg = C / groups;
    const T* xs = x + static_cast<size_t>(n) * hw * C;
    const long long rb = static_cast<long long>(s) * rc;
    const long long re = rb + rc < hw ? rb + rc : hw;
    float a1[8], a2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a1[k] = a2[k] = 0.f;
    if (r0 < R) {
        float sh[8];
        IO<T>::load8(xs + l * 8, sh);                       // the shift: row 0 of the sample, the same in every CTA
#pragma unroll 2
        for (long long r = rb + r0; r < re; r += R) {
            float v[8];
            IO<T>::load8(xs + r * C + l * 8, v);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float d = v[k] - sh[k];
                a1[k] += d;
                a2[k] = fmaf(d, d, a2[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) { s_acc[0][tid * 8 + k] = a1[k]; s_acc[1][tid * 8 + k] = a2[k]; }
    __syncthreads();
    const float nb = static_cast<float>(re - rb);
    for (int ch = tid; ch < C; ch += kGnThreads) {
        const int ll = ch >> 3, k = ch & 7;
        float t1 = 0.f, t2 = 0.f;
        for (int rr = 0; rr < R; ++rr) {
            t1 += s_acc[0][(rr * L + ll) * 8 + k];
            t2 += s_acc[1][(rr * L + ll) * 8 + k];
        }
        const float shv = IO<T>::load1(xs + ch);
        s_mean[ch] = shv + t1 / nb;
        s_m2[ch] = fmaxf(t2 - t1 * (t1 / nb), 0.f);
    }
    __syncthreads();
    float2* mine = w.part + (static_cast<size_t>(n) * S + s) * groups;
    for (int g = tid; g < groups; g += kGnThreads) {
        float cnt = nb, m = s_mean[g * cg], q = s_m2[g * cg];
        for (int j = 1; j < cg; ++j) chan_merge(cnt, m, q, nb, s_mean[g * cg + j], s_m2[g * cg + j]);
        mine[g] = make_float2(m, q);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(w.ticket + n, 1u) == static_cast<unsigned>(S - 1));
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const float2* all = w.part + static_cast<size_t>(n) * S * groups;
    for (int g = tid; g < groups; g += kGnThreads) {
        const float2 p0 = __ldcg(all + g);
        float cnt = static_cast<float>(rc < hw ? rc : hw) * cg, m = p0.x, q = p0.y;
        for (int b = 1; b < S; ++b) {
            const long long bb = static_cast<long long>(b) * rc;
            const long long be = bb + rc < hw ? bb + rc : hw;
            const float2 p = __ldcg(all + static_cast<size_t>(b) * groups + g);
            chan_merge(cnt, m, q, static_cast<float>(be - bb) * cg, p.x, p.y);
        }
        const float var = q / cnt;                          // biased, as nn.GroupNorm normalises
        stats[static_cast<size_t>(n) * groups + g] = make_float2(m, 1.0f / sqrtf(var + eps));
    }
    if (tid == 0) w.ticket[n] = 0;                          // ready for the next launch on this stream
}

// ---- forward, launch 2: y = act((x − μ)·rstd·γ + β [+ residual]) ----------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kGnThreads) gn_apply_kernel(const T* __restrict__ x, const T* __restrict__ res,
                                                                T* __restrict__ y, const float* __restrict__ gamma,
                                                                const float* __restrict__ beta,
                                                                const float2* __restrict__ stats, long long hw, int L,
                                                                int groups, int relu, long long packets) {
    const int C = 8 * L, cg = C / groups;
    for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < packets;
         p += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = p / L;
        const int l = static_cast<int>(p - r * L);
        const int n = static_cast<int>(r / hw);
        const size_t off = static_cast<size_t>(r) * C + l * 8;
        float v[8], o[8];
        IO<T>::load8(x + off, v);
        if (res != nullptr) IO<T>::load8(res + off, o);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ch = l * 8 + k;
            const float2 st = stats[static_cast<size_t>(n) * groups + ch / cg];
            float t = fmaf((v[k] - st.x) * st.y, gamma[ch], beta[ch]);
            if (res != nullptr) t += o[k];
            v[k] = relu ? fmaxf(t, 0.f) : t;
        }
        IO<T>::store8(y + off, v);
    }
}

// ---- backward, launch 1: Σdz and Σdz·x̂ per (sample, channel), then per group and over the batch ----------------
template <typename T>
__global__ void __launch_bounds__(kGnThreads) gn_bwd_reduce_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                     const T* __restrict__ y,
                                                                     const float* __restrict__ gamma,
                                                                     const float2* __restrict__ stats,
                                                                     float* __restrict__ dgamma,
                                                                     float* __restrict__ dbeta, long long hw, int L,
                                                                     int S, long long rc, int groups, int accumulate,
                                                                     GnWork w) {
    __shared__ float s_acc[2][kGnThreads * 8];
    __shared__ float s_g[2][kGnMaxC];
    __shared__ bool s_last;
    const int tid = threadIdx.x, n = blockIdx.y, s = blockIdx.x, N = gridDim.y;
    const int R = kGnThreads / L, C = 8 * L, l = tid % L, r0 = tid / L;
    const int cg = C / groups;
    const size_t base = static_cast<size_t>(n) * hw * C;
    const long long rb = static_cast<long long>(s) * rc;
    const long long re = rb + rc < hw ? rb + rc : hw;
    float a1[8], a2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a1[k] = a2[k] = 0.f;
    if (r0 < R) {
        float mu[8], rs[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float2 st = stats[static_cast<size_t>(n) * groups + (l * 8 + k) / cg];
            mu[k] = st.x; rs[k] = st.y;
        }
#pragma unroll 2
        for (long long r = rb + r0; r < re; r += R) {
            const size_t off = base + static_cast<size_t>(r) * C + l * 8;
            float g[8], v[8];
            IO<T>::load8(dy + off, g);
            IO<T>::load8(x + off, v);
            if (y != nullptr) {
                float o[8];
                IO<T>::load8(y + off, o);
#pragma unroll
                for (int k = 0; k < 8; ++k) g[k] = o[k] > 0.f ? g[k] : 0.f;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                a1[k] += g[k];
                a2[k] = fmaf(g[k], (v[k] - mu[k]) * rs[k], a2[k]);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) { s_acc[0][tid * 8 + k] = a1[k]; s_acc[1][tid * 8 + k] = a2[k]; }
    __syncthreads();
    float2* mine = w.part + (static_cast<size_t>(n) * S + s) * C;
    for (int ch = tid; ch < C; ch += kGnThreads) {
        const int ll = ch >> 3, k = ch & 7;
        float t1 = 0.f, t2 = 0.f;
        for (int rr = 0; rr < R; ++rr) {
            t1 += s_acc[0][(rr * L + ll) * 8 + k];
            t2 += s_acc[1][(rr * L + ll) * 8 + k];
        }
        mine[ch] = make_float2(t1, t2);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(w.ticket + n, 1u) == static_cast<unsigned>(S - 1));
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // the last CTA of sample n: the sample's per-channel sums in CTA order, and the per-group coefficients of dx
    const float2* all = w.part + static_cast<size_t>(n) * S * C;
    for (int ch = tid; ch < C; ch += kGnThreads) {
        float t1 = 0.f, t2 = 0.f;
        for (int b = 0; b < S; ++b) {
            const float2 p = __ldcg(all + static_cast<size_t>(b) * C + ch);
            t1 += p.x; t2 += p.y;
        }
        s_g[0][ch] = t1; s_g[1][ch] = t2;
        w.dsum[static_cast<size_t>(n) * C + ch] = make_float2(t1, t2);
    }
    __syncthreads();
    const float inv_m = 1.0f / (static_cast<float>(hw) * cg);
    for (int g = tid; g < groups; g += kGnThreads) {
        float ca = 0.f, cb = 0.f;
        for (int j = 0; j < cg; ++j) {
            const int ch = g * cg + j;
            ca = fmaf(gamma[ch], s_g[0][ch], ca);
            cb = fmaf(gamma[ch], s_g[1][ch], cb);
        }
        w.coef[static_cast<size_t>(n) * groups + g] = make_float2(ca * inv_m, cb * inv_m);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        w.ticket[n] = 0;
        s_last = (atomicAdd(w.ticket + N, 1u) == static_cast<unsigned>(N - 1));
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    // the last sample to finish: dγ, dβ as sums over the samples in order
    for (int ch = tid; ch < C; ch += kGnThreads) {
        float t1 = 0.f, t2 = 0.f;
        for (int b = 0; b < N; ++b) {
            const float2 p = __ldcg(w.dsum + static_cast<size_t>(b) * C + ch);
            t1 += p.x; t2 += p.y;
        }
        if (accumulate) { dbeta[ch] += t1; dgamma[ch] += t2; }
        else { dbeta[ch] = t1; dgamma[ch] = t2; }
    }
    if (tid == 0) w.ticket[N] = 0;
}

// ---- backward, launch 2: dx = (γ·dz − A − x̂·B)·rstd, dres = dz --------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kGnThreads) gn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                    const T* __restrict__ y, T* __restrict__ dx,
                                                                    T* __restrict__ dres, const float* __restrict__ gamma,
                                                                    const float2* __restrict__ stats,
                                                                    const float2* __restrict__ coef, long long hw,
                                                                    int L, int groups, long long packets) {
    const int C = 8 * L, cg = C / groups;
    for (long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; p < packets;
         p += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = p / L;
        const int l = static_cast<int>(p - r * L);
        const int n = static_cast<int>(r / hw);
        const size_t off = static_cast<size_t>(r) * C + l * 8;
        float g[8], v[8];
        IO<T>::load8(dy + off, g);
        IO<T>::load8(x + off, v);
        if (y != nullptr) {
            float o[8];
            IO<T>::load8(y + off, o);
#pragma unroll
            for (int k = 0; k < 8; ++k) g[k] = o[k] > 0.f ? g[k] : 0.f;
        }
        if (dres != nullptr) IO<T>::store8(dres + off, g);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int ch = l * 8 + k;
            const size_t gi = static_cast<size_t>(n) * groups + ch / cg;
            const float2 st = stats[gi];
            const float2 cf = coef[gi];
            const float xh = (v[k] - st.x) * st.y;
            v[k] = (fmaf(gamma[ch], g[k], -cf.x) - xh * cf.y) * st.y;
        }
        IO<T>::store8(dx + off, v);
    }
}

unsigned elementwise_grid(long long packets) {
    long long grid = (packets + kGnThreads - 1) / kGnThreads;
    const long long cap = 8ll * dev_info().sm_count;
    if (grid > cap) grid = cap;
    return static_cast<unsigned>(grid < 1 ? 1 : grid);
}

// ------------------------------------------------------------------------------------------------
// weight standardisation, one CTA per filter (output channel) of K = C·R·S weights, in the weight's own memory order
// (the operation is the same map for every permutation of a filter's elements, so NCHW and channels-last weights are
// both dense per filter):
//   μ = Σw / K,  v = w − μ,  σ = sqrt(Σv² / (K − 1)),  s = σ + eps,  ŵ = v / s
// The backward recomputes μ, σ with the same code (bit-identical to the forward's) and forms, with g = dŵ,
//   dw = (g − Σg / K) / s − v · (Σg·v / (s · s · (K − 1) · σ))
// which is the derivative of the reference's expression: the σ path contributes −v·Σg·v / (s²·(K−1)·σ), and the
// centring's mean of it vanishes because Σv = 0.
// ------------------------------------------------------------------------------------------------
constexpr int kWsThreads = 256;

__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();                                     // red may still be read by a previous call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = 0.f;
    for (int i = 0; i < kWsThreads / 32; ++i) t += red[i];
    return t;
}

__device__ __forceinline__ void ws_moments(const float* wf, int K, float* red, float& mu, float& sigma) {
    float a = 0.f;
    for (int i = threadIdx.x; i < K; i += kWsThreads) a += wf[i];
    mu = block_sum(a, red) / static_cast<float>(K);
    float q = 0.f;
    for (int i = threadIdx.x; i < K; i += kWsThreads) {
        const float d = wf[i] - mu;
        q = fmaf(d, d, q);
    }
    sigma = sqrtf(block_sum(q, red) / static_cast<float>(K - 1));
}

template <typename T>
__global__ void __launch_bounds__(kWsThreads) ws_fwd_kernel(const float* __restrict__ w, T* __restrict__ w_hat, int K,
                                                             float eps) {
    __shared__ float red[kWsThreads / 32];
    const float* wf = w + static_cast<size_t>(blockIdx.x) * K;
    T* of = w_hat + static_cast<size_t>(blockIdx.x) * K;
    float mu, sigma;
    ws_moments(wf, K, red, mu, sigma);
    const float s = sigma + eps;
    for (int i = threadIdx.x; i < K; i += kWsThreads) IO<T>::store1(of + i, (wf[i] - mu) / s);
}

template <typename T>
__global__ void __launch_bounds__(kWsThreads) ws_bwd_kernel(const float* __restrict__ w, const T* __restrict__ dw_hat,
                                                             float* __restrict__ dw, int K, float eps, int accumulate) {
    __shared__ float red[kWsThreads / 32];
    const size_t base = static_cast<size_t>(blockIdx.x) * K;
    const float* wf = w + base;
    const T* gf = dw_hat + base;
    float mu, sigma;
    ws_moments(wf, K, red, mu, sigma);
    const float s = sigma + eps;
    float a = 0.f, b = 0.f;
    for (int i = threadIdx.x; i < K; i += kWsThreads) {
        const float g = IO<T>::load1(gf + i);
        a += g;
        b = fmaf(g, wf[i] - mu, b);
    }
    const float sg = block_sum(a, red);
    const float sgv = block_sum(b, red);
    const float mg = sg / static_cast<float>(K);
    const float coef = sgv / (s * s * static_cast<float>(K - 1) * sigma);
    for (int i = threadIdx.x; i < K; i += kWsThreads) {
        const float v = wf[i] - mu;
        const float d = (IO<T>::load1(gf + i) - mg) / s - v * coef;
        if (accumulate) dw[base + i] += d;
        else dw[base + i] = d;
    }
}

size_t dtype_bytes(int dtype) { return dtype == SOD_F32 ? 4 : 2; }

bool aligned_to(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

int gn_check(int n, long long hw, int c, int groups, int dtype) {
    SOD_CHECK_ARG(n > 0 && hw > 0 && c > 0 && groups > 0, SOD_EINVAL);
    SOD_CHECK_ARG(dtype == SOD_F32 || dtype == SOD_BF16 || dtype == SOD_F16, SOD_EINVAL);
    SOD_CHECK_ARG(c % groups == 0, SOD_EINVAL);
    SOD_CHECK_ARG(groups == SOD_GN_GROUPS, SOD_EUNSUPPORTED);
    const int L = c / 8;
    SOD_CHECK_ARG(c % 8 == 0 && c <= kGnMaxC && (L & (L - 1)) == 0, SOD_EUNSUPPORTED);
    SOD_CHECK_ARG(n <= 65535, SOD_EUNSUPPORTED);
    return SOD_OK;
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_groupnorm_workspace_bytes(int n, int64_t hw, int c, int groups) {
    using namespace sod;
    if (gn_check(n, hw, c, groups, SOD_F32) != SOD_OK) return 0;
    return gn_work_bytes(n, gn_geometry(n, hw, c, dev_info().sm_count), c, groups);
}

extern "C" int sod_groupnorm_splits(int n, int64_t hw, int c, int groups) {
    using namespace sod;
    if (gn_check(n, hw, c, groups, SOD_F32) != SOD_OK) return 0;
    return gn_geometry(n, hw, c, dev_info().sm_count).S;
}

extern "C" int sod_groupnorm_fwd(const void* x, const void* residual, void* y, int dtype, const float* gamma,
                                 const float* beta, float* save_stats, int n, int64_t hw, int c, int groups, float eps,
                                 int relu, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && y && gamma && beta && save_stats && workspace, SOD_EINVAL);
    const int rc = gn_check(n, hw, c, groups, dtype);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(eps >= 0.f, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(x) && aligned16(y) && (residual == nullptr || aligned16(residual)) && aligned16(workspace) &&
                      aligned_to(save_stats, 8) && aligned_to(gamma, 4) && aligned_to(beta, 4),
                  SOD_EALIGN);
    const GnGeom g = gn_geometry(n, hw, c, dev_info().sm_count);
    SOD_CHECK_ARG(workspace_bytes >= gn_work_bytes(n, g, c, groups), SOD_EWORKSPACE);
    const GnWork w = gn_work(workspace, n, g, c, groups);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    float2* stats = reinterpret_cast<float2*>(save_stats);
    const long long packets = static_cast<long long>(n) * hw * g.L;
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        gn_stats_kernel<T><<<dim3(g.S, n), kGnThreads, 0, s>>>(static_cast<const T*>(x), stats, hw, g.L, g.S, g.rc,
                                                               groups, eps, w);
        gn_apply_kernel<T><<<elementwise_grid(packets), kGnThreads, 0, s>>>(
            static_cast<const T*>(x), static_cast<const T*>(residual), static_cast<T*>(y), gamma, beta, stats, hw, g.L,
            groups, relu, packets);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_groupnorm_bwd(const void* dy, const void* x, const void* y, void* dx, void* dres, int dtype,
                                 const float* gamma, const float* save_stats, float* dgamma, float* dbeta, int n,
                                 int64_t hw, int c, int groups, int relu, void* workspace, size_t workspace_bytes,
                                 int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && x && dx && gamma && save_stats && dgamma && dbeta && workspace, SOD_EINVAL);
    SOD_CHECK_ARG(!relu || y != nullptr, SOD_EINVAL);
    const int rc = gn_check(n, hw, c, groups, dtype);
    if (rc != SOD_OK) return rc;
    SOD_CHECK_ARG(aligned16(dy) && aligned16(x) && aligned16(dx) && (y == nullptr || aligned16(y)) &&
                      (dres == nullptr || aligned16(dres)) && aligned16(workspace) && aligned_to(save_stats, 8) &&
                      aligned_to(gamma, 4) && aligned_to(dgamma, 4) && aligned_to(dbeta, 4),
                  SOD_EALIGN);
    const GnGeom g = gn_geometry(n, hw, c, dev_info().sm_count);
    SOD_CHECK_ARG(workspace_bytes >= gn_work_bytes(n, g, c, groups), SOD_EWORKSPACE);
    const GnWork w = gn_work(workspace, n, g, c, groups);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const float2* stats = reinterpret_cast<const float2*>(save_stats);
    const long long packets = static_cast<long long>(n) * hw * g.L;
    const int accumulate = (flags & SOD_BN_ACCUMULATE_PARAM_GRADS) != 0;
    const void* ymask = relu ? y : nullptr;
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        gn_bwd_reduce_kernel<T><<<dim3(g.S, n), kGnThreads, 0, s>>>(
            static_cast<const T*>(dy), static_cast<const T*>(x), static_cast<const T*>(ymask), gamma, stats, dgamma,
            dbeta, hw, g.L, g.S, g.rc, groups, accumulate, w);
        gn_bwd_apply_kernel<T><<<elementwise_grid(packets), kGnThreads, 0, s>>>(
            static_cast<const T*>(dy), static_cast<const T*>(x), static_cast<const T*>(ymask), static_cast<T*>(dx),
            static_cast<T*>(dres), gamma, stats, w.coef, hw, g.L, groups, packets);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_ws_fwd(const float* w, void* w_hat, int dtype, int filters, int k, float eps, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(w && w_hat && filters > 0 && k > 1 && eps >= 0.f, SOD_EINVAL);
    SOD_CHECK_ARG(dtype == SOD_F32 || dtype == SOD_BF16 || dtype == SOD_F16, SOD_EINVAL);
    SOD_CHECK_ARG(aligned_to(w, 4) && aligned_to(w_hat, dtype_bytes(dtype)), SOD_EALIGN);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        ws_fwd_kernel<T><<<filters, kWsThreads, 0, s>>>(w, static_cast<T*>(w_hat), k, eps);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_ws_bwd(const float* w, const void* dw_hat, int dtype, float* dw, int filters, int k, float eps,
                          int flags, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(w && dw_hat && dw && filters > 0 && k > 1 && eps >= 0.f, SOD_EINVAL);
    SOD_CHECK_ARG(dtype == SOD_F32 || dtype == SOD_BF16 || dtype == SOD_F16, SOD_EINVAL);
    SOD_CHECK_ARG(aligned_to(w, 4) && aligned_to(dw, 4) && aligned_to(dw_hat, dtype_bytes(dtype)), SOD_EALIGN);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int accumulate = (flags & SOD_BN_ACCUMULATE_PARAM_GRADS) != 0;
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        ws_bwd_kernel<T><<<filters, kWsThreads, 0, s>>>(w, static_cast<const T*>(dw_hat), dw, k, eps, accumulate);
        return static_cast<int>(cudaGetLastError());
    });
}
