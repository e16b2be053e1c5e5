// resample.cu — the two resampling ops of the TestModel decoder, channels-last, forward and backward:
//   * bilinear ×2 up-sampling, align_corners=False (reference utils/tensor_ops.py:12-25 `cus_sample` /
//     `upsample_add`, used by network/TestModel.py and module/MyLightModule.py:42-52), optionally fused with the
//     addition of `upsample_add`;
//   * 2×2 / stride-2 average pooling (reference module/MyLightModule.py:14 `h2l_pool`).
// They sit on either side of the SyncBN kernels (SURVEY §8f.1).  torch's bf16 kernels for them cost ≈3.9 ms per
// iteration at bs16·320² (bilinear backward scatters with atomics: non-deterministic and slow; avg-pool backward
// runs far below bandwidth).  Here every op is a pure gather over [N,H,W,C] with 16-byte channel packets:
// deterministic, one read of each needed packet (neighbours hit L1/L2), one write.
#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 256;

// ×2 bilinear, align_corners=False: out[2k] = .25 in[k-1] + .75 in[k] (k=0: in[0]); out[2k+1] = .75 in[k] + .25 in[k+1]
// (k=H-1: in[H-1]).  Returns the two source indices and the weight of the second one.  At o = 0 the first tap has
// weight 0: the forward zeroes its operand, since 0·inf would turn an infinite in[0] into NaN.
__device__ __forceinline__ void src_of(int o, int n_in, int& i0, int& i1, float& w1) {
    const int k = o >> 1;
    if (o & 1) {
        i0 = k;
        i1 = (k + 1 < n_in) ? k + 1 : k;
        w1 = 0.25f;
    } else {
        i0 = (k > 0) ? k - 1 : 0;
        i1 = k;
        w1 = (k > 0) ? 0.75f : 1.0f;   // k == 0: both indices are 0, any split sums to in[0]
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) upsample2x_fwd_kernel(const T* __restrict__ x, const T* __restrict__ add,
                                                                  T* __restrict__ y, int N, int H, int W, int C8) {
    const long long total = static_cast<long long>(N) * (2 * H) * (2 * W) * C8;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int ow = static_cast<int>(r % (2 * W)); r /= (2 * W);
        const int oh = static_cast<int>(r % (2 * H));
        const int n = static_cast<int>(r / (2 * H));
        int h0, h1, w0, w1i;
        float fh, fw;
        src_of(oh, H, h0, h1, fh);
        src_of(ow, W, w0, w1i, fw);
        const T* base = x + (static_cast<long long>(n) * H * W) * C8 * 8 + static_cast<long long>(c) * 8;
        float a[8], b[8], cc[8], d[8], o[8];
        IO<T>::load8(base + (static_cast<long long>(h0) * W + w0) * C8 * 8, a);
        IO<T>::load8(base + (static_cast<long long>(h0) * W + w1i) * C8 * 8, b);
        IO<T>::load8(base + (static_cast<long long>(h1) * W + w0) * C8 * 8, cc);
        IO<T>::load8(base + (static_cast<long long>(h1) * W + w1i) * C8 * 8, d);
        if (oh == 0) {                  // row tap h0 has weight 0 (see src_of)
#pragma unroll
            for (int k = 0; k < 8; ++k) { a[k] = 0.f; b[k] = 0.f; }
        }
        if (ow == 0) {                  // column tap w0 has weight 0
#pragma unroll
            for (int k = 0; k < 8; ++k) { a[k] = 0.f; cc[k] = 0.f; }
        }
        const float w00 = (1.f - fh) * (1.f - fw), w01 = (1.f - fh) * fw, w10 = fh * (1.f - fw), w11 = fh * fw;
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = w00 * a[k] + w01 * b[k] + w10 * cc[k] + w11 * d[k];
        if (add != nullptr) {
            float t[8];
            IO<T>::load8(add + idx * 8, t);
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] += t[k];
        }
        IO<T>::store8(y + idx * 8, o);
    }
}

// gather form of the backward: input pixel k collects from outputs 2k-1 (.25), 2k (.75 | 1), 2k+1 (.75 | 1), 2k+2 (.25)
__device__ __forceinline__ int taps_of(int k, int n_in, int (&o)[4], float (&w)[4]) {
    int m = 0;
    if (k > 0) { o[m] = 2 * k - 1; w[m] = 0.25f; ++m; }
    o[m] = 2 * k; w[m] = (k > 0) ? 0.75f : 1.0f; ++m;
    o[m] = 2 * k + 1; w[m] = (k + 1 < n_in) ? 0.75f : 1.0f; ++m;
    if (k + 1 < n_in) { o[m] = 2 * k + 2; w[m] = 0.25f; ++m; }
    return m;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) upsample2x_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int N, int H,
                                                                  int W, int C8) {
    const long long total = static_cast<long long>(N) * H * W * C8;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int iw = static_cast<int>(r % W); r /= W;
        const int ih = static_cast<int>(r % H);
        const int n = static_cast<int>(r / H);
        int oh[4], ow[4];
        float wh[4], ww[4];
        const int nh = taps_of(ih, H, oh, wh), nw = taps_of(iw, W, ow, ww);
        const T* base = dy + (static_cast<long long>(n) * 2 * H * 2 * W) * C8 * 8 + static_cast<long long>(c) * 8;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        for (int a = 0; a < nh; ++a) {
#pragma unroll 4
            for (int b = 0; b < nw; ++b) {
                float t[8];
                IO<T>::load8(base + (static_cast<long long>(oh[a]) * 2 * W + ow[b]) * C8 * 8, t);
                const float wgt = wh[a] * ww[b];
#pragma unroll
                for (int k = 0; k < 8; ++k) acc[k] = fmaf(wgt, t[k], acc[k]);
            }
        }
        IO<T>::store8(dx + idx * 8, acc);
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) avgpool2x2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N, int HO,
                                                                  int WO, int C8) {
    const long long total = static_cast<long long>(N) * HO * WO * C8;
    const int W = 2 * WO;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int ow = static_cast<int>(r % WO); r /= WO;
        const int oh = static_cast<int>(r % HO);
        const int n = static_cast<int>(r / HO);
        const T* p = x + ((static_cast<long long>(n) * 2 * HO + 2 * oh) * W + 2 * ow) * C8 * 8 + static_cast<long long>(c) * 8;
        float a[8], b[8], cc[8], d[8], o[8];
        IO<T>::load8(p, a);
        IO<T>::load8(p + C8 * 8, b);
        IO<T>::load8(p + static_cast<long long>(W) * C8 * 8, cc);
        IO<T>::load8(p + static_cast<long long>(W + 1) * C8 * 8, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = 0.25f * (a[k] + b[k] + cc[k] + d[k]);
        IO<T>::store8(y + idx * 8, o);
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) avgpool2x2_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int N, int HO,
                                                                  int WO, int C8) {
    const int H = 2 * HO, W = 2 * WO;
    const long long total = static_cast<long long>(N) * H * W * C8;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int iw = static_cast<int>(r % W); r /= W;
        const int ih = static_cast<int>(r % H);
        const int n = static_cast<int>(r / H);
        float t[8];
        IO<T>::load8(dy + ((static_cast<long long>(n) * HO + (ih >> 1)) * WO + (iw >> 1)) * C8 * 8 + static_cast<long long>(c) * 8, t);
#pragma unroll
        for (int k = 0; k < 8; ++k) t[k] *= 0.25f;
        IO<T>::store8(dx + idx * 8, t);
    }
}

static unsigned grid_for(long long packets) {
    long long b = (packets + kThreads - 1) / kThreads;
    const long long cap = 16ll * dev_info().sm_count;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return static_cast<unsigned>(b);
}

static int check_dims(int n, int h, int w, int c) {
    if (n <= 0 || h <= 0 || w <= 0 || c <= 0) return SOD_EINVAL;
    if (c % 8) return SOD_EUNSUPPORTED;
    return SOD_OK;
}

}  // namespace
}  // namespace sod

extern "C" int sod_upsample2x_bilinear_fwd(const void* x, const void* add, void* y, int n, int h, int w, int c, int dtype,
                                           void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && y, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(x) && aligned16(y) && (!add || aligned16(add)), SOD_EALIGN);
    int rc = check_dims(n, h, w, c);
    if (rc != SOD_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * 2 * h * 2 * w * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        upsample2x_fwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(x), static_cast<const T*>(add),
                                                                       static_cast<T*>(y), n, h, w, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_upsample2x_bilinear_bwd(const void* dy, void* dx, int n, int h, int w, int c, int dtype, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && dx, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(dy) && aligned16(dx), SOD_EALIGN);
    int rc = check_dims(n, h, w, c);
    if (rc != SOD_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * h * w * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        upsample2x_bwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(dy), static_cast<T*>(dx), n, h, w, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_avgpool2x2_fwd(const void* x, void* y, int n, int h_out, int w_out, int c, int dtype, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && y, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(x) && aligned16(y), SOD_EALIGN);
    int rc = check_dims(n, h_out, w_out, c);
    if (rc != SOD_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * h_out * w_out * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        avgpool2x2_fwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(x), static_cast<T*>(y), n, h_out, w_out, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_avgpool2x2_bwd(const void* dy, void* dx, int n, int h_out, int w_out, int c, int dtype, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && dx, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(dy) && aligned16(dx), SOD_EALIGN);
    int rc = check_dims(n, h_out, w_out, c);
    if (rc != SOD_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * 2 * h_out * 2 * w_out * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        avgpool2x2_bwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(dy), static_cast<T*>(dx), n, h_out, w_out, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}

// ------------------------------------------------------------------------------------------------
// column sum of a channels-last matrix [rows, C] — the bias gradient of a convolution that does NOT feed a
// BatchNorm (the five `trans*` 1x1 convolutions, network/TestModel.py:32-36; their bias gradient is Σ_rows dy).
// Deterministic: per-CTA partials in a workspace, the LAST CTA to finish (ticket counter) adds them in CTA order.
// ------------------------------------------------------------------------------------------------
namespace sod {
namespace {

template <typename T>
__global__ void __launch_bounds__(256) colsum_kernel(const T* __restrict__ x, T* __restrict__ out, long long rows, int L,
                                                      float* __restrict__ partial, unsigned* __restrict__ ticket) {
    __shared__ float s_acc[256 * 8];
    __shared__ bool s_last;
    const int tid = threadIdx.x;
    const int l = tid % L, r0 = tid / L, R = 256 / L;       // L ≤ 256 lanes (8 channels each), R rows per pass
    const int C = L * 8;
    float a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = 0.f;
    if (r0 < R) {
        // four independent 16-byte loads in flight per thread (the loop is latency bound with one)
        const long long step = static_cast<long long>(gridDim.x) * R;
        long long r = static_cast<long long>(blockIdx.x) * R + r0;
        for (; r + 3 * step < rows; r += 4 * step) {
            typename IO<T>::Raw q0 = IO<T>::load_raw(x + r * C + l * 8);
            typename IO<T>::Raw q1 = IO<T>::load_raw(x + (r + step) * C + l * 8);
            typename IO<T>::Raw q2 = IO<T>::load_raw(x + (r + 2 * step) * C + l * 8);
            typename IO<T>::Raw q3 = IO<T>::load_raw(x + (r + 3 * step) * C + l * 8);
            float v0[8], v1[8], v2[8], v3[8];
            IO<T>::unpack(q0, v0); IO<T>::unpack(q1, v1); IO<T>::unpack(q2, v2); IO<T>::unpack(q3, v3);
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += (v0[k] + v1[k]) + (v2[k] + v3[k]);
        }
        for (; r < rows; r += step) {
            float v[8];
            IO<T>::load8(x + r * C + l * 8, v);
#pragma unroll
            for (int k = 0; k < 8; ++k) a[k] += v[k];
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) s_acc[tid * 8 + k] = a[k];
    __syncthreads();
    float* mine = partial + static_cast<size_t>(blockIdx.x) * C;
    for (int ch = tid; ch < C; ch += 256) {
        const int ll = ch >> 3, k = ch & 7;
        float t = 0.f;
        for (int rr = 0; rr < R; ++rr) t += s_acc[(rr * L + ll) * 8 + k];
        mine[ch] = t;
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int ch = tid; ch < C; ch += 256) {
        float t = 0.f;
        for (unsigned b = 0; b < gridDim.x; ++b) t += __ldcg(partial + static_cast<size_t>(b) * C + ch);
        IO<T>::store1(out + ch, t);
    }
    if (tid == 0) *ticket = 0;                               // ready for the next launch on this stream
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_colsum_workspace_bytes(void) { return static_cast<size_t>(296) * 2048 * sizeof(float) + 256; }

extern "C" int sod_colsum(const void* x, void* out, int64_t rows, int c, int dtype, void* workspace, size_t workspace_bytes,
                          void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && out && workspace && rows > 0 && c > 0, SOD_EINVAL);
    SOD_CHECK_ARG((c % 8) == 0 && c <= 2048, SOD_EUNSUPPORTED);
    const int L = c / 8;
    SOD_CHECK_ARG((L & (L - 1)) == 0, SOD_EUNSUPPORTED);
    SOD_CHECK_ARG(aligned16(x) && aligned16(workspace), SOD_EALIGN);
    SOD_CHECK_ARG(workspace_bytes >= sod_colsum_workspace_bytes(), SOD_EWORKSPACE);
    const int R = 256 / L;
    long long grid = (rows + static_cast<long long>(R) * 8 - 1) / (static_cast<long long>(R) * 8);   // ≥ 8 passes per CTA
    const long long cap = 2ll * dev_info().sm_count;
    if (grid > cap) grid = cap;
    if (grid > 296) grid = 296;
    if (grid < 1) grid = 1;
    unsigned* ticket = reinterpret_cast<unsigned*>(workspace);               // first 256 bytes: ticket (zeroed once by the host)
    float* partial = reinterpret_cast<float*>(static_cast<char*>(workspace) + 256);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        colsum_kernel<T><<<static_cast<unsigned>(grid), 256, 0, s>>>(static_cast<const T*>(x), static_cast<T*>(out), rows, L, partial, ticket);
        return static_cast<int>(cudaGetLastError());
    });
}
