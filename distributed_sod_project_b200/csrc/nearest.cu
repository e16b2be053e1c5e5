// nearest.cu — nearest ×2 up-sampling of the LightAIM neck (reference module/MyLightModule.py:64,146,
// `nn.Upsample(scale_factor=2, mode="nearest")`), channels-last, forward and backward, beside the resampling kernels of
// resample.cu and with the same 16-byte channel packets, launch geometry and argument checks.
#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 256;

// nearest ×2 (nn.Upsample(scale_factor=2, mode="nearest"), LightAIM's `l2h_up` / `upsample`,
// module/MyLightModule.py:64,146): out[2i + a][2j + b] = in[i][j].  One thread per INPUT packet: the forward copies it to
// its four outputs as raw 16-byte words (bit-exact in every dtype); the backward gathers those four dy packets and sums
// them in the fixed order (0,0), (0,1), (1,0), (1,1) from 0 in fp32, rounding once.  No atomics: reruns are bit-identical.
template <typename T>
__global__ void __launch_bounds__(kThreads) upsample2x_nearest_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int N,
                                                                          int H, int W, int C8) {
    const long long total = static_cast<long long>(N) * H * W * C8;
    const long long row = static_cast<long long>(2 * W) * C8 * 8;            // one output row, in elements
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int iw = static_cast<int>(r % W); r /= W;
        const int ih = static_cast<int>(r % H);
        const int n = static_cast<int>(r / H);
        using Raw = typename IO<T>::Raw;
        const Raw v = IO<T>::load_raw(x + idx * 8);
        T* p = y + ((static_cast<long long>(n) * 2 * H + 2 * ih) * (2 * W) + 2 * iw) * C8 * 8 + static_cast<long long>(c) * 8;
        *reinterpret_cast<Raw*>(p) = v;
        *reinterpret_cast<Raw*>(p + C8 * 8) = v;
        *reinterpret_cast<Raw*>(p + row) = v;
        *reinterpret_cast<Raw*>(p + row + C8 * 8) = v;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) upsample2x_nearest_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, int N,
                                                                          int H, int W, int C8) {
    const long long total = static_cast<long long>(N) * H * W * C8;
    const long long row = static_cast<long long>(2 * W) * C8 * 8;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int iw = static_cast<int>(r % W); r /= W;
        const int ih = static_cast<int>(r % H);
        const int n = static_cast<int>(r / H);
        const T* p = dy + ((static_cast<long long>(n) * 2 * H + 2 * ih) * (2 * W) + 2 * iw) * C8 * 8 + static_cast<long long>(c) * 8;
        float a[8], b[8], cc[8], d[8], acc[8];
        IO<T>::load8(p, a);
        IO<T>::load8(p + C8 * 8, b);
        IO<T>::load8(p + row, cc);
        IO<T>::load8(p + row + C8 * 8, d);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = (((0.f + a[k]) + b[k]) + cc[k]) + d[k];
        IO<T>::store8(dx + idx * 8, acc);
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

extern "C" int sod_upsample2x_nearest_fwd(const void* x, void* y, int n, int h, int w, int c, int dtype, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && y, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(x) && aligned16(y), SOD_EALIGN);
    int rc = check_dims(n, h, w, c);
    if (rc != SOD_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * h * w * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        upsample2x_nearest_fwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(x), static_cast<T*>(y), n, h, w, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_upsample2x_nearest_bwd(const void* dy, void* dx, int n, int h, int w, int c, int dtype, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && dx, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(dy) && aligned16(dx), SOD_EALIGN);
    int rc = check_dims(n, h, w, c);
    if (rc != SOD_OK) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * h * w * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        upsample2x_nearest_bwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(dy), static_cast<T*>(dx), n, h, w, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}
