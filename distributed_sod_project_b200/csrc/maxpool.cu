// maxpool.cu — MaxPool2d(kernel 3, stride 2, padding 1) of the ResNet stem (reference backbone/origin/resnet.py: `maxpool`,
// sliced into `div_4` by backbone/origin/from_origin.py:7-15), channels-last, forward and backward.
// On by default (resample.MAXPOOL_ENABLED; SOD_MAXPOOL=0 keeps torch's op).
//
// Why: on [16,64,160,160] bf16 torch's `max_pool_forward_nhwc` + `max_pool_backward_nhwc` move ≈75 MB of compulsory
// traffic each, and the backward drags an int64 index tensor (4× the size of the bf16 output).  Here: 16-byte channel packets, one byte of window position
// (kh*3+kw) per element instead of an int64 flat index, and a gather backward (every input pixel looks at the ≤4 windows
// that contain it, in ascending window order) — deterministic, fp32 accumulation like torch's.
// Tie-breaking and NaN behaviour follow torch's kernels: scan kh, kw ascending, replace on (v > max || isnan(v)),
// initial index = first in-bounds position.
#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kThreads) maxpool3x3s2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y,
                                                                    uint2* __restrict__ arg, int N, int H, int W, int HO,
                                                                    int WO, int C8) {
    const long long total = static_cast<long long>(N) * HO * WO * C8;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int ow = static_cast<int>(r % WO); r /= WO;
        const int oh = static_cast<int>(r % HO);
        const int n = static_cast<int>(r / HO);
        const int h0 = 2 * oh - 1, w0 = 2 * ow - 1;
        float m[8];
        unsigned a[8];
        bool first = true;
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
            const int ih = h0 + kh;
            if (ih < 0 || ih >= H) continue;
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
                const int iw = w0 + kw;
                if (iw < 0 || iw >= W) continue;
                const unsigned pos = kh * 3 + kw;
                float v[8];
                IO<T>::load8(x + ((static_cast<long long>(n) * H + ih) * W + iw) * C8 * 8 + static_cast<long long>(c) * 8, v);
                if (first) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) { m[k] = -INFINITY; a[k] = pos; }
                    first = false;
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (v[k] > m[k] || v[k] != v[k]) { m[k] = v[k]; a[k] = pos; }
                }
            }
        }
        IO<T>::store8(y + idx * 8, m);
        uint2 packed;
        packed.x = a[0] | (a[1] << 8) | (a[2] << 16) | (a[3] << 24);
        packed.y = a[4] | (a[5] << 8) | (a[6] << 16) | (a[7] << 24);
        arg[idx] = packed;
    }
}

template <typename T>
__global__ void __launch_bounds__(kThreads) maxpool3x3s2_bwd_kernel(const T* __restrict__ dy, const uint2* __restrict__ arg,
                                                                    T* __restrict__ dx, int N, int H, int W, int HO, int WO,
                                                                    int C8) {
    const long long total = static_cast<long long>(N) * H * W * C8;
    for (long long idx = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; idx < total;
         idx += static_cast<long long>(gridDim.x) * kThreads) {
        const int c = static_cast<int>(idx % C8);
        long long r = idx / C8;
        const int iw = static_cast<int>(r % W); r /= W;
        const int ih = static_cast<int>(r % H);
        const int n = static_cast<int>(r / H);
        // windows that contain row ih: even ih → (oh = ih/2, kh = 1); odd ih → (oh = (ih-1)/2, kh = 2), (oh = (ih+1)/2, kh = 0)
        const int noh = (ih & 1) ? 2 : 1, now = (iw & 1) ? 2 : 1;
        const int oh0 = (ih & 1) ? (ih - 1) / 2 : ih / 2, ow0 = (iw & 1) ? (iw - 1) / 2 : iw / 2;
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        for (int a = 0; a < noh; ++a) {
            const int oh = oh0 + a;
            if (oh >= HO) continue;
            const unsigned kh = (ih & 1) ? (a == 0 ? 2u : 0u) : 1u;
            for (int b = 0; b < now; ++b) {
                const int ow = ow0 + b;
                if (ow >= WO) continue;
                const unsigned kw = (iw & 1) ? (b == 0 ? 2u : 0u) : 1u;
                const unsigned pos = kh * 3 + kw;
                const long long o = ((static_cast<long long>(n) * HO + oh) * WO + ow) * C8 + c;
                const uint2 p = arg[o];
                float g[8];
                IO<T>::load8(dy + o * 8, g);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    const unsigned byte = ((k < 4 ? p.x : p.y) >> (8 * (k & 3))) & 0xFFu;
                    if (byte == pos) acc[k] += g[k];
                }
            }
        }
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

}  // namespace
}  // namespace sod

extern "C" int sod_maxpool3x3s2_fwd(const void* x, void* y, void* argmax, int n, int h, int w, int c, int dtype, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(x && y && argmax, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(x) && aligned16(y) && aligned16(argmax), SOD_EALIGN);
    if (n <= 0 || h <= 0 || w <= 0 || c <= 0) return SOD_EINVAL;
    if (c % 8) return SOD_EUNSUPPORTED;
    const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * ho * wo * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        maxpool3x3s2_fwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(x), static_cast<T*>(y),
                                                                           static_cast<uint2*>(argmax), n, h, w, ho, wo, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}

extern "C" int sod_maxpool3x3s2_bwd(const void* dy, const void* argmax, void* dx, int n, int h, int w, int c, int dtype,
                                    void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(dy && dx && argmax, SOD_EINVAL);
    SOD_CHECK_ARG(aligned16(dy) && aligned16(dx) && aligned16(argmax), SOD_EALIGN);
    if (n <= 0 || h <= 0 || w <= 0 || c <= 0) return SOD_EINVAL;
    if (c % 8) return SOD_EUNSUPPORTED;
    const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const long long packets = static_cast<long long>(n) * h * w * (c / 8);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        maxpool3x3s2_bwd_kernel<T><<<grid_for(packets), kThreads, 0, s>>>(static_cast<const T*>(dy), static_cast<const uint2*>(argmax),
                                                                           static_cast<T*>(dx), n, h, w, ho, wo, c / 8);
        return static_cast<int>(cudaGetLastError());
    });
}
