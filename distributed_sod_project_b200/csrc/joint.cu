// joint.cu — the pieces of the reference's other joint transforms (utils/joint_transforms.py:51-137) that the resize
// and augmentation kernels do not already cover, bit for bit as Pillow computes them, over ragged 8-bit batches
// ("L" and "RGB" stored HWC):
//
//   - sod_resize_nearest_u8: `Image.resize(size, NEAREST)` (RandomScaleCrop's and ScaleCenterCrop's mask resize).
//     Pillow (libImaging/Geometry.c, ImagingScaleAffine) tabulates each axis once: a = in / out, xo = a·0.5, then per
//     output pixel COORD(xo) = xo < 0 ? −1 : (int)xo and xo += a.  The repeated addition accumulates rounding, so the
//     table is built the same way, sequentially by one thread per image and axis, in double with every operation an
//     explicitly rounded intrinsic, as resize.cu builds its tables.  Taps outside the source give 0.
//     A same-size image gets a = 1 and exact half-integers, so the table is the identity: Pillow's copy.
//   - sod_window_u8: an h_o × w_o window of each image at a per-image offset (dy, dx), zeros outside the source: the
//     crops of RandomScaleCrop / ScaleCenterCrop (`Image.crop`) and PaddingSquare's centred zero padding (dy, dx < 0).
//   - sod_gaussian_blur_u8: `img.filter(GaussianBlur(r))` (RandomGaussianBlur), Pillow's extended box blur
//     (libImaging/BoxBlur.c): three horizontal passes, then three vertical ones, each rounded to 8 bits,
//       out = (ww·Σ_{|k|≤R} x[i+k] + fw·(x[i−R−1] + x[i+R+1]) + 2²³) >> 24 with indices clamped into the image.
//     R, ww and fw come from the host (sod_blur_param); the passes are exact uint32 arithmetic (at most 255·2²⁴ + 2²³),
//     so Pillow's running sum and this direct sum give the same bytes.
//
// Every launch is images × `per` CTAs of 256 threads, grid-stride over the image's output bytes (or, for the tables,
// one thread per image and axis).
#include <cmath>
#include <vector>

#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 256;
constexpr int kCtasPerSm = 8;
constexpr int kMaxPer = 128;
constexpr int kMaxBlurRadius = 1024;

long long align16(long long v) { return (v + 15) & ~15ll; }

// CTAs per image: about 8 waves in all, at most what the largest image needs (given on the host) and kMaxPer
int ctas_per_image(int n, long long max_bytes) {
    long long per = (static_cast<long long>(kCtasPerSm) * dev_info().sm_count + n - 1) / n;
    const long long need = (max_bytes + kThreads - 1) / kThreads;
    if (per > need) per = need;
    if (per > kMaxPer) per = kMaxPer;
    return per < 1 ? 1 : static_cast<int>(per);
}

// ---- NEAREST resize ------------------------------------------------------------------------------------------------
struct NearestParams {
    const unsigned char* src;
    const long long* src_off;
    const int* src_hw;
    unsigned char* dst;
    const long long* dst_off;
    const int* dst_hw;
    int* tab;                   // per image [ow] source columns then [oh] source rows, −1 = outside
    const long long* tab_off;   // [n] int offsets into tab, in the workspace
    int n, ch;
};

__global__ void nearest_table_kernel(const __grid_constant__ NearestParams p) {
    const int b = blockIdx.x, axis = threadIdx.x;      // 0: columns, 1: rows
    if (axis > 1) return;
    const int in = p.src_hw[2 * b + 1 - axis], out = p.dst_hw[2 * b + 1 - axis];
    int* t = p.tab + p.tab_off[b] + (axis ? p.dst_hw[2 * b + 1] : 0);
    const double a = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
    double xo = __dmul_rn(a, 0.5);
    for (int x = 0; x < out; ++x) {
        const int xi = xo < 0.0 ? -1 : static_cast<int>(xo);
        t[x] = xi >= 0 && xi < in ? xi : -1;
        xo = __dadd_rn(xo, a);
    }
}

template <int CH>
__device__ void nearest_copy(const NearestParams& p, int b) {
    const int iw = p.src_hw[2 * b + 1], oh = p.dst_hw[2 * b], ow = p.dst_hw[2 * b + 1];
    const int* tx = p.tab + p.tab_off[b];
    const int* ty = tx + ow;
    const unsigned char* src = p.src + p.src_off[b];
    unsigned char* dst = p.dst + p.dst_off[b];
    const long long total = static_cast<long long>(oh) * ow * CH;
    for (long long e = static_cast<long long>(blockIdx.y) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.y) * blockDim.x) {
        const long long px = CH == 1 ? e : e / CH;
        const int c = static_cast<int>(e - px * CH);
        const int y = static_cast<int>(px / ow), x = static_cast<int>(px - static_cast<long long>(y) * ow);
        const int yi = ty[y], xi = tx[x];
        dst[e] = yi >= 0 && xi >= 0 ? src[(static_cast<long long>(yi) * iw + xi) * CH + c] : 0;
    }
}

__global__ void __launch_bounds__(kThreads) nearest_copy_kernel(const __grid_constant__ NearestParams p) {
    if (p.ch == 1) nearest_copy<1>(p, blockIdx.x);
    else nearest_copy<3>(p, blockIdx.x);
}

// ---- window --------------------------------------------------------------------------------------------------------
struct WindowParams {
    const unsigned char* src;
    const long long* src_off;
    const int* src_hw;
    unsigned char* dst;
    const long long* dst_off;
    const int* dst_hw;
    const int* offset;          // [n][2] (dy, dx), in the workspace
    int n, ch;
};

template <int CH>
__device__ void window_copy(const WindowParams& p, int b) {
    const int ih = p.src_hw[2 * b], iw = p.src_hw[2 * b + 1], ow = p.dst_hw[2 * b + 1];
    const int dy = p.offset[2 * b], dx = p.offset[2 * b + 1];
    const unsigned char* src = p.src + p.src_off[b];
    unsigned char* dst = p.dst + p.dst_off[b];
    const long long total = static_cast<long long>(p.dst_hw[2 * b]) * ow * CH;
    for (long long e = static_cast<long long>(blockIdx.y) * blockDim.x + threadIdx.x; e < total;
         e += static_cast<long long>(gridDim.y) * blockDim.x) {
        const long long px = CH == 1 ? e : e / CH;
        const int c = static_cast<int>(e - px * CH);
        const int y = static_cast<int>(px / ow), x = static_cast<int>(px - static_cast<long long>(y) * ow);
        const long long ys = static_cast<long long>(y) + dy, xs = static_cast<long long>(x) + dx;
        dst[e] = ys >= 0 && ys < ih && xs >= 0 && xs < iw ? src[(ys * iw + xs) * CH + c] : 0;
    }
}

__global__ void __launch_bounds__(kThreads) window_kernel(const __grid_constant__ WindowParams p) {
    if (p.ch == 1) window_copy<1>(p, blockIdx.x);
    else window_copy<3>(p, blockIdx.x);
}

// ---- box-blur pass -------------------------------------------------------------------------------------------------
struct BlurPass {
    const unsigned char* src;   // [n][h][w][ch]
    unsigned char* dst;
    const sod_blur_param* prm;  // [n], in the workspace
    int h, w, ch, vertical;
};

template <int CH>
__device__ void blur_pass(const BlurPass& p, int b) {
    const sod_blur_param P = p.prm[b];
    const long long plane = static_cast<long long>(p.h) * p.w * CH;
    const unsigned char* src = p.src + plane * b;
    unsigned char* dst = p.dst + plane * b;
    const int R = P.radius, len = p.vertical ? p.h : p.w;
    const long long stride = p.vertical ? static_cast<long long>(p.w) * CH : CH;
    for (long long e = static_cast<long long>(blockIdx.y) * blockDim.x + threadIdx.x; e < plane;
         e += static_cast<long long>(gridDim.y) * blockDim.x) {
        const long long px = CH == 1 ? e : e / CH;
        const int y = static_cast<int>(px / p.w), x = static_cast<int>(px - static_cast<long long>(y) * p.w);
        const int i = p.vertical ? y : x;
        const unsigned char* line = src + (e - static_cast<long long>(i) * stride);     // element 0 of this line
        unsigned int acc = 0;
        for (int k = -R; k <= R; ++k) acc += line[static_cast<long long>(min(max(i + k, 0), len - 1)) * stride];
        const unsigned int far = static_cast<unsigned int>(line[static_cast<long long>(max(i - R - 1, 0)) * stride]) +
                                 line[static_cast<long long>(min(i + R + 1, len - 1)) * stride];
        dst[e] = static_cast<unsigned char>((acc * P.ww + far * P.fw + (1u << 23)) >> 24);
    }
}

__global__ void __launch_bounds__(kThreads) blur_pass_kernel(const __grid_constant__ BlurPass p) {
    if (p.ch == 1) blur_pass<1>(p, blockIdx.x);
    else blur_pass<3>(p, blockIdx.x);
}

bool valid_blur_param(const sod_blur_param& q) {
    if (q.radius < 0 || q.radius > kMaxBlurRadius) return false;
    const unsigned long long sum = static_cast<unsigned long long>(2 * q.radius + 1) * q.ww + 2ull * q.fw;
    return q.ww > 0 && sum <= (1ull << 24);
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_resize_nearest_u8_workspace_bytes(int n, const int32_t* src_hw, const int32_t* dst_hw, int channels) {
    using namespace sod;
    if (n <= 0 || !src_hw || !dst_hw || (channels != 1 && channels != 3)) return 0;
    long long ints = 0;
    for (int i = 0; i < n; ++i) {
        if (src_hw[2 * i] <= 0 || src_hw[2 * i + 1] <= 0 || dst_hw[2 * i] <= 0 || dst_hw[2 * i + 1] <= 0) return 0;
        ints += static_cast<long long>(dst_hw[2 * i]) + dst_hw[2 * i + 1];
    }
    return static_cast<size_t>(align16(8ll * n) + 4 * ints);
}

extern "C" int sod_resize_nearest_u8(const void* src, const int64_t* src_off, const int32_t* src_hw, void* dst,
                                     const int64_t* dst_off, const int32_t* dst_hw, const int32_t* src_hw_host,
                                     const int32_t* dst_hw_host, int n, int channels, void* workspace,
                                     size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(src && src_off && src_hw && dst && dst_off && dst_hw && src_hw_host && dst_hw_host && workspace, SOD_EINVAL);
    SOD_CHECK_ARG(n > 0 && (channels == 1 || channels == 3), SOD_EINVAL);
    const size_t need = sod_resize_nearest_u8_workspace_bytes(n, src_hw_host, dst_hw_host, channels);
    SOD_CHECK_ARG(need > 0 && workspace_bytes >= need, SOD_EINVAL);
    // table offsets on the host, from the host copy of the sizes; copied to the head of the workspace
    std::vector<long long> off(n);
    long long ints = 0, max_bytes = 0;
    for (int i = 0; i < n; ++i) {
        off[i] = ints;
        ints += static_cast<long long>(dst_hw_host[2 * i]) + dst_hw_host[2 * i + 1];
        const long long bytes = static_cast<long long>(dst_hw_host[2 * i]) * dst_hw_host[2 * i + 1] * channels;
        if (bytes > max_bytes) max_bytes = bytes;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    NearestParams p;
    p.src = static_cast<const unsigned char*>(src); p.src_off = reinterpret_cast<const long long*>(src_off); p.src_hw = src_hw;
    p.dst = static_cast<unsigned char*>(dst); p.dst_off = reinterpret_cast<const long long*>(dst_off); p.dst_hw = dst_hw;
    p.tab_off = static_cast<const long long*>(workspace);
    p.tab = reinterpret_cast<int*>(static_cast<unsigned char*>(workspace) + align16(8ll * n));
    p.n = n; p.ch = channels;
    // pageable source: the offsets are staged before cudaMemcpyAsync returns, so `off` may go out of scope
    const cudaError_t e = cudaMemcpyAsync(const_cast<long long*>(p.tab_off), off.data(), 8ull * n, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return static_cast<int>(e);
    nearest_table_kernel<<<n, 32, 0, s>>>(p);
    const dim3 grid(static_cast<unsigned>(n), static_cast<unsigned>(ctas_per_image(n, max_bytes)));
    nearest_copy_kernel<<<grid, kThreads, 0, s>>>(p);
    return static_cast<int>(cudaGetLastError());
}

extern "C" size_t sod_window_u8_workspace_bytes(int n) {
    if (n <= 0) return 0;
    return static_cast<size_t>(sod::align16(8ll * n));
}

extern "C" int sod_window_u8(const void* src, const int64_t* src_off, const int32_t* src_hw, void* dst, const int64_t* dst_off,
                             const int32_t* dst_hw, const int32_t* dst_hw_host, const int32_t* offset, int n, int channels,
                             void* workspace, size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(src && src_off && src_hw && dst && dst_off && dst_hw && dst_hw_host && offset && workspace, SOD_EINVAL);
    SOD_CHECK_ARG(n > 0 && (channels == 1 || channels == 3), SOD_EINVAL);
    SOD_CHECK_ARG(workspace_bytes >= sod_window_u8_workspace_bytes(n), SOD_EINVAL);
    long long max_bytes = 0;
    for (int i = 0; i < n; ++i) {
        SOD_CHECK_ARG(dst_hw_host[2 * i] > 0 && dst_hw_host[2 * i + 1] > 0, SOD_EINVAL);
        const long long bytes = static_cast<long long>(dst_hw_host[2 * i]) * dst_hw_host[2 * i + 1] * channels;
        if (bytes > max_bytes) max_bytes = bytes;
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    WindowParams p;
    p.src = static_cast<const unsigned char*>(src); p.src_off = reinterpret_cast<const long long*>(src_off); p.src_hw = src_hw;
    p.dst = static_cast<unsigned char*>(dst); p.dst_off = reinterpret_cast<const long long*>(dst_off); p.dst_hw = dst_hw;
    p.offset = static_cast<const int*>(workspace);
    p.n = n; p.ch = channels;
    // the offsets are copied out of the caller's (pageable) memory before this call returns
    cudaError_t e = cudaMemcpyAsync(workspace, offset, 8ull * n, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return static_cast<int>(e);
    const dim3 grid(static_cast<unsigned>(n), static_cast<unsigned>(ctas_per_image(n, max_bytes)));
    window_kernel<<<grid, kThreads, 0, s>>>(p);
    return static_cast<int>(cudaGetLastError());
}

extern "C" size_t sod_gaussian_blur_u8_workspace_bytes(int n, int h, int w, int channels) {
    if (n <= 0 || h <= 0 || w <= 0 || (channels != 1 && channels != 3)) return 0;
    return static_cast<size_t>(sod::align16(static_cast<long long>(n) * sizeof(sod_blur_param)) +
                               static_cast<long long>(n) * h * w * channels);
}

extern "C" int sod_gaussian_blur_u8(const void* src, void* dst, int n, int h, int w, int channels, const sod_blur_param* params,
                                    void* workspace, size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(src && dst && params && workspace, SOD_EINVAL);
    const size_t need = sod_gaussian_blur_u8_workspace_bytes(n, h, w, channels);
    SOD_CHECK_ARG(need > 0 && workspace_bytes >= need, SOD_EINVAL);
    for (int i = 0; i < n; ++i) SOD_CHECK_ARG(valid_blur_param(params[i]), SOD_EINVAL);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    const sod_blur_param* prm = reinterpret_cast<const sod_blur_param*>(ws);
    unsigned char* tmp = ws + align16(static_cast<long long>(n) * sizeof(sod_blur_param));
    // the parameters are copied out of the caller's (pageable) memory before this call returns
    cudaError_t e = cudaMemcpyAsync(ws, params, sizeof(sod_blur_param) * n, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) return static_cast<int>(e);
    const dim3 grid(static_cast<unsigned>(n),
                    static_cast<unsigned>(ctas_per_image(n, static_cast<long long>(h) * w * channels)));
    // src → tmp → dst → tmp (horizontal), tmp → dst → tmp → dst (vertical): src is only read
    const unsigned char* in[6] = {static_cast<const unsigned char*>(src), tmp, static_cast<unsigned char*>(dst), tmp,
                                  static_cast<unsigned char*>(dst), tmp};
    unsigned char* out[6] = {tmp, static_cast<unsigned char*>(dst), tmp, static_cast<unsigned char*>(dst), tmp,
                             static_cast<unsigned char*>(dst)};
    for (int k = 0; k < 6; ++k) {
        BlurPass p;
        p.src = in[k]; p.dst = out[k]; p.prm = prm; p.h = h; p.w = w; p.ch = channels; p.vertical = k >= 3;
        blur_pass_kernel<<<grid, kThreads, 0, s>>>(p);
    }
    return static_cast<int>(cudaGetLastError());
}
