// resize.cu — Pillow's 8-bit resampler, `Image.resize(size, BILINEAR | BICUBIC)` with box = the whole image and
// reducing_gap=None, over a ragged batch ("L" and "RGB" stored HWC).
//
// The reference resizes every 8-bit prediction to its ground truth's size with `ToPILImage()(out).resize(gt.size)`
// (train.py:392-395, BICUBIC) and feeds test images through torchvision `Resize((S, S))` (utils/dataset.py:97-104,
// Pillow BILINEAR).  Pillow's algorithm (libImaging/Resample.c):
//   - per axis, scale = in / out, filterscale = max(scale, 1), support = filter support · filterscale; output pixel x
//     reads taps [xmin, xmin + cnt) with center = (x + 0.5)·scale, xmin = (int)(center − support + 0.5) clamped at 0,
//     xmax = (int)(center + support + 0.5) clamped at in; weights filter((tap − center + 0.5) · (1 / filterscale)),
//     summed in tap order, divided by that sum, then rounded to 22-bit fixed point half away from zero;
//   - two passes, horizontal first; the horizontal pass only produces the source rows the vertical pass reads; a pass
//     runs only if its axis changes size, and an unchanged image is copied;
//   - accumulation in int32 from 2^21, >> 22, clipped to [0, 255].
// The coefficient tables are the only floating-point part.  nvcc would contract `a*b + c` into an FMA, which Pillow's
// x86-64 build does not do, so every double operation below is an explicitly rounded intrinsic.  After that the passes
// add exact integers, so any thread mapping writes the same bytes.
//
// Three launches per call, each over images × rows: coefficient tables, horizontal pass (or the copy), vertical pass.
#include <cmath>

#include "common.cuh"

namespace sod {
namespace {

constexpr int kPrecisionBits = 22;
constexpr int kThreads = 256;

__host__ __device__ inline double filter_support(int filter) { return filter == SOD_RESIZE_BICUBIC ? 2.0 : 1.0; }

// ksize of precompute_coeffs: the row length of one output pixel's weight table.  One division, one multiplication and
// a ceil: rounded identically on the host (workspace query) and on the device.
__host__ __device__ inline int axis_ksize(int in, int out, int filter) {
    double fs = static_cast<double>(in) / out;
    if (fs < 1.0) fs = 1.0;
    return static_cast<int>(ceil(filter_support(filter) * fs)) * 2 + 1;
}

__host__ __device__ inline long long align16(long long v) { return (v + 15) & ~15ll; }

// workspace bytes of one image: horizontal table [out_w][2 + ksize_h], vertical table [out_h][2 + ksize_v] (int32: tap
// start, tap count, weights), and the intermediate rows when both passes run (at most in_h rows of out_w pixels)
__host__ __device__ inline long long image_ws_bytes(int ih, int iw, int oh, int ow, int ch, int filter) {
    if (ih <= 0 || iw <= 0 || oh <= 0 || ow <= 0) return 0;
    long long b = align16(4ll * ow * (2 + axis_ksize(iw, ow, filter)));
    b += align16(4ll * oh * (2 + axis_ksize(ih, oh, filter)));
    if (ow != iw && oh != ih) b += align16(static_cast<long long>(ih) * ow * ch);
    return b;
}

struct ResizeParams {
    const unsigned char* src;
    const long long* src_off;   // [n] byte offsets
    const int* src_hw;          // [n][2]
    unsigned char* dst;
    const long long* dst_off;
    const int* dst_hw;
    unsigned char* ws;
    long long ws_bytes;
    int n, ch, filter;
};

struct ImageGeo {
    int ih, iw, oh, ow, kh, kv;
    long long ws_off, ws_len;
    int* coef_h;                // [ow][2 + kh]
    int* coef_v;                // [oh][2 + kv]
    unsigned char* tmp;         // [rows the vertical pass reads][ow][ch], when both passes run
    bool fits;
};

// geometry of image b; the workspace offset is the sum of the preceding images' sizes, summed by the whole CTA
__device__ ImageGeo image_geo(const ResizeParams& p, int b) {
    __shared__ unsigned long long s_off;
    if (threadIdx.x == 0) s_off = 0;
    __syncthreads();
    unsigned long long part = 0;
    for (int j = threadIdx.x; j < b; j += blockDim.x)
        part += static_cast<unsigned long long>(image_ws_bytes(p.src_hw[2 * j], p.src_hw[2 * j + 1], p.dst_hw[2 * j],
                                                               p.dst_hw[2 * j + 1], p.ch, p.filter));
    if (part) atomicAdd(&s_off, part);
    __syncthreads();
    ImageGeo g;
    g.ih = p.src_hw[2 * b]; g.iw = p.src_hw[2 * b + 1];
    g.oh = p.dst_hw[2 * b]; g.ow = p.dst_hw[2 * b + 1];
    g.ws_off = static_cast<long long>(s_off);
    g.ws_len = image_ws_bytes(g.ih, g.iw, g.oh, g.ow, p.ch, p.filter);
    g.fits = g.ws_len > 0 && g.ws_off + g.ws_len <= p.ws_bytes;
    g.kh = g.fits ? axis_ksize(g.iw, g.ow, p.filter) : 0;
    g.kv = g.fits ? axis_ksize(g.ih, g.oh, p.filter) : 0;
    g.coef_h = reinterpret_cast<int*>(p.ws + g.ws_off);
    g.coef_v = reinterpret_cast<int*>(p.ws + g.ws_off + align16(4ll * g.ow * (2 + g.kh)));
    g.tmp = p.ws + g.ws_off + align16(4ll * g.ow * (2 + g.kh)) + align16(4ll * g.oh * (2 + g.kv));
    return g;
}

// Pillow's filters, one rounded operation at a time (bicubic: Keys' cubic with a = −0.5; a + 2 and a + 3 are exact)
__device__ __forceinline__ double eval_filter(int filter, double x) {
    x = fabs(x);
    if (filter == SOD_RESIZE_BILINEAR) return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
    return 0.0;
}

// precompute_coeffs + normalize_coeffs_8bpc for output pixel xx of an axis: row[0] = first tap, row[1] = tap count,
// row[2 ..] = weights in 22-bit fixed point
__device__ void axis_coeffs(int in, int out, int filter, int xx, int* row) {
    const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = __dmul_rn(filter_support(filter), filterscale);
    const double ss = __ddiv_rn(1.0, filterscale);
    const double center = __dmul_rn(__dadd_rn(static_cast<double>(xx), 0.5), scale);
    int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, support), 0.5));
    if (xmin < 0) xmin = 0;
    int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, support), 0.5));
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x)
        ww = __dadd_rn(ww, eval_filter(filter, __dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss)));
    row[0] = xmin;
    row[1] = xmax;
    for (int x = 0; x < xmax; ++x) {
        double k = eval_filter(filter, __dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
        if (ww != 0.0) k = __ddiv_rn(k, ww);
        const double s = __dmul_rn(k, static_cast<double>(1 << kPrecisionBits));
        row[2 + x] = static_cast<int>(k < 0.0 ? __dadd_rn(s, -0.5) : __dadd_rn(s, 0.5));      // (int): towards zero
    }
}

__device__ __forceinline__ unsigned char clip8(int acc) {
    acc >>= kPrecisionBits;                                   // arithmetic shift, as Pillow's clip8
    return static_cast<unsigned char>(acc < 0 ? 0 : (acc > 255 ? 255 : acc));
}

__global__ void __launch_bounds__(kThreads) resize_coeff_kernel(const __grid_constant__ ResizeParams p) {
    const int b = blockIdx.x;
    const ImageGeo g = image_geo(p, b);
    if (!g.fits) return;
    const int total = g.ow + g.oh;
    for (int t = blockIdx.y * blockDim.x + threadIdx.x; t < total; t += gridDim.y * blockDim.x) {
        if (t < g.ow) axis_coeffs(g.iw, g.ow, p.filter, t, g.coef_h + static_cast<long long>(t) * (2 + g.kh));
        else axis_coeffs(g.ih, g.oh, p.filter, t - g.ow, g.coef_v + static_cast<long long>(t - g.ow) * (2 + g.kv));
    }
}

// horizontal pass: rows [ybox_first, ybox_last) of the source → intermediate (or straight to dst when the height does
// not change); an image whose size does not change at all is copied here
template <int CH>
__device__ void horizontal(const ResizeParams& p, const ImageGeo& g, int b) {
    const unsigned char* src = p.src + p.src_off[b];
    unsigned char* dst = p.dst + p.dst_off[b];
    if (g.ow == g.iw) {
        if (g.oh == g.ih) {
            const long long bytes = static_cast<long long>(g.ih) * g.iw * CH;
            for (long long i = static_cast<long long>(blockIdx.y) * blockDim.x + threadIdx.x; i < bytes;
                 i += static_cast<long long>(gridDim.y) * blockDim.x)
                dst[i] = src[i];
        }
        return;
    }
    const bool vertical_next = g.oh != g.ih;
    const int* last_v = g.coef_v + static_cast<long long>(g.oh - 1) * (2 + g.kv);
    const int first = g.coef_v[0], rows = last_v[0] + last_v[1] - first;
    unsigned char* out = vertical_next ? g.tmp : dst;
    const int row_elems = g.ow * CH;
    for (int r = blockIdx.y; r < rows; r += gridDim.y) {
        const unsigned char* in_row = src + static_cast<long long>(first + r) * g.iw * CH;
        unsigned char* out_row = out + static_cast<long long>(r) * row_elems;
        for (int e = threadIdx.x; e < row_elems; e += blockDim.x) {
            const int xx = CH == 1 ? e : e / CH, c = CH == 1 ? 0 : e - xx * CH;
            const int* k = g.coef_h + static_cast<long long>(xx) * (2 + g.kh);
            const int xmin = k[0], cnt = k[1];
            int acc = 1 << (kPrecisionBits - 1);
            for (int x = 0; x < cnt; ++x) acc += static_cast<int>(in_row[(xmin + x) * CH + c]) * k[2 + x];
            out_row[e] = clip8(acc);
        }
    }
}

// vertical pass: intermediate (tap starts shifted by ybox_first) or, when the width does not change, the source → dst
template <int CH>
__device__ void vertical(const ResizeParams& p, const ImageGeo& g, int b) {
    if (g.oh == g.ih) return;
    const bool from_tmp = g.ow != g.iw;
    const unsigned char* in = from_tmp ? g.tmp : p.src + p.src_off[b];
    const int shift = from_tmp ? g.coef_v[0] : 0;
    unsigned char* dst = p.dst + p.dst_off[b];
    const int row_elems = g.ow * CH;
    for (int yy = blockIdx.y; yy < g.oh; yy += gridDim.y) {
        const int* k = g.coef_v + static_cast<long long>(yy) * (2 + g.kv);
        const int ymin = k[0] - shift, cnt = k[1];
        unsigned char* out_row = dst + static_cast<long long>(yy) * row_elems;
        for (int e = threadIdx.x; e < row_elems; e += blockDim.x) {
            int acc = 1 << (kPrecisionBits - 1);
            for (int y = 0; y < cnt; ++y) acc += static_cast<int>(in[static_cast<long long>(ymin + y) * row_elems + e]) * k[2 + y];
            out_row[e] = clip8(acc);
        }
    }
}

__global__ void __launch_bounds__(kThreads) resize_horizontal_kernel(const __grid_constant__ ResizeParams p) {
    const int b = blockIdx.x;
    const ImageGeo g = image_geo(p, b);
    if (!g.fits) return;
    if (p.ch == 1) horizontal<1>(p, g, b);
    else horizontal<3>(p, g, b);
}

__global__ void __launch_bounds__(kThreads) resize_vertical_kernel(const __grid_constant__ ResizeParams p) {
    const int b = blockIdx.x;
    const ImageGeo g = image_geo(p, b);
    if (!g.fits) return;
    if (p.ch == 1) vertical<1>(p, g, b);
    else vertical<3>(p, g, b);
}

bool valid_resize_mode(int channels, int filter) {
    return (channels == 1 || channels == 3) && (filter == SOD_RESIZE_BILINEAR || filter == SOD_RESIZE_BICUBIC);
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_resize_u8_workspace_bytes(int n, const int32_t* src_hw, const int32_t* dst_hw, int channels, int filter) {
    using namespace sod;
    if (n <= 0 || !src_hw || !dst_hw || !valid_resize_mode(channels, filter)) return 0;
    long long total = 0;
    for (int i = 0; i < n; ++i) {
        const long long b = image_ws_bytes(src_hw[2 * i], src_hw[2 * i + 1], dst_hw[2 * i], dst_hw[2 * i + 1], channels, filter);
        if (b == 0) return 0;
        total += b;
    }
    return static_cast<size_t>(total);
}

extern "C" int sod_resize_u8(const void* src, const int64_t* src_off, const int32_t* src_hw, void* dst, const int64_t* dst_off,
                             const int32_t* dst_hw, int n, int channels, int filter, void* workspace, size_t workspace_bytes,
                             void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(src && src_off && src_hw && dst && dst_off && dst_hw && n > 0, SOD_EINVAL);
    SOD_CHECK_ARG(valid_resize_mode(channels, filter), SOD_EINVAL);
    SOD_CHECK_ARG(workspace && workspace_bytes > 0, SOD_EINVAL);
    ResizeParams p;
    p.src = static_cast<const unsigned char*>(src); p.src_off = reinterpret_cast<const long long*>(src_off); p.src_hw = src_hw;
    p.dst = static_cast<unsigned char*>(dst); p.dst_off = reinterpret_cast<const long long*>(dst_off); p.dst_hw = dst_hw;
    p.ws = static_cast<unsigned char*>(workspace); p.ws_bytes = static_cast<long long>(workspace_bytes);
    p.n = n; p.ch = channels; p.filter = filter;
    // rows per image are only known on the device: a fixed number of row-CTAs per image, about 8 waves in all
    int per = (8 * dev_info().sm_count + n - 1) / n;
    per = per < 1 ? 1 : (per > 128 ? 128 : per);
    const dim3 grid(static_cast<unsigned>(n), static_cast<unsigned>(per));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    resize_coeff_kernel<<<grid, kThreads, 0, s>>>(p);
    resize_horizontal_kernel<<<grid, kThreads, 0, s>>>(p);
    resize_vertical_kernel<<<grid, kThreads, 0, s>>>(p);
    return static_cast<int>(cudaGetLastError());
}
