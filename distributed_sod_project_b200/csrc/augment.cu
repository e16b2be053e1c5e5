// augment.cu — the reference's random training augmentation after JointResize, bit for bit, for given per-sample
// parameters (utils/joint_transforms.py:20-48, utils/dataset.py:86-95):
//   RandomHorizontallyFlip → RandomRotate(10): img.rotate(deg, BILINEAR), mask.rotate(deg, NEAREST) →
//   ColorJitter(0.1, 0.1, 0.1) on the image (brightness, contrast, saturation in a drawn order).
//
// Pillow's rotate (libImaging/Geometry.c) maps output pixel (x, y) to the source through an affine matrix a[6]:
//   - "RGB" BILINEAR, the generic transform in double: x' = a0·(x+.5) + a1·(y+.5) + a2 (same for y'); outside
//     [0, w) × [0, h) → 0; else x' − .5, floor, taps x0 / x0+1 clamped into the image, row y clamped, row y+1 only if it
//     exists (else the first row's value); lerp in x, then in y; truncated to 8 bits;
//   - "L" NEAREST, 16.16 fixed point: FIX(v) = floor(v·65536 + .5) of a0, a1, a3, a4 and of a2 + a0/2 + a1/2,
//     a5 + a3/2 + a4/2, then integer stepping and >> 16.  Integer addition is associative, so A2 + y·A1 + x·A0 gives the
//     stepped value exactly.
// The flip comes first and is exact, so it is folded into the source column index.  Every double operation is an
// explicitly rounded intrinsic: Pillow's x86-64 build contracts nothing, and nvcc would fuse a·b + c into an FMA.
//
// ColorJitter's operations are `Image.blend(degenerate, img, f)` = d + f·(x − d) in float32, clipped and truncated:
// brightness d = 0, contrast d = int(mean(L) + .5) over the whole image as it stands, saturation d = L of the pixel,
// L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16.  The contrast mean comes from an exact integer sum, so the reduction
// order does not matter.
//
// Two launches over images × row tiles: (A) flip + rotate of image and mask, the operations before contrast and the
// L sums; (B) contrast and the operations after it, in place.
#include <cmath>

#include "common.cuh"

namespace sod {
namespace {

constexpr int kThreads = 256;
constexpr int kPixelsPerCta = 1024;
constexpr int kMaxSize = 16384;          // keeps every 16.16 coordinate of a ±90° rotation inside Pillow's fixed-point range
enum { kBrightness = 0, kContrast = 1, kSaturation = 2 };

struct AugmentParams {
    const unsigned char* img;
    const unsigned char* mask;
    unsigned char* img_out;
    unsigned char* mask_out;
    const sod_augment_param* prm;       // [n], in the workspace
    unsigned long long* lsum;           // [n] Σ L of the image entering contrast
    int n, size, rows_per_tile;
};

__device__ __forceinline__ int luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ int blend(int d, int x, float f) {
    float t = __fadd_rn(static_cast<float>(d), __fmul_rn(f, static_cast<float>(x - d)));
    t = t <= 0.0f ? 0.0f : (t >= 255.0f ? 255.0f : t);
    return static_cast<int>(t);
}

// one jitter operation on one pixel; `mean` is the contrast degenerate
__device__ __forceinline__ void jitter(int op, float f, int mean, int& r, int& g, int& b) {
    const int d = op == kBrightness ? 0 : (op == kContrast ? mean : luma(r, g, b));
    r = blend(d, r, f);
    g = blend(d, g, f);
    b = blend(d, b, f);
}

__device__ __forceinline__ int fix16(double v) { return static_cast<int>(floor(__dadd_rn(__dmul_rn(v, 65536.0), 0.5))); }

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void __launch_bounds__(kThreads) augment_rotate_kernel(const __grid_constant__ AugmentParams p) {
    const int b = blockIdx.x, S = p.size;
    const sod_augment_param& P = p.prm[b];
    const long long plane = static_cast<long long>(S) * S;
    const unsigned char* img = p.img + plane * 3 * b;
    const unsigned char* mask = p.mask + plane * b;
    unsigned char* img_out = p.img_out + plane * 3 * b;
    unsigned char* mask_out = p.mask_out + plane * b;
    const bool flip = P.flip != 0, ident = P.identity != 0;
    const double a0 = P.rot[0], a1 = P.rot[1], a2 = P.rot[2], a3 = P.rot[3], a4 = P.rot[4], a5 = P.rot[5];
    const int f0 = fix16(a0), f1 = fix16(a1), f3 = fix16(a3), f4 = fix16(a4);
    const int f2 = fix16(__dadd_rn(__dadd_rn(a2, __dmul_rn(a0, 0.5)), __dmul_rn(a1, 0.5)));
    const int f5 = fix16(__dadd_rn(__dadd_rn(a5, __dmul_rn(a3, 0.5)), __dmul_rn(a4, 0.5)));
    int pre = 0;                                              // operations before contrast
    while (pre < 3 && P.ops[pre] != kContrast) ++pre;
    const int y_begin = blockIdx.y * p.rows_per_tile;
    const int y_end = min(S, y_begin + p.rows_per_tile);
    const int count = (y_end - y_begin) * S;
    unsigned int part = 0;
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
        const int y = y_begin + i / S, x = i - (i / S) * S;
        const long long o = static_cast<long long>(y) * S + x;
        int c[3];
        if (ident) {
            const long long s = static_cast<long long>(y) * S + (flip ? S - 1 - x : x);
            mask_out[o] = mask[s];
            for (int k = 0; k < 3; ++k) c[k] = img[3 * s + k];
        } else {
            // mask: nearest, 16.16 fixed point (int32 wrap-around as Pillow's stepping)
            const int xi = static_cast<int>(static_cast<unsigned int>(f2) + static_cast<unsigned int>(y) * f1 + static_cast<unsigned int>(x) * f0) >> 16;
            const int yi = static_cast<int>(static_cast<unsigned int>(f5) + static_cast<unsigned int>(y) * f4 + static_cast<unsigned int>(x) * f3) >> 16;
            mask_out[o] = (xi >= 0 && xi < S && yi >= 0 && yi < S)
                              ? mask[static_cast<long long>(yi) * S + (flip ? S - 1 - xi : xi)] : 0;
            // image: bilinear in double
            const double xs = x + 0.5, ys = y + 0.5;
            double xin = __dadd_rn(__dadd_rn(__dmul_rn(a0, xs), __dmul_rn(a1, ys)), a2);
            double yin = __dadd_rn(__dadd_rn(__dmul_rn(a3, xs), __dmul_rn(a4, ys)), a5);
            if (xin < 0.0 || xin >= S || yin < 0.0 || yin >= S) {
                c[0] = c[1] = c[2] = 0;
            } else {
                xin = __dsub_rn(xin, 0.5);
                yin = __dsub_rn(yin, 0.5);
                const double xf = floor(xin), yf = floor(yin);
                const double dx = __dsub_rn(xin, xf), dy = __dsub_rn(yin, yf);
                const int xl = static_cast<int>(xf), yl = static_cast<int>(yf);
                int xa = clampi(xl, 0, S - 1), xb = clampi(xl + 1, 0, S - 1);
                if (flip) { xa = S - 1 - xa; xb = S - 1 - xb; }
                const unsigned char* r0 = img + static_cast<long long>(clampi(yl, 0, S - 1)) * S * 3;
                const bool has2 = yl + 1 >= 0 && yl + 1 < S;
                const unsigned char* r1 = img + static_cast<long long>(has2 ? yl + 1 : 0) * S * 3;
                for (int k = 0; k < 3; ++k) {
                    const int u0 = r0[3 * xa + k], u1 = r0[3 * xb + k];
                    const double v1 = __dadd_rn(static_cast<double>(u0), __dmul_rn(static_cast<double>(u1 - u0), dx));
                    double v2 = v1;
                    if (has2) {
                        const int w0 = r1[3 * xa + k], w1 = r1[3 * xb + k];
                        v2 = __dadd_rn(static_cast<double>(w0), __dmul_rn(static_cast<double>(w1 - w0), dx));
                    }
                    c[k] = static_cast<int>(__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy)));
                }
            }
        }
        for (int j = 0; j < pre; ++j) jitter(P.ops[j], P.factor[P.ops[j]], 0, c[0], c[1], c[2]);
        part += luma(c[0], c[1], c[2]);
        for (int k = 0; k < 3; ++k) img_out[3 * o + k] = static_cast<unsigned char>(c[k]);
    }
    for (int d = 16; d > 0; d >>= 1) part += __shfl_down_sync(0xffffffffu, part, d);
    if ((threadIdx.x & 31) == 0 && part) atomicAdd(p.lsum + b, static_cast<unsigned long long>(part));
}

__global__ void __launch_bounds__(kThreads) augment_contrast_kernel(const __grid_constant__ AugmentParams p) {
    const int b = blockIdx.x, S = p.size;
    const sod_augment_param& P = p.prm[b];
    const long long plane = static_cast<long long>(S) * S;
    unsigned char* img = p.img_out + plane * 3 * b;
    // ImageStat's mean (an exact sum over the pixel count, one rounding), + .5, int()
    const int mean = static_cast<int>(__dadd_rn(__ddiv_rn(static_cast<double>(p.lsum[b]), static_cast<double>(plane)), 0.5));
    int first = 0;
    while (first < 3 && P.ops[first] != kContrast) ++first;
    const int y_begin = blockIdx.y * p.rows_per_tile;
    const int y_end = min(S, y_begin + p.rows_per_tile);
    const long long base = static_cast<long long>(y_begin) * S;
    const int count = (y_end - y_begin) * S;
    for (int i = threadIdx.x; i < count; i += blockDim.x) {
        unsigned char* px = img + 3 * (base + i);
        int c0 = px[0], c1 = px[1], c2 = px[2];
        for (int j = first; j < 3; ++j) jitter(P.ops[j], P.factor[P.ops[j]], mean, c0, c1, c2);
        px[0] = static_cast<unsigned char>(c0);
        px[1] = static_cast<unsigned char>(c1);
        px[2] = static_cast<unsigned char>(c2);
    }
}

long long align16(long long v) { return (v + 15) & ~15ll; }

}  // namespace
}  // namespace sod

extern "C" size_t sod_augment_u8_workspace_bytes(int n) {
    if (n <= 0) return 0;
    return static_cast<size_t>(sod::align16(static_cast<long long>(n) * sizeof(sod_augment_param)) + 8ll * n);
}

extern "C" int sod_augment_u8(const void* img, const void* mask, void* img_out, void* mask_out, int n, int size,
                              const sod_augment_param* params, void* workspace, size_t workspace_bytes, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(img && mask && img_out && mask_out && params && workspace, SOD_EINVAL);
    SOD_CHECK_ARG(n > 0 && size > 0 && size <= kMaxSize, SOD_EINVAL);
    SOD_CHECK_ARG(workspace_bytes >= sod_augment_u8_workspace_bytes(n), SOD_EINVAL);
    for (int i = 0; i < n; ++i) {
        unsigned seen = 0;
        for (int k = 0; k < 3; ++k) {
            const int op = params[i].ops[k];
            SOD_CHECK_ARG(op >= 0 && op < 3, SOD_EINVAL);
            seen |= 1u << op;
        }
        SOD_CHECK_ARG(seen == 7u, SOD_EINVAL);
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    AugmentParams p;
    p.img = static_cast<const unsigned char*>(img); p.mask = static_cast<const unsigned char*>(mask);
    p.img_out = static_cast<unsigned char*>(img_out); p.mask_out = static_cast<unsigned char*>(mask_out);
    p.prm = static_cast<const sod_augment_param*>(workspace);
    p.lsum = reinterpret_cast<unsigned long long*>(static_cast<unsigned char*>(workspace) +
                                                   align16(static_cast<long long>(n) * sizeof(sod_augment_param)));
    p.n = n; p.size = size;
    // row tiles of about kPixelsPerCta pixels: bs 16 at 320² is 16 × 107 CTAs
    p.rows_per_tile = size >= kPixelsPerCta ? 1 : kPixelsPerCta / size;
    const int tiles = (size + p.rows_per_tile - 1) / p.rows_per_tile;
    // the parameters are copied out of the caller's (pageable) memory before this call returns
    cudaError_t e = cudaMemcpyAsync(const_cast<sod_augment_param*>(p.prm), params, sizeof(sod_augment_param) * n,
                                    cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(p.lsum, 0, 8ull * n, s);
    if (e != cudaSuccess) return static_cast<int>(e);
    const dim3 grid(static_cast<unsigned>(n), static_cast<unsigned>(tiles));
    augment_rotate_kernel<<<grid, kThreads, 0, s>>>(p);
    augment_contrast_kernel<<<grid, kThreads, 0, s>>>(p);
    return static_cast<int>(cudaGetLastError());
}
