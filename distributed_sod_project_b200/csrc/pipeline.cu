// pipeline.cu — the two data-side neighbours of the training iteration (SURVEY §8f.2 and §8f.4):
//
//  (a) batch pre-processing: what the reference does per sample on DataLoader workers and in its collate function
//      (utils/dataset.py:86-96 ToTensor + Normalize, :110-116 mask ToTensor, :125-132 multi-scale collate with
//      F.interpolate bilinear / nearest) as ONE kernel over the uint8 batch: the host ships 4 bytes per pixel
//      (RGB + mask, uint8) instead of 16 (fp32 planes), and normalisation, the optional horizontal flip
//      (utils/joint_transforms.py:19-23) and the resize to the batch's training size never touch HBM as separate passes.
//      Output is written channels-last, the layout the first convolution wants.
//
//  (b) saliency-metric sufficient statistics: the reference evaluates MAE / F-measure / S-measure / E-measure per image
//      with ≈40 numpy passes on the CPU (utils/saliency_metric.py:8-239).  After the reference's own normalisation
//      (train.py:399-409) a prediction is k/D with integer k = u - min(u), D = max(u) - min(u) ≤ 255, and the ground
//      truth is binary, so EVERY one of those metrics is a function of the joint histogram of (k, gt) taken separately
//      over the four quadrants around the ground truth's centre of mass (S-measure's region term).  Two small integer
//      kernels per batch produce those histograms — exact (integer atomics: no rounding, no order dependence) — and
//      the host evaluates the reference's formulas on 2048 counters per image.
#include "common.cuh"

namespace sod {
namespace {

// ---------------------------------------------------------------------------------------------------------------
// (a) pre-processing
// ---------------------------------------------------------------------------------------------------------------
struct PrepParams {
    const unsigned char* img;    // [N, Hs, Ws, 3]
    const unsigned char* mask;   // [N, Hs, Ws] or null
    const unsigned char* flip;   // [N] (non-zero: mirror left-right) or null
    void* out_img;               // [N, Ho, Wo, 3] (channels-last storage of an [N,3,Ho,Wo] tensor), fp32 or bf16
    float* out_mask;             // [N, 1, Ho, Wo] fp32 or null
    int n, hs, ws, ho, wo;
    float mean[3], stdv[3];
    float scale_h, scale_w;      // hs/ho, ws/wo as torch computes them (area_pixel_compute_scale, align_corners=False)
};

// ToTensor → Normalize in torch's operation order: (u / 255) - mean, then / std, all fp32
__device__ __forceinline__ float norm_px(unsigned char u, float mean, float stdv) {
    return (static_cast<float>(u) / 255.0f - mean) / stdv;
}

template <typename T>
__global__ void __launch_bounds__(256) preprocess_kernel(const __grid_constant__ PrepParams p) {
    const long long total = static_cast<long long>(p.n) * p.ho * p.wo;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ox = static_cast<int>(i % p.wo);
        const int oy = static_cast<int>((i / p.wo) % p.ho);
        const int b = static_cast<int>(i / (static_cast<long long>(p.wo) * p.ho));
        const bool mirror = p.flip != nullptr && p.flip[b] != 0;
        const unsigned char* im = p.img + static_cast<size_t>(b) * p.hs * p.ws * 3;
        float v[3];
        if (p.hs == p.ho && p.ws == p.wo) {
            const int sx = mirror ? p.ws - 1 - ox : ox;
            const unsigned char* px = im + (static_cast<size_t>(oy) * p.ws + sx) * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[c] = norm_px(px[c], p.mean[c], p.stdv[c]);
        } else {
            // upsample_bilinear2d, align_corners=False: src = scale * (dst + 0.5) - 0.5, clamped at 0
            float fy = p.scale_h * (static_cast<float>(oy) + 0.5f) - 0.5f;
            float fx = p.scale_w * (static_cast<float>(ox) + 0.5f) - 0.5f;
            fy = fy < 0.f ? 0.f : fy;
            fx = fx < 0.f ? 0.f : fx;
            const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
            const int y1 = y0 + (y0 < p.hs - 1 ? 1 : 0), x1 = x0 + (x0 < p.ws - 1 ? 1 : 0);
            const float ly = fy - static_cast<float>(y0), lx = fx - static_cast<float>(x0);
            const float hy = 1.f - ly, hx = 1.f - lx;
            // the flip happened BEFORE the tensor existed (PIL transpose): sample the mirrored image
            const int a0 = mirror ? p.ws - 1 - x0 : x0, a1 = mirror ? p.ws - 1 - x1 : x1;
            const unsigned char* r0 = im + static_cast<size_t>(y0) * p.ws * 3;
            const unsigned char* r1 = im + static_cast<size_t>(y1) * p.ws * 3;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float v00 = norm_px(r0[a0 * 3 + c], p.mean[c], p.stdv[c]), v01 = norm_px(r0[a1 * 3 + c], p.mean[c], p.stdv[c]);
                const float v10 = norm_px(r1[a0 * 3 + c], p.mean[c], p.stdv[c]), v11 = norm_px(r1[a1 * 3 + c], p.mean[c], p.stdv[c]);
                v[c] = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
            }
        }
        T* o = static_cast<T*>(p.out_img) + i * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) IO<T>::store1(o + c, v[c]);
        if (p.mask != nullptr && p.out_mask != nullptr) {
            // nearest (legacy 'nearest' of F.interpolate): src = min(floor(dst * scale), in - 1)
            int sy = static_cast<int>(floorf(static_cast<float>(oy) * p.scale_h));
            int sx = static_cast<int>(floorf(static_cast<float>(ox) * p.scale_w));
            sy = sy < p.hs - 1 ? sy : p.hs - 1;
            sx = sx < p.ws - 1 ? sx : p.ws - 1;
            if (mirror) sx = p.ws - 1 - sx;
            p.out_mask[i] = static_cast<float>(p.mask[(static_cast<size_t>(b) * p.hs + sy) * p.ws + sx]) / 255.0f;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// (b) saliency-metric statistics
// ---------------------------------------------------------------------------------------------------------------
// Images live where MetricGeo (common.cuh) says; the ground truth is binarised by metric_fg (common.cuh).

// pass 1, one CTA per image: min / max of the uint8 prediction, max of the uint8 ground truth (the reference divides by
// it before thresholding, train.py:400-401), and — once that threshold is known — Σ g, Σ y·g, Σ x·g (centre of mass).
// head[b] = {min_u, max_u, max_gt, _, n_fg, sum_y, sum_x, _} as int64
__global__ void __launch_bounds__(512) metric_head_kernel(const unsigned char* __restrict__ pred, const unsigned char* __restrict__ gt,
                                                          const MetricGeo geo, long long* __restrict__ head) {
    __shared__ int s_min, s_max, s_gmax;
    __shared__ unsigned long long s_n, s_y, s_x;
    const int b = blockIdx.x;
    size_t base;
    int h, w;
    geo.get(b, base, h, w);
    if (threadIdx.x == 0) { s_min = 255; s_max = 0; s_gmax = 0; s_n = 0; s_y = 0; s_x = 0; }
    __syncthreads();
    int mn = 255, mx = 0, gm = 0;
    for (int i = threadIdx.x; i < h * w; i += blockDim.x) {
        const int u = pred[base + i], g = gt[base + i];
        mn = u < mn ? u : mn; mx = u > mx ? u : mx; gm = g > gm ? g : gm;
    }
    atomicMin(&s_min, mn); atomicMax(&s_max, mx); atomicMax(&s_gmax, gm);
    __syncthreads();
    const int gmax = s_gmax;
    unsigned long long n = 0, sy = 0, sx = 0;
    for (int i = threadIdx.x; i < h * w; i += blockDim.x) {
        const int g = gt[base + i];
        if (metric_fg(g, gmax)) { ++n; sy += static_cast<unsigned>(i / w); sx += static_cast<unsigned>(i % w); }
    }
    atomicAdd(&s_n, n); atomicAdd(&s_y, sy); atomicAdd(&s_x, sx);
    __syncthreads();
    if (threadIdx.x == 0) {
        long long* o = head + static_cast<size_t>(b) * 8;
        o[0] = s_min; o[1] = s_max; o[2] = s_gmax; o[3] = 0;
        o[4] = static_cast<long long>(s_n); o[5] = static_cast<long long>(s_y); o[6] = static_cast<long long>(s_x); o[7] = 0;
    }
}

// pass 2, several CTAs per image: joint histogram hist[b][quadrant][gt_bin][k], k = u - min_u, quadrants split at
// (cy[b], cx[b]) — the host derives them from pass 1 exactly as the reference does (int(round(centre)) + 1)
__global__ void __launch_bounds__(256) metric_hist_kernel(const unsigned char* __restrict__ pred, const unsigned char* __restrict__ gt,
                                                          const MetricGeo geo, const long long* __restrict__ head,
                                                          const int* __restrict__ split_yx, unsigned* __restrict__ hist) {
    __shared__ unsigned s_h[4 * 2 * 256];
    const int b = blockIdx.y;
    for (int i = threadIdx.x; i < 2048; i += blockDim.x) s_h[i] = 0;
    __syncthreads();
    size_t base;
    int h, w;
    geo.get(b, base, h, w);
    const int mn = static_cast<int>(head[static_cast<size_t>(b) * 8 + 0]);
    const int gmax = static_cast<int>(head[static_cast<size_t>(b) * 8 + 2]);
    const int cy = split_yx[2 * b], cx = split_yx[2 * b + 1];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < h * w; i += gridDim.x * blockDim.x) {
        const int y = i / w, x = i % w;
        const int q = (y >= cy ? 2 : 0) + (x >= cx ? 1 : 0);          // LT, RT, LB, RB
        const int g = metric_fg(static_cast<int>(gt[base + i]), gmax) ? 1 : 0;
        atomicAdd(&s_h[(q * 2 + g) * 256 + (static_cast<int>(pred[base + i]) - mn)], 1u);
    }
    __syncthreads();
    unsigned* out = hist + static_cast<size_t>(b) * 2048;
    for (int i = threadIdx.x; i < 2048; i += blockDim.x)
        if (s_h[i]) atomicAdd(out + i, s_h[i]);
}

// float prediction in [0,1] → the uint8 the reference's ToPILImage produces (mul(255).byte(): truncation)
template <typename T>
__global__ void quantize_kernel(const T* __restrict__ p, unsigned char* __restrict__ out, long long n, int apply_sigmoid) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        float v = IO<T>::load1(p + i);
        if (apply_sigmoid) v = 1.0f / (1.0f + expf(-v));
        v = v * 255.0f;
        v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v);
        out[i] = static_cast<unsigned char>(v);
    }
}

}  // namespace
}  // namespace sod

extern "C" int sod_preprocess_batch(const void* img_u8, const void* mask_u8, const void* flip_u8, void* out_img, int out_dtype,
                                    float* out_mask, int n, int hs, int ws, int ho, int wo, const float* mean3,
                                    const float* std3, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(img_u8 && out_img && mean3 && std3 && n > 0 && hs > 0 && ws > 0 && ho > 0 && wo > 0, SOD_EINVAL);
    SOD_CHECK_ARG((mask_u8 == nullptr) == (out_mask == nullptr), SOD_EINVAL);
    PrepParams p;
    p.img = static_cast<const unsigned char*>(img_u8); p.mask = static_cast<const unsigned char*>(mask_u8);
    p.flip = static_cast<const unsigned char*>(flip_u8); p.out_img = out_img; p.out_mask = out_mask;
    p.n = n; p.hs = hs; p.ws = ws; p.ho = ho; p.wo = wo;
    for (int c = 0; c < 3; ++c) {
        p.mean[c] = mean3[c]; p.stdv[c] = std3[c];
        if (!(std3[c] != 0.f)) return SOD_EINVAL;
    }
    p.scale_h = static_cast<float>(hs) / static_cast<float>(ho);
    p.scale_w = static_cast<float>(ws) / static_cast<float>(wo);
    const long long total = static_cast<long long>(n) * ho * wo;
    long long blocks = (total + 255) / 256;
    const long long cap = 16ll * dev_info().sm_count;
    if (blocks > cap) blocks = cap;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (out_dtype == SOD_F32) preprocess_kernel<float><<<static_cast<unsigned>(blocks), 256, 0, s>>>(p);
    else if (out_dtype == SOD_BF16) preprocess_kernel<__nv_bfloat16><<<static_cast<unsigned>(blocks), 256, 0, s>>>(p);
    else if (out_dtype == SOD_F16) preprocess_kernel<__half><<<static_cast<unsigned>(blocks), 256, 0, s>>>(p);
    else return SOD_EINVAL;
    return static_cast<int>(cudaGetLastError());
}

extern "C" int sod_saliency_quantize(const void* pred, int dtype, void* out_u8, int64_t n, int apply_sigmoid, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred && out_u8 && n > 0, SOD_EINVAL);
    long long blocks = (n + 255) / 256;
    const long long cap = 8ll * dev_info().sm_count;
    if (blocks > cap) blocks = cap;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return SOD_DISPATCH_DTYPE(dtype, T, [&]() -> int {
        quantize_kernel<T><<<static_cast<unsigned>(blocks), 256, 0, s>>>(static_cast<const T*>(pred), static_cast<unsigned char*>(out_u8), n, apply_sigmoid);
        return static_cast<int>(cudaGetLastError());
    });
}

namespace sod {
namespace {

int launch_head(const void* pred_u8, const void* gt_u8, int n, MetricGeo geo, int64_t* head, void* stream) {
    metric_head_kernel<<<n, 512, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const unsigned char*>(pred_u8),
                                                                       static_cast<const unsigned char*>(gt_u8), geo,
                                                                       reinterpret_cast<long long*>(head));
    return static_cast<int>(cudaGetLastError());
}

int launch_hist(const void* pred_u8, const void* gt_u8, int n, MetricGeo geo, int per, const int64_t* head,
                const int32_t* split_yx, uint32_t* hist, void* stream) {
    metric_hist_kernel<<<dim3(per, n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const unsigned char*>(pred_u8), static_cast<const unsigned char*>(gt_u8), geo,
        reinterpret_cast<const long long*>(head), split_yx, hist);
    return static_cast<int>(cudaGetLastError());
}

}  // namespace
}  // namespace sod

extern "C" int sod_saliency_head(const void* pred_u8, const void* gt_u8, int n, int h, int w, int64_t* head, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred_u8 && gt_u8 && head && n > 0 && h > 0 && w > 0, SOD_EINVAL);
    SOD_CHECK_ARG(static_cast<long long>(h) * w < (1ll << 31), SOD_EUNSUPPORTED);
    return launch_head(pred_u8, gt_u8, n, MetricGeo{nullptr, nullptr, h, w}, head, stream);
}

extern "C" int sod_saliency_hist(const void* pred_u8, const void* gt_u8, int n, int h, int w, const int64_t* head,
                                 const int32_t* split_yx, uint32_t* hist, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred_u8 && gt_u8 && head && split_yx && hist && n > 0 && h > 0 && w > 0, SOD_EINVAL);
    SOD_CHECK_ARG(static_cast<long long>(h) * w < (1ll << 31), SOD_EUNSUPPORTED);
    int per = (h * w + 256 * 16 - 1) / (256 * 16);
    if (per < 1) per = 1;
    if (per > 64) per = 64;
    return launch_hist(pred_u8, gt_u8, n, MetricGeo{nullptr, nullptr, h, w}, per, head, split_yx, hist, stream);
}

extern "C" int sod_saliency_head_ragged(const void* pred_u8, const void* gt_u8, int n, const int64_t* offsets,
                                        const int32_t* hw, int64_t* head, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred_u8 && gt_u8 && offsets && hw && head && n > 0, SOD_EINVAL);
    return launch_head(pred_u8, gt_u8, n, MetricGeo{reinterpret_cast<const long long*>(offsets), hw, 0, 0}, head, stream);
}

extern "C" int sod_saliency_hist_ragged(const void* pred_u8, const void* gt_u8, int n, const int64_t* offsets,
                                        const int32_t* hw, const int64_t* head, const int32_t* split_yx, uint32_t* hist,
                                        void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred_u8 && gt_u8 && offsets && hw && head && split_yx && hist && n > 0, SOD_EINVAL);
    // image sizes live on the device: a fixed number of CTAs per image, about 4 waves in all
    int per = (4 * dev_info().sm_count + n - 1) / n;
    if (per < 1) per = 1;
    if (per > 64) per = 64;
    return launch_hist(pred_u8, gt_u8, n, MetricGeo{reinterpret_cast<const long long*>(offsets), hw, 0, 0}, per, head,
                       split_yx, hist, stream);
}
