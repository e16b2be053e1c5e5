// wfm.cu — the weighted F-measure of the reference (utils/saliency_metric.py:232-303) over a ragged batch of 8-bit
// predictions and ground truths, on scipy's exact nearest-foreground indices.
//
// Per image, with gt binarised and pred normalised as the histogram kernels do (metric_fg, head = min/max/max_gt):
//   Dst, Idx = distance_transform_edt(gt == 0, return_indices=True); E = |pred − gt|; Et = E at Idx (the nearest
//   foreground pixel; a foreground pixel is its own); EA = 7×7 Gaussian of Et, zero padded; Ew = min(E, EA) on the
//   foreground where EA < E, E·(2 − exp(log(0.5)/5 · Dst)) on the background;
//   sums = {ΣEw[gt], ΣEw[~gt], n_fg}.
// The host forms Q from the sums.
//
// The feature transform is scipy's (ndimage/src/ni_morphology.c), two separable 1-D lower-envelope sweeps, and what has
// to match is the INDEX it picks on ties, not only the distance: Et takes the error of that pixel.
//   column pass  one thread per (image, column).  With no perpendicular distance (R ≡ 0) the envelope keeps every
//                site and the query picks the nearest foreground row, the upper one on a tie: a downward sweep records
//                the last foreground row above, an upward sweep the next one below, and the strictly nearer wins.
//                Writes the row, or −1 for a column without foreground.
//   row pass     one thread per (image, row), the column pass's rows as sites with R(s) = (row_s − y)²: envelope build
//                (pop v while c·R(v) > b·R(u) + a·R(w) + a·b·c, the same test as scipy's rearranged so that every term
//                is non-negative) and query (move on only while strictly nearer), in int64 — every quantity is an
//                integer, so the comparisons are exact.  Each warp stages 32 rows × 32 columns in shared memory, so
//                reads and writes of the row-major maps stay coalesced.  Writes the nearest (y, x) and the prediction
//                byte there (Et as one byte per pixel).
//   weighted pass  one CTA per 32 × 32 tile: the 7×7 stencil over the tile's Et with a 3-pixel halo in shared
//                memory, then Ew and two per-tile partial sums in a fixed slot; the last CTA of an image (ticket)
//                adds the image's slots in a fixed order.  No floating-point atomics: an image's sums depend on its own
//                pixels alone, bit for bit, whatever shares its batch.
// The stencil's weights and log(0.5)/5 come from the host (the reference's numpy expressions); the stencil adds its 49
// products in scipy's order with explicitly rounded operations, so no FMA contraction separates it from scipy.
#include <cmath>

#include "common.cuh"

namespace sod {
namespace {

constexpr int kColThreads = 128;
constexpr int kRowThreads = 128;          // 4 warps of 32 rows
constexpr int kChunk = 32;                // columns staged per warp at a time
constexpr int kTile = 32;
constexpr int kTileThreads = 256;
constexpr int kHalo = kTile + 6;
constexpr int kMaxWidth = 1 << 21;        // keeps c·R(v) and b·R(u) + a·R(w) + a·b·c below 2^63 when h·w < 2^31

__host__ __device__ inline long long cdiv_ll(long long a, long long b) { return (a + b - 1) / b; }
__host__ __device__ inline long long image_tiles(int h, int w) { return cdiv_ll(h, kTile) * cdiv_ll(w, kTile); }
__host__ __device__ inline long long align16(long long v) { return (v + 15) & ~15ll; }

struct WfmLayout {                        // workspace regions, each 16-byte aligned
    long long col, stack, near, et, part, ticket, total;
};

__host__ __device__ inline WfmLayout wfm_layout(long long px, long long tiles, int n) {
    WfmLayout l;
    l.col = 0;
    l.stack = l.col + align16(4 * px);
    l.near = l.stack + align16(8 * px);
    l.et = l.near + align16(8 * px);
    l.part = l.et + align16(px);
    l.ticket = l.part + align16(16 * tiles);
    l.total = l.ticket + align16(4ll * n);
    return l;
}

struct WfmParams {
    const unsigned char* pred;
    const unsigned char* gt;
    MetricGeo geo;
    const long long* head;    // [n][8] of metric_head_kernel
    int* col;                 // [Σ h·w] column pass: nearest foreground row in the column, −1 if none
    int2* stack;              // [Σ h·w] row pass: envelope (x, row of the site), w entries per row
    int2* near;               // [Σ h·w] (y, x) of the nearest foreground pixel (the caller's nearest_yx, or workspace)
    unsigned char* et;        // [Σ h·w] prediction byte at the nearest foreground pixel
    double* part;             // [Σ tiles][2] per-tile ΣEw[gt], ΣEw[~gt]
    unsigned* ticket;         // [n] tiles of the image finished
    double* sums;             // [n][4]
    double k[49];             // 7×7 Gaussian, row-major
    double log_half_over_5;
};

// image b's pixel and tile offsets in the workspace (the sums of the preceding images' sizes); every thread of the
// CTA must call it
__device__ void image_prefix(const WfmParams& p, int b, long long& px0, long long& tile0) {
    if (p.geo.off == nullptr) {
        px0 = static_cast<long long>(b) * p.geo.h * p.geo.w;
        tile0 = static_cast<long long>(b) * image_tiles(p.geo.h, p.geo.w);
        return;
    }
    __shared__ unsigned long long s_px, s_tiles;
    if (threadIdx.x == 0) { s_px = 0; s_tiles = 0; }
    __syncthreads();
    unsigned long long a = 0, t = 0;
    for (int j = threadIdx.x; j < b; j += blockDim.x) {
        const int h = p.geo.hw[2 * j], w = p.geo.hw[2 * j + 1];
        a += static_cast<unsigned long long>(h) * w;
        t += static_cast<unsigned long long>(image_tiles(h, w));
    }
    if (a) atomicAdd(&s_px, a);
    if (t) atomicAdd(&s_tiles, t);
    __syncthreads();
    px0 = static_cast<long long>(s_px);
    tile0 = static_cast<long long>(s_tiles);
}

__global__ void __launch_bounds__(kColThreads) wfm_column_kernel(const __grid_constant__ WfmParams p) {
    const int b = blockIdx.y;
    size_t base;
    int h, w;
    p.geo.get(b, base, h, w);
    long long px0, tile0;
    image_prefix(p, b, px0, tile0);
    if (blockIdx.x == 0 && threadIdx.x == 0) p.ticket[b] = 0;
    const int x = blockIdx.x * kColThreads + threadIdx.x;
    if (x >= w) return;
    const int gmax = static_cast<int>(p.head[static_cast<size_t>(b) * 8 + 2]);
    const unsigned char* g = p.gt + base + x;
    int* c = p.col + px0 + x;
    int above = -1;
    for (int y = 0; y < h; ++y) {
        if (metric_fg(g[static_cast<size_t>(y) * w], gmax)) above = y;
        c[static_cast<size_t>(y) * w] = above;
    }
    int below = -1;
    for (int y = h - 1; y >= 0; --y) {
        if (metric_fg(g[static_cast<size_t>(y) * w], gmax)) below = y;
        const int a = c[static_cast<size_t>(y) * w];
        c[static_cast<size_t>(y) * w] = (a < 0 || (below >= 0 && below - y < y - a)) ? below : a;
    }
}

__device__ __forceinline__ long long sq(long long v) { return v * v; }

__global__ void __launch_bounds__(kRowThreads) wfm_row_kernel(const __grid_constant__ WfmParams p) {
    __shared__ int s_a[kRowThreads / 32][32][kChunk + 1];     // column rows in; nearest y out
    __shared__ int s_b[kRowThreads / 32][32][kChunk + 1];     // nearest x out
    const int b = blockIdx.y;
    size_t base;
    int h, w;
    p.geo.get(b, base, h, w);
    long long px0, tile0;
    image_prefix(p, b, px0, tile0);
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    const int y0 = blockIdx.x * kRowThreads + warp * 32;
    if (y0 >= h) return;                                       // warp-uniform: no block-wide barrier follows
    const int y = y0 + lane;
    const bool live = y < h;
    int (*sa)[kChunk + 1] = s_a[warp];
    int (*sb)[kChunk + 1] = s_b[warp];
    int2* stk = p.stack + px0 + static_cast<long long>(live ? y : 0) * w;
    int top = 0;
    // envelope build
    for (int c0 = 0; c0 < w; c0 += kChunk) {
        const int cols = min(kChunk, w - c0);
        for (int r = 0; r < 32; ++r)
            if (y0 + r < h && lane < cols) sa[r][lane] = p.col[px0 + static_cast<long long>(y0 + r) * w + c0 + lane];
        __syncwarp();
        if (live) {
            for (int j = 0; j < cols; ++j) {
                const int row = sa[lane][j];
                if (row < 0) continue;
                const int x = c0 + j;
                const long long rw = sq(row - y);
                while (top >= 2) {
                    const int2 v = stk[top - 1], u = stk[top - 2];
                    const long long a = v.x - u.x, bb = x - v.x, c = a + bb;
                    if (c * sq(v.y - y) > bb * sq(u.y - y) + a * rw + a * bb * c) --top;
                    else break;
                }
                stk[top++] = make_int2(x, row);
            }
        }
        __syncwarp();
    }
    // query, and the nearest (y, x) and its prediction byte out, staged back through shared memory
    int l = 0;
    for (int c0 = 0; c0 < w; c0 += kChunk) {
        const int cols = min(kChunk, w - c0);
        if (live) {
            for (int j = 0; j < cols; ++j) {
                const int x = c0 + j;
                int ny = -1, nx = -1;
                if (top > 0) {
                    int2 cur = stk[l];
                    long long dc = sq(cur.x - x) + sq(cur.y - y);
                    while (l + 1 < top) {
                        const int2 nxt = stk[l + 1];
                        const long long dn = sq(nxt.x - x) + sq(nxt.y - y);
                        if (dn < dc) { ++l; cur = nxt; dc = dn; }
                        else break;
                    }
                    ny = cur.y; nx = cur.x;
                }
                sa[lane][j] = ny;
                sb[lane][j] = nx;
            }
        }
        __syncwarp();
        for (int r = 0; r < 32; ++r) {
            if (y0 + r < h && lane < cols) {
                const int ny = sa[r][lane], nx = sb[r][lane];
                const long long i = px0 + static_cast<long long>(y0 + r) * w + c0 + lane;
                p.near[i] = make_int2(ny, nx);
                p.et[i] = ny >= 0 ? p.pred[base + static_cast<size_t>(ny) * w + nx] : 0;
            }
        }
        __syncwarp();
    }
}

// the reference's normalisation: (u − min)/(max − min), or u/255 when max == min
__device__ __forceinline__ double pred_value(int u, int mn, int d) {
    return d > 0 ? __ddiv_rn(static_cast<double>(u - mn), static_cast<double>(d)) : __ddiv_rn(static_cast<double>(u), 255.0);
}

__device__ double block_sum(double v, double* s_warp) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
    if (threadIdx.x % 32 == 0) s_warp[threadIdx.x / 32] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int i = 0; i < kTileThreads / 32; ++i) t = __dadd_rn(t, s_warp[i]);
    __syncthreads();
    return t;                                                  // valid in thread 0
}

__global__ void __launch_bounds__(kTileThreads) wfm_weighted_kernel(const __grid_constant__ WfmParams p) {
    __shared__ double s_et[kHalo][kHalo];
    __shared__ double s_warp[2][kTileThreads / 32];
    __shared__ bool s_last;
    const int b = blockIdx.y;
    size_t base;
    int h, w;
    p.geo.get(b, base, h, w);
    long long px0, tile0;
    image_prefix(p, b, px0, tile0);
    const int tiles_x = static_cast<int>(cdiv_ll(w, kTile));
    const int nt = static_cast<int>(image_tiles(h, w));
    const int t = blockIdx.x;
    if (t >= nt) return;                                       // CTA-uniform
    const long long* hd = p.head + static_cast<size_t>(b) * 8;
    const int mn = static_cast<int>(hd[0]), d = static_cast<int>(hd[1] - hd[0]), gmax = static_cast<int>(hd[2]);
    const long long n_fg = hd[4];
    double acc_fg = 0.0, acc_bg = 0.0;
    if (n_fg > 0) {
        const int ty0 = (t / tiles_x) * kTile, tx0 = (t % tiles_x) * kTile;
        for (int i = threadIdx.x; i < kHalo * kHalo; i += kTileThreads) {
            const int r = i / kHalo, c = i % kHalo, yy = ty0 - 3 + r, xx = tx0 - 3 + c;
            double v = 0.0;                                    // convolve(mode="constant", cval=0)
            if (yy >= 0 && yy < h && xx >= 0 && xx < w)
                v = __dsub_rn(1.0, pred_value(p.et[px0 + static_cast<long long>(yy) * w + xx], mn, d));   // |pred − 1|
            s_et[r][c] = v;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < kTile * kTile; i += kTileThreads) {
            const int r = i / kTile, c = i % kTile, yy = ty0 + r, xx = tx0 + c;
            if (yy >= h || xx >= w) continue;
            const size_t pix = static_cast<size_t>(yy) * w + xx;
            const double v = pred_value(p.pred[base + pix], mn, d);
            if (metric_fg(p.gt[base + pix], gmax)) {
                const double e = __dsub_rn(1.0, v);
                double ea = 0.0;
#pragma unroll
                for (int dy = 0; dy < 7; ++dy)
#pragma unroll
                    for (int dx = 0; dx < 7; ++dx) ea = __dadd_rn(ea, __dmul_rn(s_et[r + dy][c + dx], p.k[dy * 7 + dx]));
                acc_fg = __dadd_rn(acc_fg, ea < e ? ea : e);
            } else {
                const int2 nr = p.near[px0 + static_cast<long long>(pix)];      // (y, x)
                const long long d2 = sq(nr.x - yy) + sq(nr.y - xx);
                const double bw = __dsub_rn(2.0, exp(__dmul_rn(p.log_half_over_5, sqrt(static_cast<double>(d2)))));
                acc_bg = __dadd_rn(acc_bg, __dmul_rn(v, bw));
            }
        }
    }
    acc_fg = block_sum(acc_fg, s_warp[0]);
    acc_bg = block_sum(acc_bg, s_warp[1]);
    double* slot = p.part + 2 * (tile0 + t);
    if (threadIdx.x == 0) {
        slot[0] = acc_fg;
        slot[1] = acc_bg;
        __threadfence();
        s_last = atomicAdd(p.ticket + b, 1u) == static_cast<unsigned>(nt - 1);
    }
    __syncthreads();
    if (!s_last) return;
    // last CTA of the image: its tiles' slots in a fixed order (thread i: tiles i, i + 256, …; then the tree above)
    __threadfence();
    double f = 0.0, g = 0.0;
    for (int i = threadIdx.x; i < nt; i += kTileThreads) {
        f = __dadd_rn(f, __ldcg(p.part + 2 * (tile0 + i)));
        g = __dadd_rn(g, __ldcg(p.part + 2 * (tile0 + i) + 1));
    }
    f = block_sum(f, s_warp[0]);
    g = block_sum(g, s_warp[1]);
    if (threadIdx.x == 0) {
        double* o = p.sums + static_cast<size_t>(b) * 4;
        o[0] = f; o[1] = g; o[2] = static_cast<double>(n_fg); o[3] = 0.0;
    }
}

bool valid_size(int h, int w) { return h > 0 && w > 0; }
bool supported_size(int h, int w) { return static_cast<long long>(h) * w < (1ll << 31) && w <= kMaxWidth; }

int launch_wfm(const void* pred_u8, const void* gt_u8, int n, MetricGeo geo, int max_h, int max_w, long long max_tiles,
               long long px, long long tiles, const int64_t* head, const double* coef, void* workspace, size_t workspace_bytes,
               double* sums, int32_t* nearest_yx, void* stream) {
    const WfmLayout lay = wfm_layout(px, tiles, n);
    SOD_CHECK_ARG(static_cast<long long>(workspace_bytes) >= lay.total, SOD_EWORKSPACE);
    SOD_CHECK_ARG(aligned16(workspace), SOD_EALIGN);
    SOD_CHECK_ARG(n <= 65535 && max_tiles <= 0x7fffffffll, SOD_EUNSUPPORTED);
    WfmParams p;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    p.pred = static_cast<const unsigned char*>(pred_u8);
    p.gt = static_cast<const unsigned char*>(gt_u8);
    p.geo = geo;
    p.head = reinterpret_cast<const long long*>(head);
    p.col = reinterpret_cast<int*>(ws + lay.col);
    p.stack = reinterpret_cast<int2*>(ws + lay.stack);
    p.near = nearest_yx != nullptr ? reinterpret_cast<int2*>(nearest_yx) : reinterpret_cast<int2*>(ws + lay.near);
    p.et = ws + lay.et;
    p.part = reinterpret_cast<double*>(ws + lay.part);
    p.ticket = reinterpret_cast<unsigned*>(ws + lay.ticket);
    p.sums = sums;
    for (int i = 0; i < 49; ++i) p.k[i] = coef[i];
    p.log_half_over_5 = coef[49];
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const unsigned gy = static_cast<unsigned>(n);
    wfm_column_kernel<<<dim3(static_cast<unsigned>(cdiv_ll(max_w, kColThreads)), gy), kColThreads, 0, s>>>(p);
    wfm_row_kernel<<<dim3(static_cast<unsigned>(cdiv_ll(max_h, kRowThreads)), gy), kRowThreads, 0, s>>>(p);
    wfm_weighted_kernel<<<dim3(static_cast<unsigned>(max_tiles), gy), kTileThreads, 0, s>>>(p);
    return static_cast<int>(cudaGetLastError());
}

}  // namespace
}  // namespace sod

extern "C" size_t sod_saliency_wfm_workspace_bytes(int n, const int32_t* hw_host) {
    using namespace sod;
    if (n <= 0 || !hw_host) return 0;
    long long px = 0, tiles = 0;
    for (int i = 0; i < n; ++i) {
        const int h = hw_host[2 * i], w = hw_host[2 * i + 1];
        if (!valid_size(h, w) || !supported_size(h, w)) return 0;
        px += static_cast<long long>(h) * w;
        tiles += image_tiles(h, w);
    }
    return static_cast<size_t>(wfm_layout(px, tiles, n).total);
}

extern "C" int sod_saliency_wfm(const void* pred_u8, const void* gt_u8, int n, int h, int w, const int64_t* head,
                                const double* coef_host, void* workspace, size_t workspace_bytes, double* sums,
                                int32_t* nearest_yx, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred_u8 && gt_u8 && head && coef_host && workspace && sums && n > 0 && valid_size(h, w), SOD_EINVAL);
    SOD_CHECK_ARG(supported_size(h, w), SOD_EUNSUPPORTED);
    const long long px = static_cast<long long>(n) * h * w, tiles = static_cast<long long>(n) * image_tiles(h, w);
    return launch_wfm(pred_u8, gt_u8, n, MetricGeo{nullptr, nullptr, h, w}, h, w, image_tiles(h, w), px, tiles, head,
                      coef_host, workspace, workspace_bytes, sums, nearest_yx, stream);
}

extern "C" int sod_saliency_wfm_ragged(const void* pred_u8, const void* gt_u8, int n, const int64_t* offsets,
                                       const int32_t* hw, const int32_t* hw_host, const int64_t* head,
                                       const double* coef_host, void* workspace, size_t workspace_bytes, double* sums,
                                       int32_t* nearest_yx, void* stream) {
    using namespace sod;
    SOD_CHECK_ARG(pred_u8 && gt_u8 && offsets && hw && hw_host && head && coef_host && workspace && sums && n > 0, SOD_EINVAL);
    int max_h = 0, max_w = 0;
    long long px = 0, tiles = 0, max_tiles = 0;
    for (int i = 0; i < n; ++i) {
        const int h = hw_host[2 * i], w = hw_host[2 * i + 1];
        SOD_CHECK_ARG(valid_size(h, w), SOD_EINVAL);
        SOD_CHECK_ARG(supported_size(h, w), SOD_EUNSUPPORTED);
        max_h = h > max_h ? h : max_h;
        max_w = w > max_w ? w : max_w;
        px += static_cast<long long>(h) * w;
        tiles += image_tiles(h, w);
        max_tiles = image_tiles(h, w) > max_tiles ? image_tiles(h, w) : max_tiles;
    }
    return launch_wfm(pred_u8, gt_u8, n, MetricGeo{reinterpret_cast<const long long*>(offsets), hw, 0, 0}, max_h, max_w,
                      max_tiles, px, tiles, head, coef_host, workspace, workspace_bytes, sums, nearest_yx, stream);
}
