// common.cuh — device helpers shared by the sm_90a kernels of libsod_b200.so.
#pragma once
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "sod_b200.h"

namespace sod {

namespace cg = cooperative_groups;

#define SOD_CHECK_ARG(cond, code) \
    do {                          \
        if (!(cond)) return (code); \
    } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ------------------------------------------------------------------------------------------------
// device properties (cached per device)
// ------------------------------------------------------------------------------------------------
struct DevInfo {
    int sm_count = 0, cc_major = 0, cc_minor = 0, max_smem_optin = 0, l2_bytes = 0;
};
const DevInfo& dev_info();  // api.cu

// ------------------------------------------------------------------------------------------------
// saliency metrics: the layout and the ground-truth rule shared by the histogram (pipeline.cu) and the weighted
// F-measure (wfm.cu) kernels
// ------------------------------------------------------------------------------------------------
// Where image b lives: a batch of equal-size images (off == nullptr: image b at b·h·w, every image h × w) or a ragged
// batch (byte offsets and (h, w) per image).  Prediction and ground truth share the layout.
struct MetricGeo {
    const long long* off;
    const int* hw;
    int h, w;
    __device__ __forceinline__ void get(int b, size_t& base, int& hh, int& ww) const {
        if (off != nullptr) { base = static_cast<size_t>(off[b]); hh = hw[2 * b]; ww = hw[2 * b + 1]; }
        else { base = static_cast<size_t>(b) * h * w; hh = h; ww = w; }
    }
};

// gt_bin = (gt / (max + 1e-8) > 0.5): with integer gt this is 2·gt > max (the 1e-8 cannot move an integer comparison
// unless 2·gt == max, where gt / (max + 1e-8) < 0.5 — i.e. strictly greater is exact); max == 0 → all background
__device__ __forceinline__ bool metric_fg(int g, int gmax) { return gmax > 0 && 2 * g > gmax; }

// ------------------------------------------------------------------------------------------------
// 8-element packets: one 16-byte transaction for 16-bit types, two for fp32
// ------------------------------------------------------------------------------------------------
template <typename T>
struct IO;

template <>
struct IO<float> {
    static constexpr int kBytes = 4;
    __device__ __forceinline__ static void load8(const float* p, float (&f)[8]) {
        const float4 a = *reinterpret_cast<const float4*>(p);
        const float4 b = *reinterpret_cast<const float4*>(p + 4);
        f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    }
    __device__ __forceinline__ static void store8(float* p, const float (&f)[8]) {
        *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
        *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
    }
    __device__ __forceinline__ static float load1(const float* p) { return *p; }
    __device__ __forceinline__ static void store1(float* p, float v) { *p = v; }
    struct Raw { float4 a, b; };
    __device__ __forceinline__ static Raw load_raw(const float* p) {
        Raw r; r.a = *reinterpret_cast<const float4*>(p); r.b = *reinterpret_cast<const float4*>(p + 4); return r;
    }
    __device__ __forceinline__ static void unpack(const Raw& r, float (&f)[8]) {
        f[0] = r.a.x; f[1] = r.a.y; f[2] = r.a.z; f[3] = r.a.w; f[4] = r.b.x; f[5] = r.b.y; f[6] = r.b.z; f[7] = r.b.w;
    }
};

template <>
struct IO<__nv_bfloat16> {
    static constexpr int kBytes = 2;
    __device__ __forceinline__ static void load8(const __nv_bfloat16* p, float (&f)[8]) {
        const uint4 u = *reinterpret_cast<const uint4*>(p);
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 t = __bfloat1622float2(h[i]);
            f[2 * i] = t.x; f[2 * i + 1] = t.y;
        }
    }
    __device__ __forceinline__ static void store8(__nv_bfloat16* p, const float (&f)[8]) {
        uint4 u;
        __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
        *reinterpret_cast<uint4*>(p) = u;
    }
    __device__ __forceinline__ static float load1(const __nv_bfloat16* p) { return __bfloat162float(*p); }
    __device__ __forceinline__ static void store1(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
    using Raw = uint4;
    __device__ __forceinline__ static Raw load_raw(const __nv_bfloat16* p) { return *reinterpret_cast<const uint4*>(p); }
    __device__ __forceinline__ static void unpack(const Raw& u, float (&f)[8]) {
        const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 t = __bfloat1622float2(h[i]);
            f[2 * i] = t.x; f[2 * i + 1] = t.y;
        }
    }
};

template <>
struct IO<__half> {
    static constexpr int kBytes = 2;
    __device__ __forceinline__ static void load8(const __half* p, float (&f)[8]) {
        const uint4 u = *reinterpret_cast<const uint4*>(p);
        const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 t = __half22float2(h[i]);
            f[2 * i] = t.x; f[2 * i + 1] = t.y;
        }
    }
    __device__ __forceinline__ static void store8(__half* p, const float (&f)[8]) {
        uint4 u;
        __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        *reinterpret_cast<uint4*>(p) = u;
    }
    __device__ __forceinline__ static float load1(const __half* p) { return __half2float(*p); }
    __device__ __forceinline__ static void store1(__half* p, float v) { *p = __float2half_rn(v); }
    using Raw = uint4;
    __device__ __forceinline__ static Raw load_raw(const __half* p) { return *reinterpret_cast<const uint4*>(p); }
    __device__ __forceinline__ static void unpack(const Raw& u, float (&f)[8]) {
        const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 t = __half22float2(h[i]);
            f[2 * i] = t.x; f[2 * i + 1] = t.y;
        }
    }
};

// dtype dispatch: FN is a generic lambda taking a value of the element type as a tag
#define SOD_DISPATCH_DTYPE(dt, T, ...)                                        \
    [&]() -> int {                                                            \
        switch (dt) {                                                         \
            case SOD_F32: { using T = float; return __VA_ARGS__(); }          \
            case SOD_BF16: { using T = __nv_bfloat16; return __VA_ARGS__(); } \
            case SOD_F16: { using T = __half; return __VA_ARGS__(); }         \
            default: return (int)SOD_EINVAL;                                  \
        }                                                                     \
    }()

// ------------------------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA engine without a tensor map; SASS: UBLKCP / SYNCS)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// same copy with an L2 eviction-priority hint (the 64-bit policy encodings CUTLASS uses for TMA loads on sm_90+)
constexpr uint64_t kL2EvictFirst = 0x12F0000000000000ull;   // last use: let it go first
constexpr uint64_t kL2EvictLast = 0x14F0000000000000ull;    // will be read again: keep if possible
__device__ __forceinline__ void bulk_g2s_hint(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar,
                                              uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}
constexpr uint64_t kL2EvictNormal = 0x1000000000000000ull;
// 16-byte global store with an L2 eviction-priority hint
__device__ __forceinline__ void st16_hint(void* p, uint4 v, uint64_t policy) {
    asm volatile("st.global.L2::cache_hint.v4.b32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w),
                 "l"(policy)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    }
}

// ------------------------------------------------------------------------------------------------
// system-scope flag traffic and NVLS (multimem) accesses for the peer-memory collectives
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_v2(void* p, uint32_t a, uint32_t b) {
    asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint2 ld_relaxed_sys_v2(const void* p) {
    uint2 v;
    asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 multimem_ld_reduce_add_f32x4(const void* mc_ptr) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(mc_ptr)
                 : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st_f32x4(void* mc_ptr, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_ptr), "f"(v.x),
                 "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ void multimem_st_b64(void* mc_ptr, uint32_t a, uint32_t b) {
    const uint64_t v = (static_cast<uint64_t>(b) << 32) | a;
    asm volatile("multimem.st.relaxed.sys.global.b64 [%0], %1;" ::"l"(mc_ptr), "l"(v) : "memory");
}
__device__ __forceinline__ float4 ld_peer_f32x4(const void* p) {
    float4 v;
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ void st_peer_f32x4(void* p, float4 v) {
    asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y),
                 "f"(v.z), "f"(v.w)
                 : "memory");
}

// Device-side view of sod_comm. Signal area at the head of every arena:
//   uint32 flags[SOD_COMM_CHANNELS][SOD_COMM_MAX_BLOCKS][SOD_MAX_WORLD]
struct CommDev {
    int rank, world;
    uint64_t peer[SOD_MAX_WORLD];
    uint64_t mc;
    uint32_t* error_flag;
    unsigned long long timeout_cycles;
    uint32_t* block_seq;
};

static inline int make_comm_dev(const sod_comm* c, CommDev& d) {
    if (c == nullptr) {
        d.rank = 0; d.world = 1; d.mc = 0; d.error_flag = nullptr; d.timeout_cycles = 0; d.block_seq = nullptr;
        for (int i = 0; i < SOD_MAX_WORLD; ++i) d.peer[i] = 0;
        return SOD_OK;
    }
    if (c->world < 1 || c->world > SOD_MAX_WORLD || c->rank < 0 || c->rank >= c->world) return SOD_ECOMM;
    d.rank = c->rank; d.world = c->world; d.mc = c->mc; d.error_flag = c->error_flag; d.block_seq = c->block_seq;
    if (c->world > 1 && c->block_seq == nullptr) return SOD_ECOMM;
    d.timeout_cycles = c->timeout_cycles ? c->timeout_cycles : 40000000000ull;  // ~20 s at 2 GHz
    for (int i = 0; i < SOD_MAX_WORLD; ++i) d.peer[i] = (i < c->world) ? c->peer[i] : 0;
    for (int i = 0; i < c->world; ++i)
        if (d.peer[i] == 0 || (d.peer[i] & 15u)) return SOD_ECOMM;
    return SOD_OK;
}

__device__ __forceinline__ uint32_t* comm_flag(uint64_t arena, int channel, int block, int src_rank) {
    return reinterpret_cast<uint32_t*>(arena) +
           ((static_cast<size_t>(channel) * SOD_COMM_MAX_BLOCKS + block) * SOD_MAX_WORLD + src_rank);
}

// Barrier between block `block` of every rank on `channel`: on return every peer's block has reached
// the same call (release/acquire at system scope, so peer writes issued before it are visible).
// The sequence number lives in device memory (c.block_seq) and is advanced here, identically on all
// ranks because every rank issues the same calls with the same grids. Returns false on timeout.
__device__ __forceinline__ bool comm_block_barrier(const CommDev& c, int channel, int block) {
    __shared__ int s_ok;
    __shared__ uint32_t s_val;
    if (threadIdx.x == 0) {
        s_ok = 1;
        uint32_t* slot = c.block_seq + channel * SOD_COMM_MAX_BLOCKS + block;
        s_val = *slot + 1u;
        *slot = s_val;
    }
    __syncthreads();
    const uint32_t value = s_val;
    if (threadIdx.x < static_cast<unsigned>(c.world)) {
        const int peer = threadIdx.x;
        __threadfence_system();
        st_release_sys(comm_flag(c.peer[peer], channel, block, c.rank), value);
        const uint32_t* mine = comm_flag(c.peer[c.rank], channel, block, peer);
        const long long t0 = clock64();
        while (static_cast<int32_t>(ld_acquire_sys(mine) - value) < 0) {
            if (static_cast<unsigned long long>(clock64() - t0) > c.timeout_cycles) {
                if (c.error_flag) atomicExch(c.error_flag, 0xDEAD0000u | static_cast<uint32_t>(channel));
                s_ok = 0;
                break;
            }
        }
    }
    __syncthreads();
    return s_ok != 0;
}

}  // namespace sod
