// membench.cu — streaming-read microbenchmark used to choose the SyncBN staging scheme (tools only).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o membench membench.cu && ./membench
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void bulk(void* d, const void* s, uint32_t bytes, uint64_t* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(d)), "l"(s), "r"(bytes), "r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t par) {
    uint32_t done = 0;
    while (!done) asm volatile("{.reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0,1,0,p;}" : "=r"(done) : "r"(smem_u32(b)), "r"(par) : "memory");
}

// ---- variant A: one producer thread, TMA ring, all threads consume -------------------------------------------------
__global__ void __launch_bounds__(512, 1) tma_ring(const uint4* __restrict__ src, size_t bytes_per_cta, int chunk, int nstage, float* out, int producer_warp) {
    extern __shared__ __align__(128) unsigned char sm[];
    uint64_t* full = (uint64_t*)sm; uint64_t* empty = full + 32;
    unsigned char* st = sm + 512;
    const int tid = threadIdx.x;
    const char* base = (const char*)src + (size_t)blockIdx.x * bytes_per_cta;
    const int n = (int)(bytes_per_cta / chunk);
    const int nconsumer_warps = producer_warp ? 15 : 16;
    if (tid == 0) { for (int s = 0; s < nstage; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], nconsumer_warps); } asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    float acc = 0.f;
    if (producer_warp && tid >= 480) {   // dedicated producer warp (warp 15)
        if (tid == 480) {
            uint32_t epar = 0;
            for (int i = 0; i < n; ++i) {
                const int s = i % nstage;
                if (i >= nstage) { mbar_wait(&empty[s], (epar >> s) & 1); epar ^= 1u << s; }
                mbar_expect(&full[s], chunk); bulk(st + (size_t)s * chunk, base + (size_t)i * chunk, chunk, &full[s]);
            }
        }
    } else {
        if (!producer_warp && tid == 0) for (int i = 0; i < (n < nstage ? n : nstage); ++i) { mbar_expect(&full[i], chunk); bulk(st + (size_t)i * chunk, base + (size_t)i * chunk, chunk, &full[i]); }
        uint32_t fpar = 0, epar = 0;
        const int nthr = producer_warp ? 480 : 512;
        for (int i = 0; i < n; ++i) {
            const int s = i % nstage;
            mbar_wait(&full[s], (fpar >> s) & 1); fpar ^= 1u << s;
            const uint4* p = (const uint4*)(st + (size_t)s * chunk);
            for (int q = tid; q < chunk / 16; q += nthr) { uint4 v = p[q]; acc += __uint_as_float(v.x) + __uint_as_float(v.y) + __uint_as_float(v.z) + __uint_as_float(v.w); }
            if (producer_warp) { __syncwarp(); if ((tid & 31) == 0) mbar_arrive(&empty[s]); }
            else if (i + nstage < n) {
                __syncwarp(); if ((tid & 31) == 0) mbar_arrive(&empty[s]);
                if (tid == 0) { mbar_wait(&empty[s], (epar >> s) & 1); epar ^= 1u << s; mbar_expect(&full[s], chunk); bulk(st + (size_t)s * chunk, base + (size_t)(i + nstage) * chunk, chunk, &full[s]); }
            }
        }
    }
    if (acc == 123.456f) out[0] = acc;
}

// ---- variant B: plain LDG.128 streaming, UNROLL loads in flight per thread -----------------------------------------
template <int UNROLL>
__global__ void ldg_stream(const uint4* __restrict__ src, size_t nvec, float* out) {
    float acc = 0.f;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + (UNROLL - 1) * stride < nvec; i += UNROLL * stride) {
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(src + i + u * stride));
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) acc += __uint_as_float(v[u].x) + __uint_as_float(v[u].y) + __uint_as_float(v[u].z) + __uint_as_float(v[u].w);
    }
    if (acc == 123.456f) out[0] = acc;
}
// contiguous-per-CTA variant of B (each CTA owns a contiguous slice, like the BN strips)
template <int UNROLL>
__global__ void ldg_strip(const uint4* __restrict__ src, size_t vec_per_cta, float* out) {
    float acc = 0.f;
    const uint4* p = src + (size_t)blockIdx.x * vec_per_cta;
    for (size_t i = threadIdx.x; i + (UNROLL - 1) * blockDim.x < vec_per_cta; i += UNROLL * blockDim.x) {
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(p + i + u * blockDim.x));
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) acc += __uint_as_float(v[u].x) + __uint_as_float(v[u].y) + __uint_as_float(v[u].z) + __uint_as_float(v[u].w);
    }
    if (acc == 123.456f) out[0] = acc;
}
// streaming copy (read + write), the shape of phase 2
template <int UNROLL>
__global__ void copy_strip(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t vec_per_cta) {
    const uint4* p = src + (size_t)blockIdx.x * vec_per_cta; uint4* d = dst + (size_t)blockIdx.x * vec_per_cta;
    for (size_t i = threadIdx.x; i + (UNROLL - 1) * blockDim.x < vec_per_cta; i += UNROLL * blockDim.x) {
        uint4 v[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) v[u] = p[i + u * blockDim.x];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) d[i + u * blockDim.x] = v[u];
    }
}

template <typename F> float timeit(F f, int iters = 10) {
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    f(); cudaDeviceSynchronize();
    cudaEventRecord(a); for (int i = 0; i < iters; ++i) f(); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b); return ms / iters;
}

int main() {
    const size_t total = 1ull << 30;  // 1 GiB source: far larger than L2
    uint4* src; uint4* dst; float* out; cudaMalloc(&src, total); cudaMalloc(&dst, total); cudaMalloc(&out, 4); cudaMemset(src, 1, total);
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    printf("SMs %d\n", sms);
    cudaFuncSetAttribute(tma_ring, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
    for (int pw = 0; pw < 2; ++pw)
        for (int chunk : {4096, 8192, 16384, 32768})
            for (int stages : {4, 8, 12, 24, 48}) {
                if ((size_t)chunk * stages > 200 * 1024 || stages > 32) continue;
                size_t per = (total / sms) / chunk * chunk;
                float ms = timeit([&] { tma_ring<<<sms, 512, 512 + chunk * stages>>>(src, per, chunk, stages, out, pw); });
                printf("tma_ring producer_warp=%d chunk=%5d stages=%2d inflight=%3zuKB : %7.1f GB/s\n", pw, chunk, stages, (size_t)chunk * stages / 1024, per * sms / ms / 1e6);
            }
    for (int mult : {1, 2, 4, 8}) for (int thr : {256, 512, 1024}) {
        size_t nvec = total / 16;
        float ms = timeit([&] { ldg_stream<4><<<sms * mult, thr>>>(src, nvec, out); });
        float ms8 = timeit([&] { ldg_stream<8><<<sms * mult, thr>>>(src, nvec, out); });
        printf("ldg_stream ctas=%dxSM thr=%4d : unroll4 %7.1f GB/s  unroll8 %7.1f GB/s\n", mult, thr, total / ms / 1e6, total / ms8 / 1e6);
    }
    for (int mult : {1, 2, 4}) for (int thr : {512, 1024}) {
        size_t vpc = total / 16 / (sms * mult);
        float ms = timeit([&] { ldg_strip<8><<<sms * mult, thr>>>(src, vpc, out); });
        float msc = timeit([&] { copy_strip<4><<<sms * mult, thr>>>(src, dst, vpc); });
        printf("ldg_strip ctas=%dxSM thr=%4d unroll8: %7.1f GB/s | copy_strip unroll4: %7.1f GB/s (r+w)\n", mult, thr, vpc * 16.0 * sms * mult / ms / 1e6, 2.0 * vpc * 16.0 * sms * mult / msc / 1e6);
    }
    cudaError_t e = cudaDeviceSynchronize(); printf("status %s\n", cudaGetErrorString(e));
    return 0;
}
