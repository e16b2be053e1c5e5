// api.cu — version / error strings / device probe of libsod_b200.so.
#include <mutex>

#include "common.cuh"

namespace sod {

const DevInfo& dev_info() {
    static DevInfo cache[64];
    static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    std::lock_guard<std::mutex> lock(mu);
    DevInfo& d = cache[dev];
    if (d.sm_count == 0) {
        cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev);
        cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
        cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaDeviceGetAttribute(&d.l2_bytes, cudaDevAttrL2CacheSize, dev);
    }
    return d;
}

}  // namespace sod

extern "C" int sod_version(void) { return SOD_ABI_VERSION; }

extern "C" const char* sod_strerror(int code) {
    switch (code) {
        case SOD_OK: return "ok";
        case SOD_EINVAL: return "invalid argument (null pointer, non-positive size or bad enum)";
        case SOD_EALIGN: return "pointer or offset is not 16-byte aligned";
        case SOD_EWORKSPACE: return "workspace too small";
        case SOD_EUNSUPPORTED: return "unsupported shape / dtype combination or not an sm_90 device";
        case SOD_ECOMM: return "invalid communicator";
        default: break;
    }
    if (code > 0) return cudaGetErrorString(static_cast<cudaError_t>(code));
    return "unknown error";
}

extern "C" int sod_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) return static_cast<int>(e);
    if (n == 0) return static_cast<int>(cudaErrorNoDevice);
    const sod::DevInfo& d = sod::dev_info();
    if (sm_count) *sm_count = d.sm_count;
    if (cc_major) *cc_major = d.cc_major;
    if (cc_minor) *cc_minor = d.cc_minor;
    return SOD_OK;
}

extern "C" size_t sod_comm_flag_bytes(void) {
    return sizeof(uint32_t) * SOD_COMM_CHANNELS * SOD_COMM_MAX_BLOCKS * SOD_MAX_WORLD;
}
