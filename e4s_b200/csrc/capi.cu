// Library identity / capability entry points of the C ABI (include/e4s_b200.h).
#include "common.cuh"

extern "C" int e4s_version(void) { return 300; /* 0.3.0: RealESRNet x4 kernels */ }

extern "C" const char* e4s_build_arch(void) { return "sm_90a"; }

extern "C" int e4s_device_ok(void) {
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        return E4S_ERR_ARCH;
    }
    int major = 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
        cudaGetLastError();
        return E4S_ERR_ARCH;
    }
    int minor = 0;
    if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) {
        cudaGetLastError();
        return E4S_ERR_ARCH;
    }
    return (major == 9 && minor == 0) ? E4S_OK : E4S_ERR_ARCH;
}

// ---- run-to-run bit reproducibility of the tensor-core convolutions -------------------------------------------------------
// The forward kernels of csrc/modconv_tc.cu accumulate every output in a fixed order, so they are bit reproducible with the
// switch on or off; it is kept so that callers can state the requirement (and for any future kernel that needs it).
// Initial value: environment variable E4S_B200_DETERMINISTIC (1 / 0).
#include <atomic>
#include <cstdlib>
static std::atomic<int> g_deterministic{-1};

extern "C" int e4s_get_deterministic(void) {
    int v = g_deterministic.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("E4S_B200_DETERMINISTIC");
        v = (e && atoi(e) != 0) ? 1 : 0;
        g_deterministic.store(v, std::memory_order_relaxed);
    }
    return v;
}

extern "C" int e4s_set_deterministic(int on) {
    g_deterministic.store(on ? 1 : 0, std::memory_order_relaxed);
    return E4S_OK;
}
