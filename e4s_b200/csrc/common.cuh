// Shared helpers for the e4s_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include "../../include/e4s_b200.h"

#define E4S_NUM_SMS 132  // H100 SXM: fallback SM count when no device can be queried

#define E4S_REQUIRE(cond, code) \
    do {                        \
        if (!(cond)) return (code); \
    } while (0)

// Launch-error check that never synchronises: reports bad launch configuration only.
static inline int e4s_launch_status() {
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) {
        cudaGetLastError();  // clear
        return (int)e;
    }
    return E4S_OK;
}

static inline bool e4s_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static inline int64_t e4s_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Per-DEVICE host-side caches.  The opt-in to more than 48 KB of dynamic shared memory (cudaFuncSetAttribute) and the SM
// count belong to a device, not to the process: a process that launches on a second GPU must opt in again there and
// size its persistent grids from that GPU.  Lock-free (relaxed atomics; a racing thread at worst repeats the cheap call).
constexpr int E4S_MAX_DEVICES = 64;
static inline int e4s_current_device() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess) {
        cudaGetLastError();
        d = 0;
    }
    return (d >= 0 && d < E4S_MAX_DEVICES) ? d : 0;
}
static inline int e4s_num_sms() {
    static std::atomic<int> cache[E4S_MAX_DEVICES];
    const int d = e4s_current_device();
    int n = cache[d].load(std::memory_order_relaxed);
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || n <= 0) {
            cudaGetLastError();
            n = E4S_NUM_SMS;
        }
        cache[d].store(n, std::memory_order_relaxed);
    }
    return n;
}
// the most dynamic shared memory a block may opt in to (227 KB on an H100 when no device can be queried)
static inline int e4s_smem_optin_limit() {
    static std::atomic<int> cache[E4S_MAX_DEVICES];
    const int d = e4s_current_device();
    int n = cache[d].load(std::memory_order_relaxed);
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMaxSharedMemoryPerBlockOptin, d) != cudaSuccess || n <= 0) {
            cudaGetLastError();
            n = 227 * 1024;
        }
        cache[d].store(n, std::memory_order_relaxed);
    }
    return n;
}
// CTAs of `threads` threads with `smem` bytes of dynamic shared memory that fit on one SM, for one static cache per
// kernel instantiation: the last answer per device is kept as (smem << 8 | CTAs), so a launch with the same shared
// memory as the previous one makes no driver query.  0 when the query fails.
struct E4sOccupancy {
    std::atomic<int64_t> last[E4S_MAX_DEVICES];
};
template <typename Kernel>
static inline int e4s_ctas_per_sm(E4sOccupancy& st, Kernel kernel, int threads, size_t smem) {
    const int d = e4s_current_device();
    const int64_t v = st.last[d].load(std::memory_order_relaxed);
    if (v && (size_t)(v >> 8) == smem) return (int)(v & 0xFF);
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    st.last[d].store(((int64_t)smem << 8) | (n & 0xFF), std::memory_order_relaxed);
    return n;
}
struct E4sSmemOptIn {            // one static instance per kernel instantiation
    std::atomic<size_t> bytes[E4S_MAX_DEVICES];
};
template <typename Kernel>
static inline int e4s_smem_optin(E4sSmemOptIn& st, Kernel kernel, size_t smem) {
    const int d = e4s_current_device();
    if (smem <= 48 * 1024 || smem <= st.bytes[d].load(std::memory_order_relaxed)) return E4S_OK;
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return (int)cudaGetLastError();
    st.bytes[d].store(smem, std::memory_order_relaxed);
    return E4S_OK;
}

// Streaming 128-bit accesses: data touched once should not pollute L1.
__device__ __forceinline__ float4 ld_stream_f4(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ void st_stream_f4(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z),
                 "f"(v.w)
                 : "memory");
}
__device__ __forceinline__ float ld_stream_f1(const float* p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

__device__ __forceinline__ float lrelu_scaled(float v, float alpha, float scale) {
    return (v > 0.f ? v : v * alpha) * scale;
}
