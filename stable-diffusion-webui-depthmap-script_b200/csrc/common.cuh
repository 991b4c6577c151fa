// Shared helpers for the depthmap_b200 C-ABI library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/depthmap_b200.h"

namespace dm {

void set_error(const char *fmt, ...);
int cuda_fail(cudaError_t e, const char *what);

#define DM_CUDA_CHECK(expr)                                   \
    do {                                                      \
        cudaError_t _e = (expr);                              \
        if (_e != cudaSuccess) return ::dm::cuda_fail(_e, #expr); \
    } while (0)

#define DM_LAUNCH_CHECK(name)                                         \
    do {                                                              \
        cudaError_t _e = cudaGetLastError();                          \
        if (_e != cudaSuccess) return ::dm::cuda_fail(_e, name);      \
    } while (0)

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// "have I configured this kernel on the current device yet?"  cudaFuncSetAttribute is per device, so the flag is a bit per
// device ordinal, set atomically (ADVICE r1: a process-wide bool skipped the call on the second GPU of a process).
struct PerDeviceFlag {
    unsigned long long mask = 0;
    bool test_and_set() {
        int d = 0;
        cudaGetDevice(&d);
        const unsigned long long bit = 1ull << (d & 63);
        const unsigned long long old = __atomic_fetch_or(&mask, bit, __ATOMIC_ACQ_REL);
        return (old & bit) != 0;
    }
};

// a device attribute read once per device ordinal (0 = not read yet; every attribute cached this way is positive)
struct PerDeviceAttr {
    int value[64] = {};
    cudaDeviceAttr attr;
    explicit PerDeviceAttr(cudaDeviceAttr a) : attr(a) {}
    int get() {
        int d = 0;
        cudaGetDevice(&d);
        int v = __atomic_load_n(&value[d & 63], __ATOMIC_ACQUIRE);
        if (v == 0) {
            cudaDeviceGetAttribute(&v, attr, d);
            __atomic_store_n(&value[d & 63], v, __ATOMIC_RELEASE);
        }
        return v;
    }
};

// i mod n in [0, n) for any integer i (circular padding, n > 0)
__host__ __device__ __forceinline__ int wrap_index(int i, int n) {
    const int r = i % n;
    return r < 0 ? r + n : r;
}

// order-preserving float <-> uint32 maps so min/max reductions can use integer atomics
__device__ __forceinline__ uint32_t f32_to_ordered(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ordered_to_f32(uint32_t u) {
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ uint32_t warp_min_u32(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ uint32_t warp_max_u32(uint32_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace dm
