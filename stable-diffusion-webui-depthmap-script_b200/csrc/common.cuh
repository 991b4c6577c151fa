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

// Ragged batches (include/depthmap_b200.h): the host descriptors must lie inside a buffer of `size` units, `unit` units per pixel
// (3 bytes of a uint8 RGB input, 1 float of an fp32 output), and the device copy must be 16-byte aligned (read as one record).
// Sets the largest h and w.  Runs before any launch.
static inline int check_ragged(const char *who, const void *buf, long long size, const dm_ragged_image *host, const dm_ragged_image *dev,
                               int B, int unit, int *max_h, int *max_w) {
    if (!buf || !host || !dev || B <= 0 || size < 0) { set_error("%s: bad arguments (null buffer or descriptor, or B <= 0)", who); return DM_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(dev) % 16) { set_error("%s: the device descriptors must be 16-byte aligned", who); return DM_E_INVALID; }
    int mh = 0, mw = 0;
    for (int i = 0; i < B; ++i) {
        const dm_ragged_image d = host[i];
        if (d.h <= 0 || d.w <= 0 || d.offset < 0 || d.offset > size || (long long)d.h * d.w * unit > size - d.offset) {
            set_error("%s: image %d (offset %lld, %d x %d) does not lie inside the buffer of %lld", who, i, (long long)d.offset, d.h, d.w, size);
            return DM_E_INVALID;
        }
        mh = d.h > mh ? d.h : mh;
        mw = d.w > mw ? d.w : mw;
    }
    if (max_h) *max_h = mh;
    if (max_w) *max_w = mw;
    return DM_OK;
}

// DepthModel.infer_pil's reflect pad of an n-pixel side, int(sqrt(n / 2) * 3) in float64 (numpy's arithmetic: both roots are
// correctly rounded)
__host__ __device__ __forceinline__ int zoe_pad_of(int n) { return (int)(sqrt((double)n / 2.0) * 3.0); }

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
