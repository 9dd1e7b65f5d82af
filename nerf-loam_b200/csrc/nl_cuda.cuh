// Small CUDA helpers shared by the kernels of libnerfloam_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <mutex>

#include "nl_error.h"

#define NL_CHECK_LAUNCH(what)                                                        \
    do {                                                                             \
        cudaError_t e__ = cudaGetLastError();                                        \
        if (e__ != cudaSuccess) {                                                    \
            char buf__[256];                                                         \
            std::snprintf(buf__, sizeof(buf__), "%s: %s", what, cudaGetErrorString(e__)); \
            return nl_set_error_code(NL_ERR_CUDA, buf__);                            \
        }                                                                            \
    } while (0)

static inline int nl_div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// One-time per-DEVICE initialisation (cudaFuncSetAttribute is per device): `flag` is a function-local static of the caller.
// Returns true when the calling thread has to (and may) run the initialisation for the current device; thread-safe.
struct NlPerDevice {
    static constexpr int MAX_DEV = 64;
    std::mutex mu;
    bool done[MAX_DEV] = {};
    template <class F>
    cudaError_t once(F &&init) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        if (dev < 0 || dev >= MAX_DEV) return cudaErrorInvalidDevice;
        std::lock_guard<std::mutex> lock(mu);
        if (done[dev]) return cudaSuccess;
        e = init();
        if (e == cudaSuccess) done[dev] = true;
        return e;
    }
};

// Number of SMs of the current device (132 on H100 SXM); cached.
static inline int nl_num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (sms <= 0) sms = 132;
    }
    return sms;
}

__device__ __forceinline__ float nl_bf16_to_f32(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }
// round-to-nearest-even fp32 -> bf16 (finite inputs; NaN kept quiet)
__device__ __forceinline__ uint16_t nl_f32_to_bf16(float f) {
    uint32_t u = __float_as_uint(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40u);
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
}
__device__ __forceinline__ float nl_round_bf16(float f) { return nl_bf16_to_f32(nl_f32_to_bf16(f)); }
