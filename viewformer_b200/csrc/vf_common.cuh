// Shared helpers for libvf_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/vf_b200.h"

void vf_set_error(const char* fmt, ...);

// One-time configuration that belongs to a DEVICE, not to the process: cudaFuncSetAttribute acts on the current device's context, so a
// second device used by the same process needs its own call.  Usage:
//     static vf_per_device_flag flag;  bool& configured = flag.current();  if (!configured) { ...; configured = true; }
struct vf_per_device_flag {
    static constexpr int kMaxDevices = 64;
    bool done[kMaxDevices] = {};
    bool& current() {
        int d = 0;
        if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= kMaxDevices) d = 0;
        return done[d];
    }
};

#define VF_CHECK_ARG(cond, ...)                                  \
    do {                                                         \
        if (!(cond)) {                                           \
            vf_set_error(__VA_ARGS__);                           \
            return VF_ERR_ARG;                                   \
        }                                                        \
    } while (0)

#define VF_CHECK_LAUNCH(name)                                                        \
    do {                                                                             \
        cudaError_t e__ = cudaGetLastError();                                        \
        if (e__ != cudaSuccess) {                                                    \
            vf_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));    \
            return VF_ERR_CUDA;                                                      \
        }                                                                            \
    } while (0)

static inline cudaStream_t vf_s(vf_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

__device__ __forceinline__ float vf_gelu_erf(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float vf_swish(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float vf_relu(float x) { return x < 0.0f ? 0.0f : x; }      // a NaN stays NaN (fmaxf would return 0)

// Stateless dropout hash: element i of a tensor dropped with `seed` is kept when mix32(seed * 0x9E3779B97F4A7C15 + i) >= thr,
// thr = vf_drop_threshold(rate).  vf_dropout and the fused attention kernels share it, so they drop the same elements.
__device__ __forceinline__ uint32_t mix32(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
    return (uint32_t)k;
}
__host__ __device__ __forceinline__ uint32_t vf_drop_threshold(float rate) { return (uint32_t)fminf(rate * 4294967296.0f, 4294967295.0f); }
__device__ __forceinline__ bool vf_drop_keep(unsigned long long seed, unsigned long long i, uint32_t thr) {
    return mix32(seed * 0x9E3779B97F4A7C15ULL + i) >= thr;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
