// Shared helpers for libemer_b200 (sm_90a).  Compiled with -fmad=false: every fused
// multiply-add in this library is written explicitly (fmaf), everything else rounds per
// operation exactly like the fp32 torch ops of the reference, which is what makes sample
// offsets / grid indices reproducible bit for bit against the CPU oracle.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "emer_b200.h"

namespace emer {

void set_error(const char* fmt, ...);
int current_device();   // index of the CUDA runtime's current device (0..63)
int sm_count();         // multiprocessors of the current device (cached per device)

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return -2;
    }
    return 0;
}

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// CTAs of `kernel` resident per SM, queried once per device into `cache[device]`, never inside a graph capture (1 until then)
template <typename Kernel>
int resident_ctas(Kernel kernel, int threads, size_t smem, cudaStream_t stream, int* cache) {
    int& c = cache[current_device()];
    if (c == 0) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        int v = 0;
        if (cudaStreamIsCapturing(stream, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) return 1;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, kernel, threads, smem) != cudaSuccess || v < 1) v = 1;
        c = v;
    }
    return c;
}

#define EMER_REQUIRE(cond, ...)          \
    do {                                 \
        if (!(cond)) {                   \
            emer::set_error(__VA_ARGS__); \
            return -1;                   \
        }                                \
    } while (0)

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// inclusive warp scan (sum)
__device__ __forceinline__ float warp_scan_incl(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

__device__ __forceinline__ double warp_scan_incl(double v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        double t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// min(a, b) that returns NaN when either is NaN (fminf returns the other operand)
__device__ __forceinline__ float fmin_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// inclusive warp scan (minimum); a NaN reaches every lane above it, as it does in a sum
__device__ __forceinline__ float warp_scan_min(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = fmin_nan(v, t);
    }
    return v;
}

// exclusive warp scan (sum) from the inclusive one: the inclusive sum of the lane below.  Never incl - v: where v
// outweighs the lanes below by 2^24 (a far interval's sigma * delta after near-empty space) that difference is 0.
__device__ __forceinline__ float warp_scan_excl(float incl, int lane) {
    const float below = __shfl_up_sync(0xffffffffu, incl, 1);
    return lane == 0 ? 0.0f : below;
}

// inclusive warp scan from the top lane downwards (suffix sum)
__device__ __forceinline__ float warp_scan_incl_rev(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_down_sync(0xffffffffu, v, o);
        if (lane + o < 32) v += t;
    }
    return v;
}

// exclusive suffix sum from the inclusive one: the inclusive suffix sum of the lane above (0 on lane 31), for the same
// reason as warp_scan_excl -- an opaque sample's term can outweigh the suffix behind it by 2^24.
__device__ __forceinline__ float warp_scan_excl_rev(float incl_rev, int lane) {
    const float above = __shfl_down_sync(0xffffffffu, incl_rev, 1);
    return lane == 31 ? 0.0f : above;
}

// Layer activations (EMER_ACT_*); the backward takes the stored OUTPUT y.
__device__ __forceinline__ float act_fwd(float v, int act) {
    if (act == EMER_ACT_RELU) return v > 0.0f ? v : 0.0f;
    if (act == EMER_ACT_SIGMOID) return 1.0f / (1.0f + expf(-v));
    return v;
}

__device__ __forceinline__ float act_bwd(float g, float y, int act) {
    if (act == EMER_ACT_RELU) return y > 0.0f ? g : 0.0f;
    if (act == EMER_ACT_SIGMOID) return g * (y * (1.0f - y));
    return g;
}

// Density activation trunc_exp(raw - 1) of the reference (radiance_fields/radiance_field.py:828-835); its backward
// clamps the exponent at 15.
__device__ __forceinline__ float density_fwd(float raw) { return expf(raw - 1.0f); }
__device__ __forceinline__ float density_bwd(float g, float raw) { return g * expf(fminf(raw - 1.0f, 15.0f)); }

}  // namespace emer
