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

// inclusive warp scan from the top lane downwards (suffix sum)
__device__ __forceinline__ float warp_scan_incl_rev(float v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_down_sync(0xffffffffu, v, o);
        if (lane + o < 32) v += t;
    }
    return v;
}

}  // namespace emer
