// The per-pixel arithmetic shared by gen_rays_kernel (raygen.cu), pixel_batch_kernel (raybatch.cu) and
// image_rays_kernel (errormap.cu), so they produce the same values bit for bit.
//
// The ray, in the reference's order (datasets/base/pixel_source.py:39-76; -fmad=false: every product and sum rounds
// separately):
//     cam = ((x - cx + 0.5) / fx, (y - cy + 0.5) / fy, 1)
//     dir_i = cam_0 R[i][0] + cam_1 R[i][1] + cam_2 R[i][2];  norm = sqrt(sum dir_i^2);  viewdir = dir / (norm + 1e-8)
//     origin = c2w[:3, 3]
#pragma once
#include "common.cuh"

namespace emer {

// C: the camera's c2w [4, 4] (row-major, device memory); (fx, cx, fy, cy): its intrinsics; (px, py): the pixel.
__device__ __forceinline__ void pixel_ray(const float* __restrict__ C, float fx, float cx, float fy, float cy, float px,
                                          float py, float origin[3], float viewdir[3], float& nrm) {
    const float cam[3] = {(px - cx + 0.5f) / fx, (py - cy + 0.5f) / fy, 1.0f};
    float d[3], sq = 0.0f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        float s = cam[0] * __ldg(C + r * 4 + 0);
        s = s + cam[1] * __ldg(C + r * 4 + 1);
        s = s + cam[2] * __ldg(C + r * 4 + 2);
        d[r] = s;
        sq = sq + s * s;
    }
    nrm = sqrtf(sq);
    const float inv = nrm + 1e-8f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        origin[r] = __ldg(C + r * 4 + 3);
        viewdir[r] = d[r] / inv;
    }
}

// K: the camera's intrinsics [3, 3] (row-major, device memory).
__device__ __forceinline__ void pixel_ray(const float* __restrict__ C, const float* __restrict__ K, float px, float py,
                                          float origin[3], float viewdir[3], float& nrm) {
    pixel_ray(C, __ldg(K + 0), __ldg(K + 2), __ldg(K + 4), __ldg(K + 5), px, py, origin, viewdir, nrm);
}

// y / HEIGHT for an integer tensor y: torch on CUDA divides a tensor by a host scalar as a * (1 / b)
// (div_true_kernel_cuda), so this is the product with the rounded reciprocal, not emer_gen_rays' quotient.
__device__ __forceinline__ float pixel_coord(float v, int size) { return v * __frcp_rn((float)size); }

// (y * downscale).long() of get_features (pixel_source.py:464-465): an fp32 product truncated toward zero; clamped so
// a scale that rounds up cannot read past the map (torch would raise an index error there).
__device__ __forceinline__ int64_t feature_cell(float v, float scale, int size) {
    return min((int64_t)(v * scale), (int64_t)size - 1);
}

// The feature rows of a CTA's rays, copied cooperatively: consecutive threads write consecutive floats.  row[r] is the
// offset in src of ray r's row, for the CTA's nr rays; dst holds their rows back to back.  Called by every thread,
// after a barrier that makes row[] visible.
__device__ __forceinline__ void copy_feature_rows(const float* __restrict__ src, const int64_t* row, int nr, int c,
                                                  float* __restrict__ dst, int n_threads) {
    for (int e = threadIdx.x; e < nr * c; e += n_threads) {
        const int r = e / c;
        dst[e] = __ldg(src + row[r] + (e - r * c));
    }
}

}  // namespace emer
