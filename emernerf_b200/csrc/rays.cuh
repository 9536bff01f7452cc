// The ray of one pixel, shared by gen_rays_kernel (raygen.cu) and pixel_batch_kernel (raybatch.cu), so the two produce
// the same origins, view directions and norms bit for bit.  Arithmetic in the reference's order
// (datasets/base/pixel_source.py:39-76; -fmad=false: every product and sum rounds separately):
//     cam = ((x - cx + 0.5) / fx, (y - cy + 0.5) / fy, 1)
//     dir_i = cam_0 R[i][0] + cam_1 R[i][1] + cam_2 R[i][2];  norm = sqrt(sum dir_i^2);  viewdir = dir / (norm + 1e-8)
//     origin = c2w[:3, 3]
#pragma once
#include "common.cuh"

namespace emer {

// C: the camera's c2w [4, 4], K: its intrinsics [3, 3] (row-major, device memory); (px, py): the pixel.
__device__ __forceinline__ void pixel_ray(const float* __restrict__ C, const float* __restrict__ K, float px, float py,
                                          float origin[3], float viewdir[3], float& nrm) {
    const float cam[3] = {(px - __ldg(K + 2) + 0.5f) / __ldg(K + 0), (py - __ldg(K + 5) + 0.5f) / __ldg(K + 4), 1.0f};
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

}  // namespace emer
