// Ray generation for a training batch: pixel indices -> world-space origins and unit view directions.
//
// Replaces datasets/base/pixel_source.py:39-76 (get_rays) together with the per-ray gathers in front of it
// (:716-719: c2w = cam_to_worlds[img_idx], intrinsics = intrinsics[img_idx]) and the pixel-coordinate / timestamp
// assembly of get_train_rays (:699, :711-712): one launch instead of ~15 small torch kernels and two [R,4,4] / [R,3,3]
// gathered copies.  The per-ray arithmetic is pixel_ray (rays.cuh), shared with the training-batch kernel of
// raybatch.cu.
// HBM-bound, 9 floats out per ray: trivial next to the render, it exists to keep the batch on the device.
#include "rays.cuh"

namespace emer {

__global__ void gen_rays_kernel(const int64_t* __restrict__ img_idx, const float* __restrict__ x,
                                const float* __restrict__ y, const float* __restrict__ c2w,
                                const float* __restrict__ intr, int per_ray_mats, const float* __restrict__ timestamps,
                                float height, float width, float* __restrict__ origins, float* __restrict__ viewdirs,
                                float* __restrict__ norms, float* __restrict__ pixel_coords,
                                float* __restrict__ out_times, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t m = img_idx ? img_idx[i] : (per_ray_mats ? i : 0);
    const float* C = c2w + m * 16;
    const float* K = intr + m * 9;
    const float px = __ldg(x + i), py = __ldg(y + i);
    float o[3], v[3], nrm;
    pixel_ray(C, K, px, py, o, v, nrm);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        origins[i * 3 + r] = o[r];
        viewdirs[i * 3 + r] = v[r];
    }
    if (norms) norms[i] = nrm;
    if (pixel_coords) {
        pixel_coords[i * 2 + 0] = py / height;            // (y / H, x / W): pixel_source.py:699
        pixel_coords[i * 2 + 1] = px / width;
    }
    if (out_times && timestamps) out_times[i] = __ldg(timestamps + m);
}

}  // namespace emer

using namespace emer;

extern "C" int emer_gen_rays(const int64_t* img_idx, const float* x, const float* y, const float* c2w, const float* intrinsics,
                             int per_ray_mats, const float* timestamps, int height, int width, float* origins,
                             float* viewdirs, float* norms, float* pixel_coords, float* out_times, int64_t n, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && y && c2w && intrinsics && origins && viewdirs, "emer_gen_rays: NULL pointer");
    EMER_REQUIRE(!pixel_coords || (height > 0 && width > 0), "emer_gen_rays: pixel coordinates need the image size");
    gen_rays_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(
        img_idx, x, y, c2w, intrinsics, per_ray_mats, timestamps, (float)height, (float)width, origins, viewdirs, norms, pixel_coords, out_times, n);
    return check_launch("emer_gen_rays");
}
