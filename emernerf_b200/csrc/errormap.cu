// Whole-image render rays and the pixel error map on the device.
//
// emer_image_rays is ScenePixelSource.get_render_rays (datasets/base/pixel_source.py:733-846) for one or more images
// in one launch, except the bicubic resize of the image, which stays torch's.  The ray, the pixel coordinates and the
// feature cell are rays.cuh's, the same code as emer_pixel_batch's; what is new here is the meshgrid, the intrinsics
// scaled by d, and the nearest-mode resize of the masks.
//
// emer_error_map and emer_error_map_normalize are update_pixel_error_maps (:491-517): the error of each pixel, written
// straight into the map, and the min-max normalisation over the whole map.  The minimum and maximum are folded into a
// workspace with integer atomics on the fp32 bit patterns: the errors are >= +0 (abs), or NaN, so their patterns
// order as unsigned integers like the values, with every NaN above +inf.  The minimum is kept as the maximum of the
// complemented patterns, so a zeroed workspace is the identity of both.
#include "cta_reduce.cuh"
#include "rays.cuh"

namespace emer {

constexpr int IMAGE_THREADS = 128;
constexpr int MAP_THREADS = 256;
constexpr int MAP_MAX_CTAS = 1024;

// workspace layout, in 32-bit words (EMER_ERRORMAP_WORKSPACE_BYTES)
constexpr int WS_NOT_MIN = 0;                      // max over the map of ~bits
constexpr int WS_MAX = 1;                          // max over the map of bits
constexpr int WS_MAP_TICKET = 2;                   // cta_reduce.cuh ticket of emer_error_map_normalize
static_assert(4 * 4 == EMER_ERRORMAP_WORKSPACE_BYTES, "workspace size");

// torch's nearest source index for interpolate(scale_factor=d) (UpSample.h, nearest_neighbor_compute_source_index):
// min(floor(dst * scale), size - 1), scale = (float)(1.0 / d), in fp32
__device__ __forceinline__ int nearest_source(int dst, float scale, int size) {
    return min((int)floorf((float)dst * scale), size - 1);
}

__global__ void __launch_bounds__(IMAGE_THREADS) image_rays_kernel(const EmerImageRaysIn a, const EmerImageRaysOut o) {
    __shared__ int64_t feat_row[IMAGE_THREADS];
    const int64_t plane = (int64_t)a.h * a.w, n = plane * a.n_images;
    const int64_t i0 = (int64_t)blockIdx.x * IMAGE_THREADS, i = i0 + threadIdx.x;
    if (i < n) {
        // meshgrid(arange(w), arange(h), indexing="xy"), flattened: x fastest
        const int64_t k = i / plane, rem = i - k * plane;
        const int y = (int)(rem / a.w), x = (int)(rem - (int64_t)y * a.w);
        const int64_t img = a.first_image + k;
        const float fx = (float)x, fy = (float)y;
        // intrinsics * d: torch's fp32 product of a tensor and a host scalar (K[2, 2] = 1 is not read)
        const float* K = a.intrinsics + img * 9;
        float org[3], dir[3], nrm;
        pixel_ray(a.c2w + img * 16, __ldg(K + 0) * a.downscale, __ldg(K + 2) * a.downscale,
                  __ldg(K + 4) * a.downscale, __ldg(K + 5) * a.downscale, fx, fy, org, dir, nrm);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            o.origins[i * 3 + r] = org[r];
            o.viewdirs[i * 3 + r] = dir[r];
        }
        o.norms[i] = nrm;
        o.pixel_coords[i * 2 + 0] = pixel_coord(fy, a.h);
        o.pixel_coords[i * 2 + 1] = pixel_coord(fx, a.w);
        if (o.timestamps) o.timestamps[i] = __ldg(a.timestamps + img);
        o.img_idx[i] = img;
        if (o.cam_idx) o.cam_idx[i] = __ldg(a.cam_ids + img);
        if (o.sky_masks || o.dynamic_masks) {
            const int sy = nearest_source(y, a.mask_scale_y, a.height), sx = nearest_source(x, a.mask_scale_x, a.width);
            const int64_t pix = (img * a.height + sy) * a.width + sx;
            if (o.sky_masks) o.sky_masks[i] = __ldg(a.sky_masks + pix);
            if (o.dynamic_masks) o.dynamic_masks[i] = __ldg(a.dynamic_masks + pix);
        }
        if (o.features) {
            const int64_t fr = feature_cell(fy, a.feat_scale_y, a.feat_h);
            const int64_t fc = feature_cell(fx, a.feat_scale_x, a.feat_w);
            feat_row[threadIdx.x] = ((img * a.feat_h + fr) * a.feat_w + fc) * a.feat_c;
        }
    }
    if (!o.features) return;
    __syncthreads();
    copy_feature_rows(a.features, feat_row, (int)min((int64_t)IMAGE_THREADS, n - i0), a.feat_c,
                      o.features + i0 * a.feat_c, IMAGE_THREADS);
}

__global__ void __launch_bounds__(MAP_THREADS) error_map_kernel(const float* __restrict__ gt,
                                                               const float* __restrict__ rgb,
                                                               const float* __restrict__ opacity, int64_t n,
                                                               float* __restrict__ map, uint32_t* ws) {
    __shared__ uint32_t sh[MAP_THREADS / 32];
    uint32_t hi = 0u, not_lo = 0u;
    for (int64_t i = (int64_t)blockIdx.x * MAP_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * MAP_THREADS) {
        // torch.abs(gt - pred).mean(dim=-1) on the CPU: the sum of the three in order, in fp32, then / 3
        float s = fabsf(__fsub_rn(__ldg(gt + i * 3 + 0), __ldg(rgb + i * 3 + 0)));
        s = __fadd_rn(s, fabsf(__fsub_rn(__ldg(gt + i * 3 + 1), __ldg(rgb + i * 3 + 1))));
        s = __fadd_rn(s, fabsf(__fsub_rn(__ldg(gt + i * 3 + 2), __ldg(rgb + i * 3 + 2))));
        float e = __fdiv_rn(s, 3.0f);
        // pixel_error_maps[dynamic_opacity > 0.1] *= 5: torch compares an fp32 tensor with 0.1 as fp32
        if (opacity && __ldg(opacity + i) > 0.1f) e = __fmul_rn(e, 5.0f);
        map[i] = e;
        const uint32_t b = __float_as_uint(e);
        hi = max(hi, b);
        not_lo = max(not_lo, ~b);
    }
    hi = block_max<MAP_THREADS / 32>(hi, sh);
    not_lo = block_max<MAP_THREADS / 32>(not_lo, sh);
    if (threadIdx.x == 0) {
        atomicMax(ws + WS_MAX, hi);
        atomicMax(ws + WS_NOT_MIN, not_lo);
    }
}

__global__ void __launch_bounds__(MAP_THREADS) error_map_normalize_kernel(float* __restrict__ map, int64_t n,
                                                                         uint32_t* ws) {
    // (m - m.min()) / (m.max() - m.min()) with 0-d CUDA tensors: subtractions and an IEEE division, each rounded
    const float lo = __uint_as_float(~__ldcg(ws + WS_NOT_MIN)), hi = __uint_as_float(__ldcg(ws + WS_MAX));
    const float range = __fsub_rn(hi, lo);
    for (int64_t i = (int64_t)blockIdx.x * MAP_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * MAP_THREADS)
        map[i] = __fdiv_rn(__fsub_rn(map[i], lo), range);
    // every CTA has read the extrema before it takes its ticket: the last one clears them
    if (!take_last_ticket(ws + WS_MAP_TICKET)) return;
    if (threadIdx.x == 0) {
        ws[WS_NOT_MIN] = 0u;
        ws[WS_MAX] = 0u;
    }
    release_ticket(ws + WS_MAP_TICKET);
}

static unsigned map_ctas(int64_t n) {
    const int64_t c = ceil_div(n, MAP_THREADS * 4);
    return (unsigned)(c < 1 ? 1 : (c < MAP_MAX_CTAS ? c : MAP_MAX_CTAS));
}

}  // namespace emer

using namespace emer;

extern "C" int emer_image_rays(const EmerImageRaysIn* in, const EmerImageRaysOut* out, void* stream) {
    EMER_REQUIRE(in && out, "emer_image_rays: NULL argument");
    EMER_REQUIRE(in->n_images >= 0 && in->first_image >= 0, "emer_image_rays: negative image index or count");
    EMER_REQUIRE(in->h > 0 && in->w > 0 && in->height > 0 && in->width > 0, "emer_image_rays: empty image");
    const int64_t n = in->n_images * in->h * in->w;
    if (n == 0) return 0;
    EMER_REQUIRE(in->c2w && in->intrinsics && out->origins && out->viewdirs && out->norms && out->pixel_coords &&
                     out->img_idx, "emer_image_rays: NULL pointer");
    EMER_REQUIRE(!out->sky_masks || in->sky_masks, "emer_image_rays: sky masks without a source");
    EMER_REQUIRE(!out->dynamic_masks || in->dynamic_masks, "emer_image_rays: dynamic masks without a source");
    EMER_REQUIRE(!out->timestamps || in->timestamps, "emer_image_rays: timestamps without a source");
    EMER_REQUIRE(!out->cam_idx || in->cam_ids, "emer_image_rays: camera ids without a source");
    EMER_REQUIRE(!out->features || (in->features && in->feat_h > 0 && in->feat_w > 0 && in->feat_c > 0 &&
                                    in->feat_c <= EMER_PIXEL_BATCH_MAX_FEATURES),
                 "emer_image_rays: features need a [N, h, w, C] map with 1 <= C <= %d", EMER_PIXEL_BATCH_MAX_FEATURES);
    image_rays_kernel<<<(unsigned)ceil_div(n, IMAGE_THREADS), IMAGE_THREADS, 0, (cudaStream_t)stream>>>(*in, *out);
    return check_launch("emer_image_rays");
}

extern "C" int emer_error_map(const float* gt, const float* rgb, const float* opacity, int64_t n, float* map,
                              void* workspace, void* stream) {
    EMER_REQUIRE(n >= 0, "emer_error_map: negative pixel count");
    if (n == 0) return 0;
    EMER_REQUIRE(gt && rgb && map && workspace, "emer_error_map: NULL pointer");
    error_map_kernel<<<map_ctas(n), MAP_THREADS, 0, (cudaStream_t)stream>>>(gt, rgb, opacity, n, map,
                                                                            (uint32_t*)workspace);
    return check_launch("emer_error_map");
}

extern "C" int emer_error_map_normalize(float* map, int64_t n, void* workspace, void* stream) {
    EMER_REQUIRE(n >= 0, "emer_error_map_normalize: negative size");
    EMER_REQUIRE(map && workspace, "emer_error_map_normalize: NULL pointer");
    error_map_normalize_kernel<<<map_ctas(n), MAP_THREADS, 0, (cudaStream_t)stream>>>(map, n, (uint32_t*)workspace);
    return check_launch("emer_error_map_normalize");
}
